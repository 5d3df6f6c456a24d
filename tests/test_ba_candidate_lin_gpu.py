"""Windows whose LM steps are rejected.  The single-GPU solve linearises every candidate into the window's second linearisation buffer and
takes the candidate cost from it; an accepted step flips the window's buffers, a rejected one must leave the linearisation at x in use.
These windows exercise the reject path (and its mix with accepts, per window, inside one batch) against the oracle."""
import copy

import numpy as np
import pytest

from datagen import synth_ba
from tests import oracle_api as oa

pytestmark = pytest.mark.gpu
ITERS = 12


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def solver():
    from ic_gvins_b200.ba import WindowSolver
    s = WindowSolver(max_windows=6, max_K=10, max_L=300, max_F=2700, max_gnss=16, max_marg_r=1)
    yield s
    s.close()


def rejecting_window(olib, kind, seed, K=10, L=150):
    """kind "outliers": no loss functions and 10 % of the reprojection factors moved by ~40 px; "perturbed": positions off by `sigma` m and
    inverse depths by a factor exp(N(0, 0.5))."""
    prob, _ = synth_ba.make_window(lambda *a: oa.preintegrate(olib, *a), K=K, L=L, seed=seed)
    rng = np.random.default_rng(seed)
    if kind == "outliers":
        prob["reproj_huber"], prob["gnss_huber"] = 0, 0
        fc = prob["f_const"].reshape(-1, 14)
        idx = rng.choice(prob["F"], prob["F"] // 10, replace=False)
        fc[idx, 3:5] += rng.normal(0, 0.05, (len(idx), 2))
    else:
        pose = prob["pose"].reshape(-1, 7)
        pose[:, :3] += rng.normal(0, kind, (K, 3))
        prob["invdepth"] *= np.exp(rng.normal(0, 0.5, L))
    return prob


CASES = [("outliers", 300), ("outliers", 303), (1.0, 301), (3.0, 304)]


@pytest.mark.parametrize("kind,seed", CASES)
def test_rejected_steps_match_oracle(olib, solver, kind, seed):
    prob = rejecting_window(olib, kind, seed)
    so = oa.ba_solve(olib, copy.deepcopy(prob), ITERS)
    sg = solver.solve(copy.deepcopy(prob), ITERS)[0]
    assert so["iterations"] > so["num_successful_steps"]  # the window rejects steps
    assert sg["iterations"] == so["iterations"] and sg["num_successful_steps"] == so["num_successful_steps"]
    assert sg["termination"] == so["termination"]
    assert abs(sg["initial_cost"] - so["initial_cost"]) <= 1e-9 * so["initial_cost"]


def test_rejecting_and_accepting_windows_in_one_batch_are_independent(olib, solver):
    """Windows that reject steps beside windows that accept them: the batch equals the windows solved one by one, bitwise (every window
    follows its own linearisation buffer)."""
    probs = [rejecting_window(olib, kind, seed) for kind, seed in CASES]
    for i in range(2):
        p, _ = synth_ba.make_window(lambda *a: oa.preintegrate(olib, *a), K=10, L=100 + 20 * i, seed=30 + i)
        p["ext_const"], p["td_const"] = 1, 1
        probs.insert(2 * i + 1, p)
    single, single_summ = [], []
    for p in probs:
        q = copy.deepcopy(p)
        single_summ.append(solver.solve(q, ITERS)[0])
        single.append(q)
    assert any(s["num_successful_steps"] < s["iterations"] for s in single_summ)
    batch = copy.deepcopy(probs)
    batch_summ = solver.solve(batch, ITERS)
    for a, b, sa, sb in zip(batch, single, batch_summ, single_summ):
        assert sa == sb
        for key in ("pose", "mix", "invdepth", "ext"):
            assert np.array_equal(a[key], b[key]), key
