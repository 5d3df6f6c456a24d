"""GPU parity tests for the sliding-window marginalization (SURVEY 8a row B10) through the C ABI (icg_ba_marginalize),
against the CPU oracle restatement of MarginalizationInfo (oracle/ba_ref.cpp: marginalize).

What is compared: the block structure (bit-exact), the Schur complement Hp / bp (diag-scaled, the quantity both sides compute before
any eigenvector freedom enters), and the prior as a function -- J0^T J0 and J0^T e0 (invariant under the eigenvector sign / order
freedom of the decomposition).  Hp cancels ~1e4 : 1 against cond(Hmm) ~ 1e8, so two correct FP64 eigensolvers agree to ~1e-7
(see tests/test_oracle_marg.py, where numpy's eigh shows the same gap to the oracle); the end-to-end bar is the north_star's
1e-6 relative on the SOLUTION of the next window solve that consumes the prior."""
import copy
import os

import numpy as np
import pytest

from datagen import synth_ba
from tests import oracle_api as oa

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def solver():
    from ic_gvins_b200.ba import WindowSolver
    s = WindowSolver(max_windows=4, max_K=10, max_L=300, max_F=2700, max_gnss=16, max_marg_r=160)
    yield s
    s.close()


def make(olib, **kw):
    return synth_ba.make_window(lambda *a: oa.preintegrate(olib, *a), **kw)[0]


def compare(g, o, tol_h=5e-6, tol_sqrt=1e-9, sc_floor=0.0):
    """sc_floor: the smallest column scale.  A window with unobservable directions (a vehicle standing still) has Hp diagonals at rounding
    level (1e-25); scaled by their own square root, rounding differences look like O(1).  sqrt(EPS) = 1e-4 scales such a column as one at
    the pseudo-inverse cut, below which the prior keeps nothing of it."""
    assert g["m"] == o["m"] and g["r"] == o["r"]
    assert np.array_equal(g["block_type"], o["block_type"]) and np.array_equal(g["block_node"], o["block_node"])
    assert np.array_equal(g["x0"], o["x0"])
    sc = np.maximum(np.sqrt(np.abs(np.diag(o["Hp"]))), sc_floor)
    sc[sc == 0] = 1
    dH = np.abs((g["Hp"] - o["Hp"]) / np.outer(sc, sc)).max()
    db = np.abs((g["bp"] - o["bp"]) / sc).max() / max(1.0, np.abs(o["bp"] / sc).max())
    assert dH < tol_h and db < tol_h, (dH, db)
    # the prior as a function: 0.5 |e0 + J0 dx|^2 = 0.5 dx^T (J0^T J0) dx + (J0^T e0)^T dx + const
    dJ = np.abs((g["J0"].T @ g["J0"] - o["J0"].T @ o["J0"]) / np.outer(sc, sc)).max()
    de = np.abs((g["J0"].T @ g["e0"] - o["J0"].T @ o["e0"]) / sc).max() / max(1.0, np.abs(o["bp"] / sc).max())
    assert dJ < tol_h and de < tol_h, (dJ, de)
    # J0 is a valid square root of the GPU's own Hp (retained spectrum) to FP64 rounding
    S, U = np.linalg.eigh(g["Hp"])
    keep = S > 1e-8
    Hk = (U[:, keep] * S[keep]) @ U[:, keep].T
    assert np.abs((g["J0"].T @ g["J0"] - Hk) / np.outer(sc, sc)).max() < tol_sqrt
    # rows sorted by ascending eigenvalue (Eigen::SelfAdjointEigenSolver order)
    rn = (g["J0"] ** 2).sum(axis=1)
    assert np.all(np.diff(rn) >= -1e-9 * rn.max())
    return dH, db


@pytest.mark.parametrize("with_marg", [False, True])
def test_marginalize_matches_oracle(olib, solver, with_marg):
    prob = make(olib, K=10, L=300, seed=11, with_marg=with_marg)
    o = oa.ba_marginalize(olib, copy.deepcopy(prob), 1)
    g = solver.marginalize(copy.deepcopy(prob), 1)[0]
    compare(g, o)


def test_marginalize_batch_and_flags(olib, solver):
    """a batch of different windows (one with constant extrinsic / td and culled factors, one with first-window priors, one
    marginalizing two nodes) -- and the call must leave the handle usable for the next solve"""
    a = make(olib, K=10, L=300, seed=3)
    a["ext_const"], a["td_const"] = 1, 1
    a["f_active"][::7] = 0
    b = make(olib, K=6, L=80, seed=4)
    b.update(has_pose_prior=1, pose_prior=b["pose"][:7].copy(), pose_prior_std=np.array([0.1, 0.1, 0.1, 0.01, 0.01, 0.02]),
             has_mix_prior=1, mix_prior=b["mix"][:9].copy() + 1e-3, mix_prior_std=np.array([0.1] * 3 + [1e-4] * 3 + [1e-3] * 3))
    c = make(olib, K=8, L=150, seed=5, with_marg=True)
    probs = [a, b, c]
    nm = [1, 1, 2]
    # node 1 of window c must not anchor landmarks whose reference is removed while it observes: use the generator as is
    gs = solver.marginalize([copy.deepcopy(p) for p in probs], np.array(nm, np.int32))
    for p, k, g in zip(probs, nm, gs):
        o = oa.ba_marginalize(olib, copy.deepcopy(p), k)
        compare(g, o)
    # the handle still solves (dims flags restored)
    q = copy.deepcopy(a)
    s = solver.solve(q, 5)[0]
    qo = copy.deepcopy(a)
    so = oa.ba_solve(olib, qo, 5)
    assert abs(s["final_cost"] - so["final_cost"]) <= 1e-8 * so["final_cost"]


@pytest.mark.parametrize("K,L,seed", [(8, 120, 9), (10, 300, 19)])
def test_prior_feeds_the_next_window_solve(olib, solver, K, L, seed):
    """solve -> marginalize node 0 -> drop it -> solve the shrunken window with the new prior: GPU chain vs oracle chain, 1e-6 (the north-star
    bar on the solution; also at the cfg-3 size, free extrinsic + td)"""
    prob = make(olib, K=K, L=L, seed=seed)

    def chain(solve, marg):
        p = copy.deepcopy(prob)
        solve(p, 10)
        out = marg(p)
        keep_f = p["f_ref"] >= 1
        q = copy.deepcopy(p)
        q.update(K=p["K"] - 1, pose=p["pose"][7:].copy(), mix=p["mix"][9:].copy(), F=int(keep_f.sum()),
                 f_lm=p["f_lm"][keep_f].copy(), f_ref=(p["f_ref"][keep_f] - 1).astype(np.int32), f_obs=(p["f_obs"][keep_f] - 1).astype(np.int32),
                 f_const=p["f_const"].reshape(-1, 14)[keep_f].reshape(-1).copy(), f_active=p["f_active"][keep_f].copy(),
                 n_imu=p["n_imu"] - 1, imu_blob=p["imu_blob"][480:].copy(),
                 pn_off=(p["pn_off"][1:] - p["pn_off"][1]).astype(np.int32), pn=p["pn"][4 * p["pn_off"][1]:].copy())
        g = p["gnss_node"] >= 1
        q.update(n_gnss=int(g.sum()), gnss_node=(p["gnss_node"][g] - 1).astype(np.int32), gnss_blh=p["gnss_blh"].reshape(-1, 3)[g].reshape(-1).copy(),
                 gnss_std=p["gnss_std"].reshape(-1, 3)[g].reshape(-1).copy())
        q.update(marg_r=out["r"], marg_nblocks=len(out["block_type"]), marg_block_type=out["block_type"], marg_block_node=out["block_node"],
                 marg_x0=out["x0"], marg_J0=out["J0"].reshape(-1).copy(), marg_e0=out["e0"])
        # perturb so that the second solve has work to do and the prior matters
        q["pose"] = q["pose"].copy()
        q["pose"].reshape(-1, 7)[:, :3] += 0.05
        s = solve(q, 10)
        return q, s

    qg, sg = chain(lambda p, n: solver.solve(p, n)[0], lambda p: solver.marginalize(p, 1)[0])
    qo, so = chain(lambda p, n: oa.ba_solve(olib, p, n), lambda p: oa.ba_marginalize(olib, p, 1))
    assert sg["iterations"] == so["iterations"]
    assert abs(sg["final_cost"] - so["final_cost"]) <= 1e-6 * so["final_cost"]
    for key in ("pose", "mix", "ext", "invdepth"):
        assert np.abs(qg[key] - qo[key]).max() <= 1e-6 * max(1.0, np.abs(qo[key]).max()), key


def test_resident_marginalization_equals_the_uploading_call(olib, solver):
    """icg_ba_marginalize_resident (the windows the handle has just solved, nothing uploaded again) == icg_ba_marginalize on the written-back
    arrays, bit for bit: after the two-pass solve the device copy and the caller's arrays hold the same parameters, factor activity and GNSS sigmas."""
    probs = [make(olib, K=10, L=300, seed=41 + w) for w in range(3)]
    probs[1]["f_const"].reshape(-1, 14)[5, 3] += 0.2  # an outlier: the chi2 culling must reach the marginalization through the device copy
    solver.gvins_optimization_batch(probs, 20)
    res = solver.marginalize(probs, 1, resident=True)
    up = solver.marginalize([copy.deepcopy(p) for p in probs], 1)
    for a, b in zip(res, up):
        assert a["m"] == b["m"] and a["r"] == b["r"]
        for key in ("block_type", "block_node", "x0", "J0", "e0", "Hp", "bp"):
            assert np.array_equal(a[key], b[key]), key
    o = oa.ba_marginalize(olib, copy.deepcopy(probs[1]), 1)
    compare(res[1], o, tol_sqrt=1e-8)  # numpy's eigh and the device Jacobi split the spectrum at EPS = 1e-8 with an eigenvalue within rounding of it


@pytest.mark.parametrize("env", ["ICG_MARG_PAIR_JACOBI", "ICG_MARG_GLOBAL_JACOBI"])
def test_jacobi_kernel_variants_agree(olib, solver, env):
    """the three eigensolver kernels (single CTA for n <= 118, cluster pair for n <= 160, global memory beyond) are the same algorithm:
    each one against the oracle, and against the default within 1e-9 of the scaled Schur complement"""
    prob = make(olib, K=10, L=300, seed=23, with_marg=True)
    base = solver.marginalize(copy.deepcopy(prob), 1)[0]
    os.environ[env] = "1"
    try:
        alt = solver.marginalize(copy.deepcopy(prob), 1)[0]
    finally:
        del os.environ[env]
    o = oa.ba_marginalize(olib, copy.deepcopy(prob), 1)
    compare(alt, o)
    sc = np.sqrt(np.abs(np.diag(o["Hp"])))
    sc[sc == 0] = 1
    assert np.abs((alt["Hp"] - base["Hp"]) / np.outer(sc, sc)).max() < 1e-9
    assert np.abs((alt["J0"].T @ alt["J0"] - base["J0"].T @ base["J0"]) / np.outer(sc, sc)).max() < 1e-9
