"""The marginalization at the edges of its four eigensolver kernels, at the EPS cut of its pseudo-inverses, and on a window whose
marginalized block is degenerate.  The windows and the restated kernel rule are those of tests/test_marg_sizes.py; the numerical contract
against the oracle is tests/test_marg_gpu.py's compare().

Between kernels the bar is 1e-9 of the scaled Schur complement and of J0^T J0: same input, same rotation formula, ordering and stopping
rule, so the kernels differ by rounding only.  Each point prints one line (m, r, the kernels of the two stages, the largest scaled gap to
the oracle, the largest gap between kernels)."""
import copy
import os

import numpy as np
import pytest

from datagen import synth_ba
from tests import oracle_api as oa
from tests.test_marg_gpu import compare
from tests.test_marg_large_gpu import assert_bitwise, scaled_gap
from tests.test_marg_sizes import (DESIGNED_R, REJECTED, SWEEP, check_designed, designed_window, kernel_runs, select_kernel,
                                   sized_window)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


def handle():
    """room for every window of the sweep: K = 32 with a 487-row prior (r = 472 + node 0's 15), 540 landmarks at K = 10"""
    from ic_gvins_b200.ba import WindowSolver
    return WindowSolver(max_windows=2, max_K=32, max_L=540, max_F=2700, max_gnss=16, max_marg_r=487)


@pytest.fixture(scope="module")
def s():
    h = handle()
    yield h
    h.close()


def with_envs(env, fn):
    for name in env:
        os.environ[name] = "1"
    try:
        return fn()
    finally:
        for name in env:
            del os.environ[name]


_ORACLE = {}


def oracle_of(olib, m, r, seed=0):
    """the oracle's marginalization of sized_window(m, r, seed), computed once per module (about 10 s at m = 512)"""
    if (m, r, seed) not in _ORACLE:
        _ORACLE[m, r, seed] = oa.ba_marginalize(olib, sized_window(olib, m, r, seed), 1)
    return _ORACLE[m, r, seed]


def finite(g):
    return all(np.all(np.isfinite(g[k])) for k in ("J0", "e0", "Hp", "bp"))


@pytest.mark.parametrize("m,r", SWEEP)
def test_sweep_point_on_every_kernel(olib, s, m, r):
    """the default kernels against the oracle; every kernel that can take m and r (forced through ICG_MARG_*) against the default"""
    p = sized_window(olib, m, r)
    o = oracle_of(olib, m, r)
    runs = kernel_runs(m, r)
    base = s.marginalize(copy.deepcopy(p), 1)[0]
    assert (base["m"], base["r"]) == (m, r) and finite(base)
    # an eigenvalue of Hp within rounding of EPS may split either way between numpy's eigh and the device (tests/test_marg_gpu.py)
    dH, db = compare(base, o, tol_sqrt=1e-8)
    worst = 0.0
    for kern, env in runs.items():
        if not env:
            continue
        alt = with_envs(env, lambda: s.marginalize(copy.deepcopy(p), 1)[0])
        assert (alt["m"], alt["r"]) == (m, r) and finite(alt)
        gH, gJ = scaled_gap(alt, base, o)
        assert gH < 1e-9 and gJ < 1e-9, (kern, gH, gJ)
        worst = max(worst, gH, gJ)
    print(f"\nSWEEP m={m} r={r} default={select_kernel(m)}/{select_kernel(r)} runs={'+'.join(a + '/' + b for a, b in runs)} "
          f"oracle_dH={dH:.2e} oracle_db={db:.2e} kernel_gap={worst:.2e}")


# two windows on either side of a limit in one batch: the larger one chooses the stage's kernel for both, so the smaller one runs on
# another kernel than alone
MIXED = [((118, 64), (119, 64)), ((160, 64), (161, 64)), ((320, 64), (321, 64)), ((75, 118), (75, 121)), ((75, 160), (75, 163)),
         ((75, 319), (75, 322))]


@pytest.mark.parametrize("a,b", MIXED)
def test_mixed_batch_across_a_limit(olib, s, a, b):
    pa, pb = sized_window(olib, *a), sized_window(olib, *b, seed=1)
    batch = s.marginalize([copy.deepcopy(pa), copy.deepcopy(pb)], np.array([1, 1], np.int32))
    solo = [s.marginalize([copy.deepcopy(x)], 1)[0] for x in (pa, pb)]
    for seed, size, g, one in zip((0, 1), (a, b), batch, solo):
        assert (g["m"], g["r"]) == size and (one["m"], one["r"]) == size
        assert np.array_equal(g["block_type"], one["block_type"]) and np.array_equal(g["x0"], one["x0"])
        o = oracle_of(olib, *size, seed)
        dH, dJ = scaled_gap(g, one, o)
        assert dH < 1e-9 and dJ < 1e-9, (size, dH, dJ)
    assert select_kernel(max(a[0], b[0])) == select_kernel(b[0]) and select_kernel(max(a[1], b[1])) == select_kernel(b[1])
    assert select_kernel(a[0]) != select_kernel(b[0]) or select_kernel(a[1]) != select_kernel(b[1])
    assert_bitwise(solo[1], batch[1])  # the window at the larger size takes the same kernels in both calls


def test_largest_block_is_accepted_and_one_more_row_is_refused(olib):
    """m = 512 on the global-memory kernel against the oracle; m = 513 raises ICG_EUNSUPPORTED naming the window and its m, after which the
    handle marginalizes m = 512 bit for bit like a fresh handle"""
    from ic_gvins_b200 import IcgError
    ok, bad = sized_window(olib, 512, 64), sized_window(olib, *REJECTED)
    out = []
    for refuse_first in (True, False):
        h = handle()
        try:
            if refuse_first:
                with pytest.raises(IcgError, match=r"code -4: .*window 0: m=513 "):
                    h.marginalize(copy.deepcopy(bad), 1)
            out.append(h.marginalize(copy.deepcopy(ok), 1)[0])
        finally:
            h.close()
    assert out[0]["m"] == 512
    assert_bitwise(out[0], out[1])
    compare(out[0], oracle_of(olib, 512, 64), tol_sqrt=1e-8)


@pytest.mark.parametrize("m,r", [(118, 64), (75, 160), (320, 64), (512, 64), (75, 472)])
def test_resident_call_equals_the_uploading_call(olib, s, m, r):
    """one point per kernel (one-CTA, pair, 8-CTA cluster, global for Hmm and for Hp): icg_ba_marginalize_resident on the uploaded window
    == icg_ba_marginalize, bit for bit"""
    p = sized_window(olib, m, r)
    up = s.marginalize([copy.deepcopy(p)], 1)[0]
    s.upload([copy.deepcopy(p)])
    res = s.marginalize([copy.deepcopy(p)], 1, resident=True)[0]
    assert (up["m"], up["r"]) == (m, r)
    assert_bitwise(up, res)


@pytest.mark.parametrize("r", DESIGNED_R)
def test_designed_spectrum_is_cut_at_eps_on_every_kernel(olib, s, r):
    """Hp's designed block (exact zeros, 1e-12, 0.5 / 0.8 / 1.25 / 2 EPS, a 10-fold eigenvalue, 1e6) against its eigenpairs computed in
    numpy from the design: the rows kept, the rows dropped (exactly zero), J0^T J0 and J0^T e0 on the block, on every kernel that can take r"""
    p, info = designed_window(olib, r)
    worst = (0.0, 0.0)
    for kern, env in kernel_runs(55, r).items():
        g = with_envs(env, lambda: s.marginalize(copy.deepcopy(p), 1)[0])
        assert (g["m"], g["r"]) == (55, r) and finite(g)
        dJ, de = check_designed(g, info)
        worst = (max(worst[0], dJ), max(worst[1], de))
    print(f"\nDESIGNED r={r} kernels={'+'.join(b for _, b in kernel_runs(55, r))} dJ={worst[0]:.2e} de={worst[1]:.2e}")


def drop_node0(p, out):
    """the window without node 0 and with the prior `out` (tests/test_marg_gpu.py's chain), poses moved 0.05 m so the solve has work"""
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
    q["pose"] = q["pose"].copy()
    q["pose"].reshape(-1, 7)[:, :3] += 0.05
    return q


@pytest.mark.parametrize("n_ref,kernel", [(5, "cta"), (2, "cluster")])
def test_stationary_window(olib, s, n_ref, kernel):
    """a vehicle standing still (speed 0, yaw rate 0, no heave, no perturbation): node 0's landmarks have no parallax, their Hmm columns
    are at rounding level (1e-22 against 1e10) and marg_schur must gate them away.  Finite prior, the oracle's prior, and the next-window
    solve on it against the oracle chain at 1e-6.  Neither window is solved with its reprojection factors: without parallax the inverse
    depths and the extrinsic are unobservable and the solve amplifies rounding (a 1e-13 change of the start moves the oracle's own final
    cost by up to 30%), so the chain marginalizes the window as generated and solves the next one on its IMU, GNSS and the new prior"""
    prob = synth_ba.make_window(lambda *a: oa.preintegrate(olib, *a), K=10, L=300, seed=7500 + n_ref, n_ref=n_ref, speed=0.0, yaw_rate=0.0,
                                heave=False, perturb=False)[0]
    g = s.marginalize(copy.deepcopy(prob), 1)[0]
    assert select_kernel(g["m"]) == kernel and finite(g)
    # ext rotation / td (and, at rounding level, the ext translation) carry no information without motion: Hp diagonals ~1e-25
    compare(g, oa.ba_marginalize(olib, copy.deepcopy(prob), 1), tol_sqrt=1e-8, sc_floor=1e-4)

    def chain(solve, marg):
        p = copy.deepcopy(prob)
        q = drop_node0(p, marg(p))
        q.update(f_active=np.zeros_like(q["f_active"]), ext_const=1, td_const=1)
        return q, solve(q, 10)

    qg, sg = chain(lambda p, n: s.solve(p, n)[0], lambda p: s.marginalize(p, 1)[0])
    qo, so = chain(lambda p, n: oa.ba_solve(olib, p, n), lambda p: oa.ba_marginalize(olib, p, 1))
    assert np.isfinite(sg["final_cost"]) and sg["iterations"] == so["iterations"]
    assert abs(sg["final_cost"] - so["final_cost"]) <= 1e-6 * so["final_cost"]
    for key in ("pose", "mix"):
        assert np.abs(qg[key] - qo[key]).max() <= 1e-6 * max(1.0, np.abs(qo[key]).max()), key
