"""GPU tests of the marginalization at the sizes a cfg-4 window (20 keyframes, 2000 landmarks) produces: the workspace sized by the batch
rather than by the handle, the 8-CTA cluster eigensolver (marg_jacobi_cluster, 160 < n <= 320), split-pipeline handles, and the call-time
limit of 512 rows.  The numerical contract is tests/test_marg_gpu.py's compare().  Each test asserts the m and r it got, i.e. which
eigensolver kernel served the marginalized block (Hmm, n = m) and the remained block (Hp, n = r):
    n <= 118: one CTA;  n <= 160: cluster pair;  n <= 320: 8-CTA cluster;  n <= 512: global memory."""
import copy
import os

import numpy as np
import pytest

from datagen import synth_ba
from tests import oracle_api as oa
from tests import post_solve_oracle as po
from tests.test_marg_gpu import compare
from tests.test_post_solve_gpu import CAMD, STD, cull_inputs, next_window, oracle_gvins

pytestmark = pytest.mark.gpu

KEYS = ("block_type", "block_node", "x0", "J0", "e0", "Hp", "bp")
_WINDOWS = {}


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def cam():
    from ic_gvins_b200.camera import Camera
    return Camera([CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"]], [0.0, 0.0, 0.0, 0.0])


def window_prior(prob, truth, seed):
    """a synthetic prior over pose_k, mix_k (k < K - 1), the extrinsic and td, around the true values: the blocks a sliding window's prior
    spans once it has slid a few times (15 (K - 1) + 7 = 292 rows at K = 20).  J0 = (3 I + small upper-triangular coupling) diag(scale),
    well conditioned at any size; e0 small.  Marginalizing node 0 then leaves r = 15 (K - 2) + 7 = 277 rows at K = 20 (the 8-CTA cluster)."""
    K = prob["K"]
    n = K - 1
    rng = np.random.default_rng(seed)
    types = np.array([0, 1] * n + [2, 3], np.int32)
    nodes = np.array([k for k in range(n) for _ in range(2)] + [0, 0], np.int32)
    scale = np.concatenate([np.concatenate([[10.0] * 6, [5.0] * 3, [2000.0] * 3, [500.0] * 3]) for _ in range(n)] + [[50.0] * 6, [100.0]])
    r = scale.size
    A = 3.0 * np.eye(r) + np.triu(rng.normal(0, 0.5 / np.sqrt(r), (r, r)), 1)
    x0 = np.concatenate([np.concatenate([truth["pose"][k], truth["mix"][k]]) for k in range(n)] + [truth["ext"][:7], [0.0]])
    prob.update(marg_r=r, marg_nblocks=len(types), marg_block_type=types, marg_block_node=nodes, marg_x0=x0,
                marg_J0=(A * scale[None, :]).reshape(-1).copy(), marg_e0=rng.normal(0, 0.1, r))
    return prob


def make(olib, prior=False, **kw):
    """a fresh copy of a generated window (a cfg-4 window takes about a second to generate: each is made once per module); prior=True adds
    window_prior"""
    key = tuple(sorted(kw.items()))
    if key not in _WINDOWS:
        _WINDOWS[key] = synth_ba.make_window(lambda *a: oa.preintegrate(olib, *a), **kw)
    prob, truth = copy.deepcopy(_WINDOWS[key])
    return window_prior(prob, truth, kw.get("seed", 0) + 1) if prior else prob


def handle(max_windows=2, max_K=20, max_L=2000, max_F=12000, max_marg_r=292):
    from ic_gvins_b200.ba import WindowSolver
    return WindowSolver(max_windows=max_windows, max_K=max_K, max_L=max_L, max_F=max_F, max_gnss=16, max_marg_r=max_marg_r)


@pytest.fixture(scope="module")
def s4():
    """a cfg-4 handle (split pipeline: max_K > 14) that can consume its own 292-row prior"""
    s = handle()
    yield s
    s.close()


def assert_bitwise(a, b):
    assert a["m"] == b["m"] and a["r"] == b["r"]
    for key in KEYS:
        assert np.array_equal(a[key], b[key]), key


def scaled_gap(a, b, o):
    """largest difference of the scaled Schur complement and of J0^T J0 between two device results (o: the oracle's, for the scale)"""
    sc = np.sqrt(np.abs(np.diag(o["Hp"])))
    sc[sc == 0] = 1
    dH = np.abs((a["Hp"] - b["Hp"]) / np.outer(sc, sc)).max()
    dJ = np.abs((a["J0"].T @ a["J0"] - b["J0"].T @ b["J0"]) / np.outer(sc, sc)).max()
    return dH, dJ


def with_env(name, fn):
    os.environ[name] = "1"
    try:
        return fn()
    finally:
        del os.environ[name]


def test_result_does_not_depend_on_the_handle_capacity(olib):
    """a cfg-3 window on max_L = 300 and on max_L = 2000 (the workspace follows the batch, not the capacity): equal bit for bit, through the
    uploading and the resident call"""
    prob = make(olib, K=10, L=300, seed=11, with_marg=True)
    solved = copy.deepcopy(prob)
    s = handle(max_windows=1, max_K=10, max_L=300, max_F=2700, max_marg_r=160)
    try:
        s.gvins_optimization_batch([solved], 20)
    finally:
        s.close()
    out = []
    for max_L in (300, 2000):
        s = handle(max_windows=1, max_K=10, max_L=max_L, max_F=2700, max_marg_r=160)
        try:
            up = s.marginalize([copy.deepcopy(solved)], 1)[0]
            s.upload([copy.deepcopy(solved)])
            res = s.marginalize([copy.deepcopy(solved)], 1, resident=True)[0]
        finally:
            s.close()
        assert up["m"] <= 118 and up["r"] <= 118  # the one-CTA kernel for both blocks
        assert_bitwise(up, res)
        out.append(up)
    assert_bitwise(out[0], out[1])
    compare(out[1], oa.ba_marginalize(olib, copy.deepcopy(solved), 1), tol_sqrt=1e-8)


def test_cfg4_window_against_the_oracle(olib, s4):
    """K = 20, L = 2000, default anchoring, a 292-row prior: about 400 landmarks leave with node 0 (Hmm on the global kernel), r = 277 (Hp
    on the cluster)"""
    p = make(olib, K=20, L=2000, seed=2040, prior=True)
    s4.gvins_optimization_batch([p], 20)
    res = s4.marginalize([p], 1, resident=True)[0]
    assert 320 < res["m"] <= 512 and res["r"] == 277
    up = s4.marginalize([copy.deepcopy(p)], 1)[0]
    assert_bitwise(res, up)
    o = oa.ba_marginalize(olib, copy.deepcopy(p), 1)
    compare(res, o, tol_sqrt=1e-8)  # as tests/test_marg_gpu.py's resident test: an eigenvalue within rounding of EPS = 1e-8 may split either way
    glob = with_env("ICG_MARG_GLOBAL_JACOBI", lambda: s4.marginalize([copy.deepcopy(p)], 1)[0])
    assert glob["m"] == res["m"] and glob["r"] == res["r"]
    dH, dJ = scaled_gap(glob, up, o)
    assert dH < 1e-9 and dJ < 1e-9, (dH, dJ)


def test_marginalized_block_in_the_cluster_size_class(olib, s4):
    """K = 20, L = 1000, default anchoring, a 292-row prior: about 200 landmarks on node 0 put Hmm on the cluster kernel too"""
    p = make(olib, K=20, L=1000, seed=2041, prior=True)
    g = s4.marginalize([copy.deepcopy(p)], 1)[0]
    assert 160 < g["m"] <= 320 and g["r"] == 277
    compare(g, oa.ba_marginalize(olib, copy.deepcopy(p), 1), tol_sqrt=1e-8)


def test_cluster_kernel_agrees_at_cfg3(olib):
    """ICG_MARG_CLUSTER_JACOBI sends cfg-3 blocks (which the one-CTA and pair kernels take by default) to the cluster kernel"""
    prob = make(olib, K=10, L=300, seed=23, with_marg=True)
    s = handle(max_windows=1, max_K=10, max_L=300, max_F=2700, max_marg_r=160)
    try:
        base = s.marginalize(copy.deepcopy(prob), 1)[0]
        alt = with_env("ICG_MARG_CLUSTER_JACOBI", lambda: s.marginalize(copy.deepcopy(prob), 1)[0])
    finally:
        s.close()
    assert alt["m"] == base["m"] and alt["r"] == base["r"] and alt["m"] <= 160 and alt["r"] <= 160
    o = oa.ba_marginalize(olib, copy.deepcopy(prob), 1)
    compare(alt, o)
    dH, dJ = scaled_gap(alt, base, o)
    assert dH < 1e-9 and dJ < 1e-9, (dH, dJ)


def test_chain_at_cfg4(olib, cam):
    """a window with a 292-row prior: gvins_optimization -> cull -> culled marginalization -> solve of the K = 19 window with the new
    277-row prior, all on a split-pipeline handle; the same chain on the oracle.  Anchors spread over 19 nodes (about 105 landmarks leave
    with node 0)"""
    prob = make(olib, K=20, L=2000, seed=2042, n_ref=20, prior=True)
    fc = prob["f_const"].reshape(-1, 14)
    rows = np.random.default_rng(2043).choice(prob["F"], size=25, replace=False)
    fc[rows, 3] += np.random.default_rng(2044).uniform(3, 40, 25) / synth_ba.F_PIX  # pixel outliers in pts1
    prob["ext_const"], prob["td_const"] = 1, 1  # as test_chain_into_the_next_window_solve
    ci = cull_inputs(prob, prob["ext"].copy(), 2045, bad_kp=30)
    pg, pq = copy.deepcopy(prob), copy.deepcopy(prob)
    s = handle(max_windows=1)
    try:
        s.gvins_optimization_batch([pg], 20)
        g = s.update_and_cull([pg], cam, STD, [ci])[0]
        mg = s.marginalize([pg], 1, resident=True, culled=[g])[0]
        qg = next_window(pg, mg, po.culled_factor_mask(pg, ci, g, np.ones(20, np.uint8)))
        sg = s.solve(qg, 10)[0]
    finally:
        s.close()
    assert mg["m"] <= 160 and mg["r"] == 277
    oracle_gvins(olib, pq, 20)
    assert np.array_equal(pg["f_active"], pq["f_active"])
    o = po.update_and_cull(pq, CAMD, STD, ci)
    assert np.array_equal(o["lm_outlier"], g["lm_outlier"]) and np.array_equal(o["obs_outlier"], g["obs_outlier"])
    mq = copy.deepcopy(pq)
    mq["f_active"] = po.culled_factor_mask(pq, ci, o, np.ones(20, np.uint8))
    mo = oa.ba_marginalize(olib, mq, 1)
    qo = next_window(pq, mo, mq["f_active"])
    so = oa.ba_solve(olib, qo, 10)
    assert mg["m"] == mo["m"] and mg["r"] == mo["r"] and np.array_equal(mg["block_type"], mo["block_type"])
    assert np.array_equal(mg["block_node"], mo["block_node"])
    sc = np.sqrt(np.abs(np.diag(mo["Hp"])))
    sc[sc == 0] = 1
    assert np.abs((mg["Hp"] - mo["Hp"]) / np.outer(sc, sc)).max() < 5e-6 and np.abs((mg["bp"] - mo["bp"]) / sc).max() < 5e-6
    assert sg["iterations"] == so["iterations"]
    assert abs(sg["final_cost"] - so["final_cost"]) <= 2e-4 * so["final_cost"]
    for key in ("pose", "mix", "ext", "invdepth"):
        assert np.abs(qg[key] - qo[key]).max() <= 2e-4 * max(1.0, np.abs(qo[key]).max()), key


def test_block_beyond_the_largest_kernel_is_rejected_and_leaves_the_handle_as_it_was(olib):
    """num_marg = 2 on a cfg-4 window (about 800 landmarks leave): ICG_EUNSUPPORTED naming the window and its m, before anything runs; the
    handle then re-solves and marginalizes one node bit for bit like a handle that never saw the call"""
    from ic_gvins_b200 import IcgError
    prob = make(olib, K=20, L=2000, seed=2040)

    def run(fail_first):
        s = handle(max_windows=1)
        try:
            p = copy.deepcopy(prob)
            s.gvins_optimization_batch([p], 20)
            if fail_first:
                with pytest.raises(IcgError, match=r"code -4: .*window 0: m=(\d+)") as e:
                    s.marginalize([p], 2, resident=True)
                m = int(str(e.value).split("window 0: m=")[1].split()[0])
                assert m > 512
            s.run_gvins(20, restart=True)
            return s.marginalize([p], 1, resident=True)[0]
        finally:
            s.close()

    a, b = run(True), run(False)
    assert 320 < a["m"] <= 512 and a["r"] <= 118
    assert_bitwise(a, b)


def test_mixed_batch_uses_one_kernel_per_stage(olib, s4):
    """a cfg-3 and a cfg-4 window in one batch: the batch's largest blocks choose the kernels (global for Hmm, cluster for Hp), so the
    cfg-3 window runs on other kernels than alone (one CTA for both); each window within 1e-9 of its solo call"""
    a = make(olib, K=10, L=300, seed=11, with_marg=True)
    b = make(olib, K=20, L=2000, seed=2040, prior=True)
    batch = s4.marginalize([copy.deepcopy(a), copy.deepcopy(b)], np.array([1, 1], np.int32))
    solo = [s4.marginalize([copy.deepcopy(x)], 1)[0] for x in (a, b)]
    assert solo[0]["m"] <= 118 and solo[0]["r"] <= 118
    assert 320 < solo[1]["m"] <= 512 and solo[1]["r"] == 277
    for x, g, s in zip((a, b), batch, solo):
        assert g["m"] == s["m"] and g["r"] == s["r"]
        assert np.array_equal(g["block_type"], s["block_type"]) and np.array_equal(g["x0"], s["x0"])
        o = oa.ba_marginalize(olib, copy.deepcopy(x), 1)
        dH, dJ = scaled_gap(g, s, o)
        assert dH < 1e-9 and dJ < 1e-9, (dH, dJ)
    assert_bitwise(solo[1], batch[1])  # the cfg-4 window takes the same kernels in both calls
