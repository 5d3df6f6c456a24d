"""GPU: icg_ba_slide_resident.  Each case slides one handle to the next window and uploads the same next window, with the carried values
filled in on the host, into a second handle; the two must then be indistinguishable: the two-pass solve (summaries, parameters, f_active,
gnss_std), a following resident marginalization (J0, e0, Hp, bp) and a re-solve with restart = 1 give the same bits."""
import copy

import numpy as np
import pytest

from tests import oracle_api as oa
from tests import post_solve_oracle as po
from tests.test_marg_large_gpu import make as make_large
from tests.test_post_solve_gpu import CAMD, STD, cull_inputs, make
from datagen.slide_window import build_next

pytestmark = pytest.mark.gpu

IMU = 480
PARAMS = ("pose", "mix", "ext", "invdepth", "f_active", "gnss_std")


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def cam():
    from ic_gvins_b200.camera import Camera
    return Camera([CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"]], [0.0, 0.0, 0.0, 0.0])


def handle(n=1, K=10, L=300, F=2700, R=160):
    from ic_gvins_b200.ba import WindowSolver
    return WindowSolver(max_windows=n, max_K=K, max_L=L, max_F=F, max_gnss=16, max_marg_r=R)


def compare_handles(s1, s2, slid, up, n_iter=20, marg=True):
    """s1 holds `slid` (slide done), s2 gets `up` uploaded: the two-pass solve, a resident marginalization and a restarted solve, bitwise"""
    s1.run_gvins(n_iter)
    r1 = s1.gvins_optimization_end(slid)
    r2 = s2.gvins_optimization_batch(up, n_iter)
    assert r1 == r2
    for a, b in zip(slid, up):
        for k in PARAMS:
            assert np.array_equal(a[k], b[k]), k
    if marg:
        m1, m2 = s1.marginalize(up, 1, resident=True), s2.marginalize(up, 1, resident=True)
        for a, b in zip(m1, m2):
            assert a["m"] == b["m"] and a["r"] == b["r"]
            for k in ("J0", "e0", "Hp", "bp"):
                assert np.array_equal(a[k], b[k]), k
    s1.run_gvins(n_iter, restart=True)
    s2.run_gvins(n_iter, restart=True)
    assert s1.gvins_optimization_end(slid) == s2.gvins_optimization_end(up)
    for a, b in zip(slid, up):
        for k in PARAMS:
            assert np.array_equal(a[k], b[k]), k


def chain(p, s, cam, seed, max_K):
    """gvins_optimization -> update_and_cull -> culled marginalization on handle s; the culled landmarks and outlier observations leave"""
    ci = cull_inputs(p, p["ext"].copy(), seed, bad_kp=20)
    s.gvins_optimization_batch([p], 20)
    g = s.update_and_cull([p], cam, STD, [ci])[0]
    mg = s.marginalize([p], 1, resident=True, culled=[g])[0]
    mask = po.culled_factor_mask(p, ci, g, np.ones(p["K"], np.uint8))
    return mg, np.nonzero(g["lm_outlier"])[0].tolist(), np.nonzero(mask == 0)[0].tolist()


def test_cfg3_chain(olib, cam):
    p = make(olib, outliers=25, seed=701, K=10, L=300)
    s1, s2 = handle(), handle()
    try:
        mg, bad_lm, bad_f = chain(p, s1, cam, 702, 10)
        assert bad_lm or bad_f
        up, slid, carry = build_next(p, 703, prior=mg, drop_lm=bad_lm, drop_f=bad_f)
        assert (carry["f_src"] >= 0).sum() > 100 and (carry["f_src"] < 0).sum() > 0 and (carry["lm_src"] < 0).sum() >= 4
        s1.slide([slid], [carry], True)
        compare_handles(s1, s2, [slid], [up])
    finally:
        s1.close(), s2.close()


def test_cfg4_split_pipeline_chain(olib, cam):
    p = make_large(olib, K=20, L=2000, seed=2042, n_ref=20, prior=True)
    kw = dict(K=20, L=2000, F=12000, R=292)
    s1, s2 = handle(**kw), handle(**kw)
    try:
        mg, bad_lm, bad_f = chain(p, s1, cam, 711, 20)
        assert mg["r"] == 277
        up, slid, carry = build_next(p, 712, prior=mg, drop_lm=bad_lm, drop_f=bad_f)
        s1.slide([slid], [carry], True)
        compare_handles(s1, s2, [slid], [up], n_iter=12)
    finally:
        s1.close(), s2.close()


def test_after_reintegration_with_every_gate_open(olib):
    from tests.test_reintegration_gpu import NOISE5, window
    p, rows = window(olib, 721, K=10, L=120, lin=lambda k: (np.full(3, 9 * NOISE5[2]), np.zeros(3)))
    s1, s2 = handle(), handle()
    try:
        s1.gvins_optimization_batch([p], 20)
        before = p["imu_blob"].copy()
        out = s1.reintegrate([p], NOISE5, np.zeros(3), [rows])[0]
        assert (out["status"] == 1).all() and not np.array_equal(before, p["imu_blob"])
        mg = s1.marginalize([p], 1, resident=True)[0]
        up, slid, carry = build_next(p, 722, prior=mg)
        assert (carry["imu_src"] >= 0).sum() == 8
        s1.slide([slid], [carry], True)
        compare_handles(s1, s2, [slid], [up])
    finally:
        s1.close(), s2.close()


def test_middle_node_removed_with_its_merged_blob_as_new(olib):
    p = make(olib, seed=731, K=8, L=120)
    s1, s2 = handle(K=10), handle(K=10)
    try:
        s1.gvins_optimization_batch([p], 20)
        up, slid, carry = build_next(p, 732, drop=(5,), n_new=1)
        assert list(carry["imu_src"]) == [0, 1, 2, 3, -1, 6, -1]
        s1.slide([slid], [carry], False)
        compare_handles(s1, s2, [slid], [up])
    finally:
        s1.close(), s2.close()


def test_prior_from_the_problem(olib):
    """a window not yet full that keeps its previous prior (uploaded J0 / e0, H0 formed on the device) and a window without a prior"""
    a = make_large(olib, K=8, L=150, seed=741, prior=True)
    b = make(olib, seed=742, K=6, L=80)
    s1, s2 = handle(n=2), handle(n=2)
    try:
        s1.gvins_optimization_batch([a, b], 20)
        ua, sa, ca = build_next(a, 743, drop=(), n_new=1, keep_prior=True)
        ub, sb, cb = build_next(b, 744, drop=(), n_new=1)
        assert ua["marg_r"] > 0 and ub["marg_r"] == 0
        s1.slide([sa, sb], [ca, cb], False)
        compare_handles(s1, s2, [sa, sb], [ua, ub])
    finally:
        s1.close(), s2.close()


def test_two_marginalizations_in_a_row(olib):
    """marginalize -> slide (no new node) -> marginalize -> slide, as the while (isMaximumKeframes()) loop of the reference"""
    p = make(olib, seed=751, K=10, L=300)
    s1, s2 = handle(), handle()
    try:
        s1.gvins_optimization_batch([p], 20)
        m1 = s1.marginalize([p], 1, resident=True)[0]
        u1, sl1, c1 = build_next(p, 752, prior=m1, n_new=0, n_new_lm=0)
        s1.slide([sl1], [c1], True)
        m2 = s1.marginalize([u1], 1, resident=True)[0]
        s2.upload([u1])
        m2u = s2.marginalize([u1], 1, resident=True)[0]
        for k in ("J0", "e0", "Hp", "bp"):
            assert np.array_equal(m2[k], m2u[k]), k
        u2, sl2, c2 = build_next(u1, 753, prior=m2)
        s1.slide([sl2], [c2], True)
        compare_handles(s1, s2, [sl2], [u2])
    finally:
        s1.close(), s2.close()


def test_batch_of_mixed_sizes_equals_per_window_slides(olib):
    specs = [dict(K=10, L=300, seed=761), dict(K=6, L=80, seed=762), dict(K=8, L=150, seed=763)]
    probs = [make(olib, **sp) for sp in specs]
    s = handle(n=3)
    try:
        s.gvins_optimization_batch(probs, 20)
        marg = s.marginalize(probs, 1, resident=True)
        nxt = [build_next(p, 770 + w, prior=marg[w] if w != 1 else None) for w, p in enumerate(probs)]
        s.slide([x[1] for x in nxt], [x[2] for x in nxt], [True, False, True])
        s.run_gvins(20)
        batch = s.gvins_optimization_end([x[1] for x in nxt])
    finally:
        s.close()
    for w, sp in enumerate(specs):
        p = make(olib, **sp)
        one = handle(n=1)
        try:
            one.gvins_optimization_batch([p], 20)
            m = one.marginalize([p], 1, resident=True)[0]
            _, sl, c = build_next(p, 770 + w, prior=m if w != 1 else None)
            one.slide([sl], [c], w != 1)
            one.run_gvins(20)
            assert one.gvins_optimization_end([sl])[0] == batch[w]
        finally:
            one.close()
        for k in PARAMS:
            assert np.array_equal(sl[k], nxt[w][1][k]), k


def test_rejections_leave_the_handle_as_it_was(olib):
    from ic_gvins_b200 import IcgError
    p = make(olib, seed=781, K=10, L=300)
    p0 = copy.deepcopy(p)  # as uploaded: an upload of it restores the pristine copies the restarts start from
    s = handle()

    def state():
        s.run_gvins(20, restart=True)
        q = copy.deepcopy(p)
        return s.gvins_optimization_end([q]), [q[k].copy() for k in PARAMS]

    def same(a, b):
        assert a[0] == b[0] and all(np.array_equal(x, y) for x, y in zip(a[1], b[1]))

    try:
        s.gvins_optimization_batch([p], 20)
        base = state()
        up, slid, carry = build_next(p, 782)
        bad = dict(carry, node_src=carry["node_src"].copy())
        bad["node_src"][0] = 99
        with pytest.raises(IcgError, match="out of range"):
            s.slide([slid], [bad], False)
        same(base, state())
        m = s.marginalize([p], 1, resident=True)[0]
        up, slid, carry = build_next(p, 783, prior=m)
        s.upload([copy.deepcopy(p0)])
        with pytest.raises(IcgError, match="no resident marginalization"):
            s.slide([slid], [carry], True)
        same(base, state())
        fresh = handle()
        try:
            fresh.gvins_optimization_batch([copy.deepcopy(p)], 20)
            with pytest.raises(IcgError, match="no resident marginalization"):
                fresh.slide([slid], [carry], True)
        finally:
            fresh.close()
        s.marginalize([p], 1, resident=True)
        wrong = copy.deepcopy(slid)
        wrong["marg_r"] = slid["marg_r"] - 1
        with pytest.raises(IcgError, match="marg_r="):
            s.slide([wrong], [carry], True)
        same(base, state())
        s.marginalize([p], 1, resident=True)
        big_up, big, big_c = build_next(p, 784, drop=(), n_new=1)
        with pytest.raises(IcgError, match="capacity"):
            s.slide([big], [big_c], False)
        same(base, state())
        up, slid, carry = build_next(p, 785)
        new_blob = np.nonzero(carry["imu_src"] < 0)[0][0]
        slid["imu_blob"].reshape(-1, IMU)[new_blob, 252:477] = -np.eye(15).reshape(-1)
        with pytest.raises(IcgError, match="positive-definite"):
            s.slide([slid], [carry], False)
        same(base, state())
    finally:
        s.close()
