"""GPU: icg_ba_slide_ins_resident and icg_ba_reintegrate_stored_resident.  One handle takes every integrated factor's rows from the INS
windows and its sample store; a twin handle goes through icg_ba_slide_integrate_resident / icg_ba_reintegrate_resident with the same rows
cut on the host by the std::deque restatement (tests/ins_series_oracle.cpp).  Blobs, end states and node rows, the two-pass solve, a
resident marginalization and a restarted solve must be the same bits, and the stored rows must be the twin's host rows."""
import copy

import numpy as np
import pytest

from datagen import synth_ba
from datagen.slide_window import build_next
from tests import ins_series_oracle as so
from tests import oracle_api as oa
from tests.test_oracle_gins_init import moving
from tests.test_post_solve_gpu import make
from tests.test_slide_gpu import PARAMS, handle
from tests.test_slide_integrate_gpu import CHAIN, ROW, compare, integ_for, solved_pair

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not so.HAVE_CXX, reason="no host C++ compiler for the INS restatement")]
NOISE5 = synth_ba.NOISE5
IMU = 480


@pytest.fixture(scope="module")
def cam():
    from ic_gvins_b200.camera import Camera
    from tests.test_post_solve_gpu import CAMD
    return Camera([CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"]], [0.0, 0.0, 0.0, 0.0])


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


def ins_pair(n, earth=True):
    """device and restatement INS windows of n streams, 10.0 .. 14.9 s at 200 Hz, mechanized by a redo near the front"""
    from ic_gvins_b200.ins import InsWindow
    d, o = InsWindow(n), so.OracleSeries(n)
    cfg = [{"with_earth": earth, "gravity": synth_ba.GRAVITY}] * n
    rows = [moving(10.0, 14.9, seed=50 + s, earth=earth) for s in range(n)]
    d.push(rows, cfg)
    assert o.push(rows, cfg) == 0
    st = np.zeros((n, 17))
    st[:, 7], st[:, 0] = 1, rows[0][2, 0] + 0.001
    np.testing.assert_array_equal(d.redo(st, cfg), o.redo(st, cfg))
    return d, o


def node_times(K):
    return 10.0507 + 0.5 * np.arange(K)  # inside the window the redo left, off the samples: both ends interpolated


def slide_twin(s1, s2, d, o, up, nxt, carry, g, t_new, merge=None, prior=False):
    """s1: slide_ins; s2: slide_integrate with the restatement's rows (g["imu_rows"]); then the solves, bitwise.  Returns the outputs and
    the window as the solve left it on the host (up, build_next's twin with every value row, with the solved parameters)"""
    a, b = copy.deepcopy(nxt), copy.deepcopy(nxt)
    g_dev = dict(g, imu_rows=None)
    out1 = s1.slide_ins([a], [carry], [g_dev], d, [0], [t_new], [merge], NOISE5, prior_from_marg=prior)[0]
    out2 = s2.slide_integrate([b], [carry], [g], NOISE5, prior_from_marg=prior)[0]
    for k in ("status", "blobs", "end_states"):
        np.testing.assert_array_equal(out1[k], out2[k], err_msg=k)
    assert (out1["status"][g["imu_from"] != -1] == 1).all()
    s1.download(), s2.download()
    compare(s1, s2, a, b)
    return out1, dict(up, **{k: a[k] for k in PARAMS})


def test_new_node_merged_node_and_chain(olib):
    """addNewTimeNode (NODE), then removeUnusedTimeNode (ROW merge of two stored factors) with a new node, then insertNewGnssTimeNode's
    re-created tail (NODE, CHAIN, CHAIN); carried factors keep their rows, and the store after each slide holds the twin's host rows"""
    p = make(olib, seed=951, K=8, L=120)
    s1, s2 = solved_pair(p, K=10)
    d, o = ins_pair(1)
    try:
        t = node_times(8)
        s1.imu_samples_from_ins(d, [0], [t])
        stored = [o.series(0, t[k], t[k + 1]) for k in range(7)]
        for a, b in zip(s1.imu_samples(0), stored):
            np.testing.assert_array_equal(a, b)
        # a new keyframe node from the last old node
        up, nxt, carry = build_next(p, 952, drop=(0,), n_new=1)
        t = np.r_[t[1:], t[-1] + 0.5]
        m = nxt["n_imu"]
        rows = {m - 1: o.series(0, t[m - 1], t[m])}
        out, p = slide_twin(s1, s2, d, o, up, nxt, carry, integ_for(nxt, carry, {m - 1: 7}, rows), t)
        stored = [o.series(0, t[j], t[j + 1]) for j in range(m)]  # carried: the old factor's rows; new: the cut
        assert list(out["n_rows"]) == [len(x) for x in stored]
        for a, b in zip(s1.imu_samples(0), stored):
            np.testing.assert_array_equal(a, b)
        # node 3 leaves: factors 2 and 3 merge (ROW) from their stored rows; one new node
        up, nxt, carry = build_next(p, 953, drop=(3,), n_new=1)
        assert list(carry["imu_src"][:4]) == [0, 1, -1, 4]
        merged = np.concatenate([stored[2], stored[3][1:]])
        t2 = np.r_[np.delete(t, 3), t[-1] + 0.5]
        m = nxt["n_imu"]
        state = np.zeros((m, 16))
        state[2] = np.concatenate([p["pose"].reshape(-1, 7)[2], p["mix"].reshape(-1, 9)[2]])
        rows = {2: merged, m - 1: o.series(0, t2[m - 1], t2[m])}
        merge = np.full(m, -1, np.int32)
        merge[2] = 2
        g = integ_for(nxt, carry, {2: ROW, m - 1: p["K"] - 1}, rows, state=state)
        _, p = slide_twin(s1, s2, d, o, up, nxt, carry, g, t2, merge)
        got = s1.imu_samples(0)
        np.testing.assert_array_equal(got[2], merged)
        np.testing.assert_array_equal(got[m - 1], rows[m - 1])
        for j in range(m):
            if carry["imu_src"][j] >= 0:
                np.testing.assert_array_equal(got[j], stored[carry["imu_src"][j]])
        # a GNSS node inserted after the last node and two nodes re-created from it
        up, nxt, carry = build_next(p, 954, drop=(0,), n_new=3)
        t3 = np.r_[t2[1:], t2[-1] + 0.1, t2[-1] + 0.2, t2[-1] + 0.3]
        m = nxt["n_imu"]
        rows = {k: o.series(0, t3[k], t3[k + 1]) for k in range(m - 3, m)}
        g = integ_for(nxt, carry, {m - 3: p["K"] - 1, m - 2: CHAIN, m - 1: CHAIN}, rows)
        slide_twin(s1, s2, d, o, up, nxt, carry, g, t3)
        got = s1.imu_samples(0)
        for k in range(m - 3, m):
            np.testing.assert_array_equal(got[k], rows[k])
    finally:
        s1.close(), s2.close(), d.close()


def test_reintegrate_stored(olib):
    """doReintegration from the store: the same statuses, blobs and end states as icg_ba_reintegrate_resident with the host rows, then the
    same solves; the stored rows do not change"""
    from tests.test_reintegration_gpu import window
    p, _ = window(olib, 961, K=10, L=120, lin=lambda k: (np.full(3, 9 * NOISE5[2]), np.zeros(3)))
    q = copy.deepcopy(p)
    s1, s2 = handle(), handle()
    d, o = ins_pair(1, earth=False)
    try:
        for s, x in ((s1, p), (s2, q)):
            s.gvins_optimization_batch([x], 20)
        t = node_times(p["K"])
        rows = [o.series(0, t[k], t[k + 1]) for k in range(p["n_imu"])]
        s1.imu_samples_from_ins(d, [0], [t])
        r1 = s1.reintegrate_stored([p], NOISE5)[0]
        r2 = s2.reintegrate([q], NOISE5, np.zeros(3), [rows])[0]
        assert (r1["status"] == 1).any()
        for k in ("status", "blobs", "end_states"):
            np.testing.assert_array_equal(r1[k], r2[k], err_msg=k)
        assert r1["count"] == r2["count"]
        for a, b in zip(s1.imu_samples(0), rows):
            np.testing.assert_array_equal(a, b)
        compare(s1, s2, p, q)
    finally:
        s1.close(), s2.close(), d.close()


def test_rejections_leave_the_store(olib):
    from ic_gvins_b200 import IcgError
    p = make(olib, seed=971, K=8, L=120)
    s1, s2 = solved_pair(p, K=10)
    d, o = ins_pair(1)
    try:
        t = node_times(8)
        s1.imu_samples_from_ins(d, [0], [t])
        before = s1.imu_samples(0)
        win_before = d.window(0)
        up, nxt, carry = build_next(p, 972, drop=(0,), n_new=1)
        m = nxt["n_imu"]
        t_new = np.r_[t[1:], t[-1] + 0.5]
        g = integ_for(nxt, carry, {m - 1: 7}, {m - 1: o.series(0, t_new[m - 1], t_new[m])})
        g_dev = dict(g, imu_rows=None)
        far = t_new.copy()
        far[-1] = 20.0  # after the INS window's back
        with pytest.raises(IcgError, match=f"window 0 IMU factor {m - 1}.*cannot serve") as e:
            s1.slide_ins([copy.deepcopy(nxt)], [carry], [g_dev], d, [0], [far], [None], NOISE5, prior_from_marg=False)
        assert e.value.results[0]["status"][m - 1] == -2 and not e.value.results[0]["status"][:m - 1].any()
        bad_time = t_new.copy()
        bad_time[2] = bad_time[1]
        with pytest.raises(IcgError, match="not less than"):
            s1.slide_ins([copy.deepcopy(nxt)], [carry], [g_dev], d, [0], [bad_time], [None], NOISE5, prior_from_marg=False)
        with pytest.raises(IcgError, match="out of range or not mechanized"):
            s1.slide_ins([copy.deepcopy(nxt)], [carry], [g_dev], d, [3], [t_new], [None], NOISE5, prior_from_marg=False)
        g_row = dict(g_dev, imu_from=g_dev["imu_from"].copy(), state16=np.zeros((m, 16)))
        g_row["imu_from"][m - 1] = ROW
        for bad in (-1, 7):
            merge = np.full(m, bad, np.int32)
            with pytest.raises(IcgError, match="merge_src"):
                s1.slide_ins([copy.deepcopy(nxt)], [carry], [g_row], d, [0], [t_new], [merge], NOISE5, prior_from_marg=False)
        for a, b in zip(s1.imu_samples(0), before):
            np.testing.assert_array_equal(a, b)
        w = d.window(0)
        np.testing.assert_array_equal(w[0], win_before[0]), np.testing.assert_array_equal(w[1], win_before[1])
        # the handle as it was: the good slide now matches the twin bit for bit
        _, p2 = slide_twin(s1, s2, d, o, up, nxt, carry, g, t_new)
        # a plain upload replaces the factors: the store is gone
        s1.upload([p2])
        with pytest.raises(IcgError, match="no IMU samples"):
            s1.reintegrate_stored([p2], NOISE5)
        with pytest.raises(IcgError, match="no IMU samples"):
            s1.imu_samples(0)
    finally:
        s1.close(), s2.close(), d.close()


def test_vision_form_and_mixed_batch_after_a_push(olib, cam):
    """Two windows in one call (Earth and Normal INS streams): first the vision form of slide_ins against slide_integrate of the
    host-built twin; then window 0 takes a new node and window 1 a ROW merge and a new node, cut from rows pushed to the INS windows right
    before the call (the solver's stream waits for the INS stream); the store holds each window's rows at its own offsets."""
    from tests.test_slide_vision_gpu import Keyframe, check_built, compare_all, host_twin, solve_cull_marg
    from tests.test_slide_vision_gpu import so as vso
    from ic_gvins_b200.ins import InsWindow
    probs = [make(olib, outliers=10, seed=981 + w, K=8, L=120) for w in range(2)]
    p1, p2 = probs, copy.deepcopy(probs)
    s1, s2 = handle(n=2), handle(n=2)
    d, o = InsWindow(2), so.OracleSeries(2)
    cfg = [{"with_earth": w == 0, "gravity": synth_ba.GRAVITY} for w in range(2)]
    rows = [moving(10.0, 14.9, seed=60 + w, earth=w == 0) for w in range(2)]
    cut_at = np.searchsorted(rows[0][:, 0], 14.2)  # the first slide reads up to 14.05 s, the second up to 14.55 s
    try:
        d.push([r[:cut_at] for r in rows], cfg)
        assert o.push([r[:cut_at] for r in rows], cfg) == 0
        st = np.zeros((2, 17))
        st[:, 7], st[:, 0] = 1, rows[0][2, 0] + 0.001
        np.testing.assert_array_equal(d.redo(st, cfg), o.redo(st, cfg))
        for s, x in ((s1, p1), (s2, p2)):
            s.gvins_optimization_batch(x, 20)
        t = node_times(8)
        s1.imu_samples_from_ins(d, [0, 1], [t, t])
        stored = [[o.series(w, t[k], t[k + 1]) for k in range(7)] for w in range(2)]
        refs = [vso.reference_rows(p) for p in p1]
        gs, mgs = solve_cull_marg(p1, s1, cam, 990)
        solve_cull_marg(p2, s2, cam, 990)
        kfs = [Keyframe(p, g, mg, rf, 991 + w) for w, (p, g, mg, rf) in enumerate(zip(p1, gs, mgs, refs))]
        os_ = [kf.oracle(p, rf) for kf, p, rf in zip(kfs, p1, refs)]
        a = [copy.deepcopy(kf.nxt) for kf in kfs]
        ca = [copy.deepcopy(kf.carry) for kf in kfs]
        twins = [host_twin(kf.nxt, kf.carry, x) for kf, x in zip(kfs, os_)]
        b, cb = [x[0] for x in twins], [x[1] for x in twins]
        t1 = np.r_[t[1:], t[-1] + 0.5]
        m = kfs[0].nxt["n_imu"]
        ig = [integ_for(kf.nxt, kf.carry, {m - 1: p["K"] - 1}, {m - 1: o.series(w, t1[m - 1], t1[m])}, normal=w == 1)
              for w, (kf, p) in enumerate(zip(kfs, p1))]
        r = s1.slide_ins(a, ca, [dict(g, imu_rows=None) for g in ig], d, [0, 1], [t1, t1], None, NOISE5, vision=[kf.device() for kf in kfs])
        out2 = s2.slide_integrate(b, cb, ig, NOISE5)
        for w, (x, y, ref) in enumerate(zip(r, out2, os_)):
            check_built(x, ref)
            for k in ("status", "blobs", "end_states"):
                np.testing.assert_array_equal(x[k], y[k], err_msg=k)
            assert x["status"][m - 1] == 1 and list(x["n_rows"][:m - 1]) == [len(z) for z in stored[w][1:]]
        compare_all(s1, s2, a, b)
        for w in range(2):
            got = s1.imu_samples(w)
            for k in range(m - 1):
                np.testing.assert_array_equal(got[k], stored[w][k + 1])
            np.testing.assert_array_equal(got[m - 1], ig[w]["imu_rows"][m - 1])
        stored = [s1.imu_samples(w) for w in range(2)]
        # the rest of the rows, pushed just before the next call (asynchronous on the INS stream)
        d.push([r_[cut_at:] for r_ in rows], cfg)
        assert o.push([r_[cut_at:] for r_ in rows], cfg) == 0
        full = [dict(y, **{k: x[k] for k in PARAMS}) for x, y in zip(a, b)]
        (up0, n0, c0), (up1, n1, c1) = build_next(full[0], 995, drop=(0,), n_new=1), build_next(full[1], 996, drop=(3,), n_new=1)
        t_a, t_b = np.r_[t1[1:], t1[-1] + 0.5], np.r_[np.delete(t1, 3), t1[-1] + 0.5]
        assert t_a[-1] > rows[0][cut_at - 1, 0]  # the new intervals lie in the rows just pushed
        mm = n0["n_imu"]
        g0 = integ_for(n0, c0, {mm - 1: 7}, {mm - 1: o.series(0, t_a[mm - 1], t_a[mm])})
        state = np.zeros((mm, 16))
        state[2] = np.concatenate([full[1]["pose"].reshape(-1, 7)[2], full[1]["mix"].reshape(-1, 9)[2]])
        merged = np.concatenate([stored[1][2], stored[1][3][1:]])
        g1 = integ_for(n1, c1, {2: ROW, mm - 1: 7}, {2: merged, mm - 1: o.series(1, t_b[mm - 1], t_b[mm])}, normal=True, state=state)
        merge = [None, np.array([-1, -1, 2] + [-1] * (mm - 3), np.int32)]
        a, b = [copy.deepcopy(n0), copy.deepcopy(n1)], [copy.deepcopy(n0), copy.deepcopy(n1)]
        o1 = s1.slide_ins(a, [c0, c1], [dict(g0, imu_rows=None), dict(g1, imu_rows=None)], d, [0, 1], [t_a, t_b], merge, NOISE5,
                          prior_from_marg=False)
        o2 = s2.slide_integrate(b, [c0, c1], [g0, g1], NOISE5, prior_from_marg=False)
        for x, y in zip(o1, o2):
            for k in ("status", "blobs", "end_states"):
                np.testing.assert_array_equal(x[k], y[k], err_msg=k)
        s1.download(), s2.download()
        compare_all(s1, s2, a, b)
        got = [s1.imu_samples(w) for w in range(2)]
        np.testing.assert_array_equal(got[0][mm - 1], g0["imu_rows"][mm - 1])
        np.testing.assert_array_equal(got[1][2], merged)
        np.testing.assert_array_equal(got[1][mm - 1], g1["imu_rows"][mm - 1])
        for w, c in ((0, c0), (1, c1)):
            for j in range(mm):
                if c["imu_src"][j] >= 0:
                    np.testing.assert_array_equal(got[w][j], stored[w][c["imu_src"][j]])
    finally:
        s1.close(), s2.close(), d.close()


def test_cfg4_split_pipeline(olib, cam):
    from tests.test_marg_large_gpu import make as make_large
    from tests.test_slide_gpu import chain
    p1 = make_large(olib, K=20, L=2000, seed=2042, n_ref=20, prior=True)
    p2 = copy.deepcopy(p1)
    kw = dict(K=20, L=2000, F=12000, R=292)
    s1, s2 = handle(**kw), handle(**kw)
    d, o = ins_pair(1)
    try:
        mg, bad_lm, bad_f = chain(p1, s1, cam, 941, 20)
        chain(p2, s2, cam, 941, 20)
        t = 10.0507 + 0.2 * np.arange(20)
        s1.imu_samples_from_ins(d, [0], [t])
        up, nxt, carry = build_next(p1, 942, prior=mg, drop_lm=bad_lm, drop_f=bad_f)
        t = np.r_[t[1:], t[-1] + 0.2]
        m = nxt["n_imu"]
        g = integ_for(nxt, carry, {m - 1: 19}, {m - 1: o.series(0, t[m - 1], t[m])})
        a, b = copy.deepcopy(nxt), copy.deepcopy(nxt)
        x = s1.slide_ins([a], [carry], [dict(g, imu_rows=None)], d, [0], [t], None, NOISE5)[0]
        y = s2.slide_integrate([b], [carry], [g], NOISE5)[0]
        for k in ("status", "blobs", "end_states"):
            np.testing.assert_array_equal(x[k], y[k], err_msg=k)
        s1.download(), s2.download()
        compare(s1, s2, a, b, n_iter=12)
        np.testing.assert_array_equal(s1.imu_samples(0)[m - 1], g["imu_rows"][m - 1])
    finally:
        s1.close(), s2.close(), d.close()


def test_abi_rejections_and_sharded_handles(olib):
    """integ.imu / imu_off and io.imu must be NULL; a landmark-sharded handle gets ICG_EUNSUPPORTED from all four calls; the store and every
    stream's INS window stay as they were"""
    import ctypes as C
    from ic_gvins_b200 import IcgError
    from ic_gvins_b200._lib import SlideIns, SlideWindow, lib
    from ic_gvins_b200.ba import BaProblem, ReintWindow, to_struct
    p = make(olib, seed=1001, K=8, L=120)
    s1, s2 = solved_pair(p, K=10)
    d, o = ins_pair(2)
    try:
        t = node_times(8)
        s1.imu_samples_from_ins(d, [1], [t])
        before, wins = s1.imu_samples(0), [d.window(k) for k in range(2)]
        up, nxt, carry = build_next(p, 1002, drop=(0,), n_new=1)
        t_new = np.r_[t[1:], t[-1] + 0.5]
        arr = (BaProblem * 1)(to_struct(nxt))
        cw = (SlideWindow * 1)()
        io = (SlideIns * 1)()
        junk = np.zeros(16)
        io[0].integ.imu = junk.ctypes.data_as(C.POINTER(C.c_double))
        io[0].stream, io[0].node_time = 1, t_new.ctypes.data_as(C.POINTER(C.c_double))
        nz, stn = np.ascontiguousarray(NOISE5), np.zeros(3)
        assert lib().icg_ba_slide_ins_resident(s1._h, d._h, 1, arr, cw, io, nz.ctypes.data, stn.ctypes.data, None) == -1
        assert b"must be NULL" in lib().icg_last_error()
        io[0].integ.imu, io[0].integ.imu_off = None, junk.ctypes.data_as(C.POINTER(C.c_int32))
        assert lib().icg_ba_slide_ins_resident(s1._h, d._h, 1, arr, cw, io, nz.ctypes.data, stn.ctypes.data, None) == -1
        parr = (BaProblem * 1)(to_struct(p))
        rw = (ReintWindow * 1)()
        rw[0].reintegrate, rw[0].imu = 1, junk.ctypes.data_as(C.POINTER(C.c_double))
        assert lib().icg_ba_reintegrate_stored_resident(s1._h, 1, parr, nz.ctypes.data, stn.ctypes.data, rw) == -1
        assert b"must be NULL" in lib().icg_last_error()
        s1.shard_export(0, 2)
        g = integ_for(nxt, carry, {nxt["n_imu"] - 1: 7}, {nxt["n_imu"] - 1: None})
        for call in (lambda: s1.imu_samples_from_ins(d, [1], [t]), lambda: s1.imu_samples(0), lambda: s1.reintegrate_stored([p], NOISE5),
                     lambda: s1.slide_ins([copy.deepcopy(nxt)], [carry], [g], d, [1], [t_new], None, NOISE5)):
            with pytest.raises(IcgError, match="landmark-sharded") as e:
                call()
            assert getattr(e.value, "code", -4) == -4 and "code -4" in str(e.value)
        s1.shard_leave()
        for a, b in zip(s1.imu_samples(0), before):
            np.testing.assert_array_equal(a, b)
        for k in range(2):
            w = d.window(k)
            np.testing.assert_array_equal(w[0], wins[k][0]), np.testing.assert_array_equal(w[1], wins[k][1])
    finally:
        s1.close(), s2.close(), d.close()
