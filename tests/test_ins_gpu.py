"""GPU: the device INS windows (ic_gvins_b200.ins, csrc/ins.cu) against the CPU restatement (tests/ins_oracle.cpp).

Rows, times, biases and counts must match exactly.  p / q / v are compared per group against the group's scale (|p|, 1, |v|): within 1e-12
after one sample, and within TOL over windows of up to 1000 samples.  The oracle stays within 2.5e-15 of a 40-digit restatement over such
windows (tests/test_oracle_ins.py); the device rounds at the same steps but multiplies 0.5 (I + R(qnn)) R(q) dvfb right to left (the order
the preintegration core shares) and its sin / cos / sqrt / atan2 may differ from glibc in the last ulp, so the two differ by at most the sum of
their distances to the exact chain.  TOL is 10x the 5e-15 that sum allows."""
import numpy as np
import pytest

from tests import ins_oracle as io
from tests.test_oracle_ins import EARTH, NORMAL, POSE_B_C, rows8, state_at

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not io.HAVE_CXX, reason="no host C++ compiler for the INS restatement")]
TOL = 5e-14
TOL_ONE = 1e-12
LK_EPS_PX = 0.01  # cv::TermCriteria EPS of the tracking calls (IG/tracking/tracking.cc:385-398)


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _dev(n, capacity=1000):
    from ic_gvins_b200.ins import InsWindow
    return InsWindow(n, capacity)


def _state_err(a, b):
    """worst error of p, q, v of states a vs b (k x 17), each against its group's scale"""
    if a.shape[0] == 0:
        return 0.0
    sp = np.maximum(np.linalg.norm(b[:, 1:4], axis=1), 1.0)
    sv = np.maximum(np.linalg.norm(b[:, 8:11], axis=1), 1.0)
    ep = (np.abs(a[:, 1:4] - b[:, 1:4]).max(axis=1) / sp).max()
    eq = np.abs(a[:, 4:8] - b[:, 4:8]).max()
    ev = (np.abs(a[:, 8:11] - b[:, 8:11]).max(axis=1) / sv).max()
    return max(ep, eq, ev)


def _same_window(d, o, s, tol=TOL):
    imu_d, x_d = d.window(s)
    imu_o, x_o = o.window(s)
    assert imu_d.shape == imu_o.shape, (s, imu_d.shape, imu_o.shape)
    np.testing.assert_array_equal(imu_d, imu_o)
    np.testing.assert_array_equal(x_d[:, 0], x_o[:, 0])
    np.testing.assert_array_equal(x_d[:, 11:17], x_o[:, 11:17])
    e = _state_err(x_d, x_o)
    assert e <= tol, (s, e)
    return e


def _cfgs(n):
    return [EARTH if s % 2 == 0 else NORMAL for s in range(n)]


def _states(streams_rows, idx, offset=0.0021):
    """one optimized state per stream, at row idx (+ offset) of the stream's rows"""
    out = []
    for s, r in enumerate(streams_rows):
        st = state_at(r[0, 0] + 0.1 * s)
        st[0] = r[min(idx, r.shape[0] - 2), 0] + offset
        out.append(st)
    return np.array(out)


# ---------------------------------------------------------------------------------------------- push
def test_push_b296_both_forms():
    B = 296
    cfg = _cfgs(B)
    rows = [rows8(10.0 + 0.37 * s, 10.0 + 0.37 * s + 2.0, 200.0, earth=cfg[s]["with_earth"], seed=s) for s in range(B)]
    d, o = _dev(B, 2000), io.OracleIns(B, 2000)
    head = [r[:200] for r in rows]
    d.push(head, cfg)
    assert o.push(head, cfg) == 0
    st = _states(rows, 150)
    np.testing.assert_array_equal(d.redo(st, cfg), o.redo(st, cfg))
    worst = 0.0
    for c in range(10):  # 20 samples per frame at 200 Hz / 10 Hz
        part = [r[200 + 20 * c:220 + 20 * c] for r in rows]
        d.push(part, cfg)
        assert o.push(part, cfg) == 0
        if c == 0:  # after one sample
            for s in range(B):
                xd, xo = d.window(s)[1], o.window(s)[1]
                k = xo.shape[0] - 20
                assert _state_err(xd[k:k + 1], xo[k:k + 1]) <= TOL_ONE
    for s in range(B):
        worst = max(worst, _same_window(d, o, s))
    d.close()


def test_push_mixed_batch():
    """empty, one row, initialization windows crossing 1000 rows, a mechanized window pushed to exactly its capacity"""
    n, cap = 6, 1200
    cfg = _cfgs(n)
    long = [rows8(5.0, 5.0 + 1400 / 200.0, 200.0, earth=cfg[s]["with_earth"], seed=40 + s) for s in range(n)]
    d, o = _dev(n, cap), io.OracleIns(n, cap)
    # stream 5 is mechanized first, with a window of 300
    first = [long[s][:0] for s in range(5)] + [long[5][:300]]
    d.push(first, cfg), o.push(first, cfg)
    st = np.zeros((n, 17))
    st[5] = state_at(6.0)
    st[5, 0] = long[5][3, 0] + 0.0021
    sel = [0] * 5 + [1]
    np.testing.assert_array_equal(d.redo(st, cfg, redo=sel, reserved=2), o.redo(st, cfg, redo=sel, reserved=2))
    cnt5 = o.window(5)[0].shape[0]
    batch = [long[0][:0], long[1][:1], long[2][:999], long[3][:1001], long[4][:1400], long[5][300:300 + cap - cnt5]]
    d.push(batch, cfg)
    assert o.push(batch, cfg) == 0
    for s in range(n):
        _same_window(d, o, s)
    assert d.window(5)[0].shape[0] == cap
    assert d.window(4)[0].shape[0] == 1000 and d.window(3)[0].shape[0] == 1000
    nxt = [long[0][:3], long[1][1:2], long[2][999:1010], long[3][1001:1100], long[4][:0], long[5][:0]]
    d.push(nxt, cfg), o.push(nxt, cfg)
    for s in range(n):
        _same_window(d, o, s)
    d.close()


# ---------------------------------------------------------------------------------------------- redo
@pytest.mark.parametrize("cfg", [NORMAL, EARTH], ids=["normal", "earth"])
def test_redo_cases(cfg):
    """one stream per isNeedInterpolation case (-1, 1, 2 with the split imu_pre carry, 0 with the exact-sample quirk), two prunings, and
    times outside the window (status -1, window unchanged)"""
    rows = rows8(30.0, 30.0 + 60 / 200.0, 200.0, earth=cfg["with_earth"], seed=5)
    k = 40
    times = [rows[k - 1, 0] + 0.3e-4, rows[k, 0] - 0.3e-4, rows[k - 1, 0] + 0.002, rows[k - 1, 0], rows[1, 0] + 0.002, rows[-2, 0] + 0.001,
             rows[0, 0] - 1.0, rows[-1, 0], rows[-1, 0] + 0.5]
    n = len(times)
    d, o = _dev(n), io.OracleIns(n)
    d.push([rows] * n, [cfg] * n), o.push([rows] * n, [cfg] * n)
    # mechanize every stream first, so that the quirk leaves a mechanized state (not a zero one) at its index
    st0 = np.array([state_at(30.0)] * n)
    st0[:, 0] = rows[0, 0] + 0.5e-4
    np.testing.assert_array_equal(d.redo(st0, [cfg] * n, reserved=100), [1] * n)
    o.redo(st0, [cfg] * n, reserved=100)
    st = np.array([state_at(31.0 + 0.01 * s) for s in range(n)])
    st[:, 0] = times
    sd, so = d.redo(st, [cfg] * n), o.redo(st, [cfg] * n)
    np.testing.assert_array_equal(sd, so)
    np.testing.assert_array_equal(sd, [1, 1, 1, 1, 1, 1, -1, -1, -1])
    for s in range(n):
        _same_window(d, o, s)
    N = rows.shape[0]
    assert d.window(0)[0].shape[0] == N - (k - 2)
    assert d.window(4)[0].shape[0] == N  # index 2 == reserved: nothing dropped
    # the split's imu_pre carry: the state after the split row differs from one integrated from the unsplit row
    xd = d.window(2)[1]
    j = 3  # entry index + 1 after dropping index - 2 entries
    a, b = io.interpolate(rows[k], times[2])
    assert not np.array_equal(io.mechanize(cfg, rows[k], rows[k + 1], xd[j - 1]), io.mechanize(cfg, b, rows[k + 1], xd[j - 1]))
    assert _state_err(xd[j:j + 1], io.mechanize(cfg, b, rows[k + 1], xd[j - 1])[None]) <= TOL_ONE
    d.close()


# ---------------------------------------------------------------------------------------------- camera pose
def test_camera_pose_cases():
    rows = rows8(40.0, 40.0 + 60 / 200.0, 200.0, seed=9)
    t = rows[:, 0]
    stamps = [t[0] - 0.01, t[10], t[10] + 0.0021, t[-1], t[-1] + 0.01, t[25] + 0.003]
    n = len(stamps) + 2
    cfg = [EARTH] * len(stamps) + [NORMAL, NORMAL]
    # stream n-2: identity attitude, no rotation, zero gyro bias -> dq exactly identity; stream n-1: the optimized q given with w < 0
    still = rows.copy()
    still[:, 2:5] = 0.0
    data = [rows] * len(stamps) + [still, rows]
    d, o = _dev(n), io.OracleIns(n)
    d.push(data, cfg), o.push(data, cfg)
    st = np.array([state_at(40.0)] * n)
    st[:, 0] = rows[0, 0] + 0.5e-4
    st[n - 2, 4:8] = [0.0, 0.0, 0.0, 1.0]
    st[n - 2, 11:14] = 0.0
    d.redo(st, cfg, reserved=100), o.redo(st, cfg, reserved=100)
    flip = st[n - 1].copy()
    flip[0] = t[30] - 0.3e-4  # case 1 at index 30: stored as given (normalised), w < 0, then mechanized on
    flip[4:8] = -flip[4:8]
    sel = [0] * (n - 1) + [1]
    d.redo(np.array([flip] * n), cfg, redo=sel, reserved=100), o.redo(np.array([flip] * n), cfg, redo=sel, reserved=100)
    assert o.window(n - 1)[1][30, 7] * o.window(n - 1)[1][29, 7] < 0  # dq = q30^-1 q29 has w < 0
    stamp = np.array(stamps + [t[20] + 0.002, t[29] + 0.002])
    hp, fd, dp = d.camera_pose(stamp, POSE_B_C)
    po, fo = o.camera_pose(stamp, POSE_B_C)
    np.testing.assert_array_equal(fd, fo)
    np.testing.assert_array_equal(fd, [0, 1, 1, 0, 0, 1, 1, 1])
    np.testing.assert_array_equal(hp, dp.cpu().numpy()[:n])
    err = np.abs(hp - po) / np.maximum(np.abs(po), 1.0)
    assert err.max() <= TOL, err.max(axis=0)
    # never mechanized: found -1, pose not written
    e = _dev(2)
    e.push([rows, rows[:0]], [EARTH, EARTH])
    import torch
    buf = torch.full((2, 12), 7.0, dtype=torch.float64, device="cuda")
    _, f2, buf = e.camera_pose([t[5], t[5]], POSE_B_C, dev_pose=buf)
    np.testing.assert_array_equal(f2, [-1, -1])
    assert bool((buf == 7.0).all())
    d.close(), e.close()


# ---------------------------------------------------------------------------------------------- rejection and the initialization path
def test_rejection_leaves_windows_unchanged():
    from ic_gvins_b200 import IcgError
    rows = rows8(0.0, 1300 / 200.0, 200.0, seed=2)
    d = _dev(2, 1000)
    d.push([rows[:300], rows[:10]], [EARTH, NORMAL])
    st = state_at(0.0)[None].repeat(2, 0)
    st[:, 0] = rows[5, 0] + 0.002
    d.redo(st, [EARTH, NORMAL], redo=[1, 0])
    room = 1000 - d.window(0)[0].shape[0]
    before = [d.window(s) for s in range(2)]
    for bad in ([rows[300:301], rows[9:11]], [rows[299:301], rows[10:11]], [rows[300:302][::-1], rows[10:11]],
                [rows[300:300 + room + 1], rows[10:11]]):
        with pytest.raises(IcgError, match="code -1"):
            d.push(bad, [EARTH, NORMAL])
        for s in range(2):
            for a, b in zip(d.window(s), before[s]):
                np.testing.assert_array_equal(a, b)
    d.push([rows[300:300 + room], rows[10:11]], [EARTH, NORMAL])  # exactly to capacity
    assert d.window(0)[0].shape[0] == 1000
    d.close()


def test_initialization_then_mechanization():
    rows = rows8(0.0, 1600 / 200.0, 200.0, seed=4)
    d, o = _dev(1, 2000), io.OracleIns(1, 2000)
    for a, b in ((0, 700), (700, 1400)):
        d.push([rows[a:b]], EARTH), o.push([rows[a:b]], EARTH)
    imu, x = d.window(0)
    np.testing.assert_array_equal(imu, rows[400:1400])
    assert not x.any()
    st = state_at(3.0)
    st[0] = rows[1380, 0] + 0.0013
    assert d.redo(st[None], EARTH)[0] == 1 and o.redo(st[None], EARTH)[0] == 1
    d.push([rows[1400:1600]], EARTH), o.push([rows[1400:1600]], EARTH)
    _same_window(d, o, 0)
    assert d.window(0)[0].shape[0] == 1600 - 1379  # per-sample mechanization from the redo on: no 1000-row trimming
    d.close()


# ---------------------------------------------------------------------------------------------- batches
def test_batch_equals_single_streams():
    n = 37
    cfg = _cfgs(n)
    rows = [rows8(1.0 + 0.1 * s, 1.0 + 0.1 * s + 1.0, 200.0, earth=cfg[s]["with_earth"], seed=100 + s) for s in range(n)]
    st = _states(rows, 60)
    stamp = np.array([r[150, 0] + 0.0017 for r in rows])
    bd = _dev(n)
    bd.push([r[:100] for r in rows], cfg)
    bd.redo(st, cfg)
    bd.push([r[100:180] for r in rows], cfg)
    hb, fb, _ = bd.camera_pose(stamp, POSE_B_C)
    for s in range(n):
        one = _dev(1)
        one.push([rows[s][:100]], cfg[s])
        one.redo(st[s:s + 1], cfg[s])
        one.push([rows[s][100:180]], cfg[s])
        h1, f1, _ = one.camera_pose(stamp[s:s + 1], POSE_B_C)
        for a, b in zip(one.window(0), bd.window(s)):
            np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(h1[0], hb[s])
        assert f1[0] == fb[s]
        one.close()
    bd.close()


# ---------------------------------------------------------------------------------------------- a ring that has wrapped
def test_redo_and_pose_on_wrapped_rings():
    """redo and camera pose on windows whose ring head has wrapped past the capacity (the steady state of a long run), in both forms"""
    cap, cfg = 1000, [EARTH, NORMAL]
    rows = [rows8(0.0, 1900 / 200.0, 200.0, earth=c["with_earth"], seed=70 + s) for s, c in enumerate(cfg)]
    d, o = _dev(2, cap), io.OracleIns(2, cap)
    d.push([r[:300] for r in rows], cfg), o.push([r[:300] for r in rows], cfg)
    end, straddled = 300, 0
    for cyc in range(16):
        st = np.array([state_at(r[end - 120, 0]) for r in rows])
        st[:, 0] = [r[end - 120 - 7 * cyc % 40, 0] + 0.0021 for r in rows]
        sd = d.redo(st, cfg)
        np.testing.assert_array_equal(sd, o.redo(st, cfg))
        assert (sd == 1).all()
        for s in range(2):
            _same_window(d, o, s)
            imu = d.window(s)[0]
            head = int(np.searchsorted(rows[s][:, 0], imu[0, 0])) % cap  # the ring's head: every entry before it was dropped
            straddled += head + imu.shape[0] > cap
        stamp = np.array([r[end - 30, 0] + 0.0017 for r in rows])
        hp, fd, dp = d.camera_pose(stamp, POSE_B_C)
        po, fo = o.camera_pose(stamp, POSE_B_C)
        np.testing.assert_array_equal(fd, [1, 1])
        np.testing.assert_array_equal(fd, fo)
        np.testing.assert_array_equal(hp, dp.cpu().numpy()[:2])
        assert (np.abs(hp - po) / np.maximum(np.abs(po), 1.0)).max() <= TOL
        d.push([r[end:end + 100] for r in rows], cfg), o.push([r[end:end + 100] for r in rows], cfg)
        end += 100
    assert straddled > 0, "no window ever straddled the end of its ring"
    d.close()


# ---------------------------------------------------------------------------------------------- the chain into the tracking step
def test_chain_solve_redo_pose_track(oracle):
    """icg_ba_gvins_optimization_begin / end -> icg_ins_redo from each window's last node (state17 = its pose and mix rows) -> icg_ins_push
    -> icg_ins_camera_pose -> icg_klt_track_frames_dev with those poses as R_pre / R_cur / t_cur.
    Pins both bindings: the pose at the redone entry is stateToCameraPose of the solved node, read from the solver's pose7 / mix9 layout, and
    the tracking call fed the device poses equals the one fed the restatement's poses and the one on the same scene in the camera frame."""
    import ctypes as C

    import torch

    from ic_gvins_b200._lib import BaProblem, lib
    from ic_gvins_b200.ba import WindowSolver, to_struct
    from ic_gvins_b200.klt import KltTracker
    from datagen import synth_ba
    from datagen import synth_klt as synth
    from tests import oracle_api as oa
    from tests.test_track_frame_gpu import MAXP, H, W, Rz, dev_lists, make_case, params_struct

    oa.declare_ba(oracle)
    B, K = 3, 6
    probs = [synth_ba.make_window(lambda *a: oa.preintegrate(oracle, *a), K=K, L=60, seed=500 + w)[0] for w in range(B)]
    solver = WindowSolver(max_windows=B, max_K=K, max_L=60, max_F=max(p["F"] for p in probs), max_gnss=8, max_marg_r=1)
    arr = (BaProblem * B)(*[to_struct(p) for p in probs])
    assert lib().icg_ba_gvins_optimization_begin(solver._h, B, arr, 20) == 0
    solver.gvins_optimization_end(probs)
    solver.close()
    t_node = (K - 1) * 0.5  # synth_ba's node times: k * dt_node
    state17 = np.array([np.concatenate([[t_node], p["pose"].reshape(K, 7)[K - 1], p["mix"].reshape(K, 9)[K - 1]]) for p in probs])
    # a row 0.5e-4 after the node: isNeedInterpolation case 1 stores the solved state there as given (q normalised)
    cfg = [EARTH, NORMAL, EARTH]
    rows = [rows8(t_node + 0.5e-4 - 1.0, t_node + 0.5e-4 + 0.3, 200.0, earth=c["with_earth"], seed=600 + w) for w, c in enumerate(cfg)]
    r = 200
    assert all(abs(x[r, 0] - t_node - 0.5e-4) < 1e-9 for x in rows)
    d, o = _dev(B), io.OracleIns(B)
    d.push([x[:241] for x in rows], cfg), o.push([x[:241] for x in rows], cfg)
    sd = d.redo(state17, cfg)
    np.testing.assert_array_equal(sd, [1] * B)
    np.testing.assert_array_equal(sd, o.redo(state17, cfg))
    d.push([x[241:261] for x in rows], cfg), o.push([x[241:261] for x in rows], cfg)
    for w in range(B):
        _same_window(d, o, w)
    # the node itself: pose at the stored entry's time == stateToCameraPose(solved node); bg / ba stored as solved; v enters p
    hp0, f0, _ = d.camera_pose([x[r, 0] for x in rows], POSE_B_C)
    np.testing.assert_array_equal(f0, [1] * B)
    Rbc, tbc = POSE_B_C[:9].reshape(3, 3), POSE_B_C[9:]
    for w in range(B):
        pose7, mix9 = state17[w, 1:8], state17[w, 8:17]
        Rq = synth_ba.q_mat(pose7[3:7] / np.linalg.norm(pose7[3:7]))
        np.testing.assert_allclose(hp0[w, :9], (Rq @ Rbc).reshape(9), rtol=0, atol=1e-12)
        np.testing.assert_allclose(hp0[w, 9:], pose7[:3] + Rq @ tbc, rtol=0, atol=1e-10)
        imu, x = d.window(w)
        e = int(np.searchsorted(imu[:, 0], rows[w][r, 0]))
        np.testing.assert_array_equal(x[e, 11:17], mix9[3:9])
        assert np.abs((x[e + 1, 1:4] - x[e, 1:4]) - 0.005 * mix9[:3]).max() < 1e-3
    # the frame: prior poses from the device and from the restatement
    stamp = np.array([x[255, 0] + 0.0021 for x in rows])
    hp, fd, dp = d.camera_pose(stamp, POSE_B_C)
    po, fo = o.camera_pose(stamp, POSE_B_C)
    np.testing.assert_array_equal(fd, fo)
    np.testing.assert_array_equal(hp, dp.cpu().numpy()[:B])
    d.close()

    stream = synth.KltStream(W, H, 400, 1234)
    trk = KltTracker(W, H, n_slots=4, max_points=MAXP)
    for s, f in enumerate((0, 1, 2)):
        trk.upload(s, stream.frame(f))
    trk.sync()

    def in_world(case, pose):
        """the case's scene moved into the world frame of a camera at `pose` (R camera-to-world row-major, t): the same pixels"""
        P, ml, rl = case
        Rw, tw = pose[:9].reshape(3, 3), pose[9:]
        P = dict(P, R_pre=Rw, R_cur=Rw, R_ref=Rw @ Rz(0.003), t_cur=tw)
        return P, dict(ml, pw=np.ascontiguousarray(ml["pw"] @ Rw.T + tw)), rl

    def track(cases):
        D = dev_lists(cases)
        n_out = torch.zeros(2 * B, dtype=torch.int32, device="cuda")
        par = torch.zeros(2 * B, dtype=torch.float64, device="cuda")
        par_n = torch.zeros(2 * B, dtype=torch.int32, device="cuda")
        trk.track_frames_dev([params_struct(c[0], w % 2, 1 + w % 2) for w, c in enumerate(cases)], D["map"][0], D["map"][2], D["ref"][0],
                             D["ref"][2], n_out.data_ptr(), par.data_ptr(), par_n.data_ptr())
        trk.sync()
        out = {k: {n: v.cpu().numpy() for n, v in D[k][1].items()} for k in ("map", "ref")}
        return n_out.cpu().numpy(), out, {k: D[k][0] for k in ("map", "ref")}

    base = [make_case(stream, 1 + w % 2, 80, 80, 300 + w) for w in range(B)]
    # the poses agree to rounding, so the predicted pixels differ by at most an ulp of float; from starts that close, two LK runs stop within
    # their termination step (criteria EPS 0.01 px, tracking.cc:385-398) of each other: positions are compared against that step
    assert (np.abs(hp - po) / np.maximum(np.abs(po), 1.0)).max() <= TOL
    n_d, out_d, off = track([in_world(c, hp[w]) for w, c in enumerate(base)])
    n_o, out_o, _ = track([in_world(c, po[w]) for w, c in enumerate(base)])
    n_c, out_c, _ = track(base)
    np.testing.assert_array_equal(n_d, n_o)
    np.testing.assert_array_equal(n_d, n_c)
    for w in range(B):
        for which in ("map", "ref"):
            a0, a1 = int(off[which][w]), int(off[which][w + 1])
            keep = out_d[which]["keep"][a0:a1]
            if which == "map":  # predicted from R_cur / t_cur: a pose read with the wrong layout loses the points
                assert keep.sum() >= 0.5 * (a1 - a0), (w, keep.sum())
            for name, other in (("restatement's poses", out_o), ("camera frame", out_c)):
                np.testing.assert_array_equal(keep, other[which]["keep"][a0:a1])
                m = keep.reshape(-1) != 0
                dd = np.abs(out_d[which]["fwd_xy"][a0:a1][m] - other[which]["fwd_xy"][a0:a1][m])
                assert dd.max(initial=0.0) <= LK_EPS_PX, (name, w, which, dd.max())
            if np.array_equal(hp[w], po[w]):
                for k, v in out_d[which].items():
                    assert np.array_equal(v[a0:a1], out_o[which][k][a0:a1]), (w, which, k)
    trk.close()
