"""CPU: the restatement of Tracking::triangulation (tests/triangulation_oracle.py, IG/tracking/tracking.cc:690-798) pinned by hand cases for every
branch and gate, and by noise-free scenes where the triangulated points recover the ground truth."""
import numpy as np

from oracle import camera_ref as cref
from tests import triangulation_oracle as tri
from tests.tracking_oracle import cam_dict

INTR = [400.0, 400.0, 320.0, 240.0, 0.0]
FAR = [5000.0, 5000.0, 320.0, 240.0, 0.0]  # a long focal length: enough parallax for points hundreds of metres away
D0 = [0.0, 0.0, 0.0, 0.0, 0.0]
I3 = np.eye(3)
REF_ID, CUR_ID = 10, 20


def Ry(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def pixel(intr, R, t, pw):
    return cref.cam2pixel(cam_dict(intr, D0), np.array([tri.world2cam(pw, R, t)]))[0]


def params(t_cur, R_cur=I3, intr=INTR, window_normal=False, std=1.5, **kw):
    return dict(intrinsic=intr, distortion=D0, R_cur=R_cur, t_cur=np.asarray(t_cur, float), cur_id=CUR_ID, ref_id=REF_ID, window_normal=window_normal,
                reprojection_error_std=std, **kw)


def one(P, kfs, pw, fid=REF_ID, R0=I3, t0=(0, 0, 0), noise=(0, 0, 0, 0)):
    """a one-point list: pw seen from the keyframe (R0, t0) and the current pose, with pixel noise (ref x, y, cur x, y)"""
    r = pixel(P["intrinsic"], R0, t0, pw) + np.float32(noise[:2])
    c = pixel(P["intrinsic"], P["R_cur"], P["t_cur"], pw) + np.float32(noise[2:])
    return dict(ref_out_xy=np.float32([r]), ref_frame_id_out=np.int64([fid]), cur_xy=np.float32([c]), velocity_ref_out=np.array([[0.25, -0.5]]),
                velocity=np.array([[1.5, 2.5]]))


def run(P, kfs, lists):
    return tri.triangulation(P, kfs, lists)


KF = {REF_ID: (I3, (0.0, 0.0, 0.0), True), 5: (I3, (0.0, 0.0, 0.0), False)}


def test_empty_list_returns_false():
    lo, new, cnt, _, _ = run(params((1, 0, 0)), KF, None)
    assert list(cnt) == [-1, 0, 0, 0, 0] and len(new["pw"]) == 0 and len(lo["cur_xy"]) == 0


def test_success_recovers_the_point_and_fills_the_new_map_point():
    P = params((1, 0, 0))
    L = one(P, KF, (0.5, -0.3, 8.0))
    lo, new, cnt, st, _ = run(P, KF, L)
    assert list(cnt) == [0, 1, 0, 0, 0] and list(st) == [2] and len(lo["cur_xy"]) == 0
    assert np.abs(new["pw"][0] - [0.5, -0.3, 8.0]).max() <= 1e-6 * 8
    assert abs(new["depth"][0] - 8.0) <= 1e-5
    assert np.array_equal(new["ref_xy"][0], L["ref_out_xy"][0]) and np.array_equal(new["cur_xy"][0], L["cur_xy"][0])
    assert np.array_equal(new["velocity_ref"][0], [0.25, -0.5]) and np.array_equal(new["velocity_cur"][0], [1.5, 2.5])
    assert new["ref_frame_id"][0] == REF_ID and new["src"][0] == 0


def test_reset_precedes_the_window_test_and_keeps_velocity_ref():
    P = params((1, 0, 0), window_normal=True)
    kfs = dict(KF)
    kfs[15] = (I3, (0.0, 0.0, 0.0), False)  # a newer frame that has left the map: the reset rule still comes first
    L = one(P, kfs, (0.5, -0.3, 8.0), fid=15)
    lo, new, cnt, st, _ = run(P, kfs, L)
    assert list(cnt) == [1, 0, 0, 1, 0] and list(st) == [1]
    assert np.array_equal(lo["ref_out_xy"][0], L["cur_xy"][0]) and lo["ref_frame_id_out"][0] == CUR_ID
    assert np.array_equal(lo["velocity_ref_out"][0], [0.25, -0.5]) and np.array_equal(lo["cur_xy"][0], L["cur_xy"][0])


def test_out_of_window_only_when_the_window_is_normal():
    P = params((1, 0, 0), window_normal=True)
    L = one(P, KF, (0.5, -0.3, 8.0), fid=5)
    _, _, cnt, st, _ = run(P, KF, L)
    assert list(cnt) == [0, 0, 0, 0, 1] and list(st) == [0]
    _, new, cnt, st, _ = run(dict(P, window_normal=False), KF, L)  # the same point triangulates when the window is not full
    assert list(cnt) == [0, 1, 0, 0, 0] and len(new["pw"]) == 1
    _, _, cnt, _, _ = run(P, KF, one(P, KF, (0.5, -0.3, 8.0), fid=REF_ID))  # in the map: not out of window
    assert list(cnt) == [0, 1, 0, 0, 0]


def test_low_parallax_keeps_the_point():
    P = params((0.1, 0, 0))  # 400 * 0.1 / 8 = 5 px < 10
    lo, _, cnt, st, diag = run(P, KF, one(P, KF, (0.5, -0.3, 8.0)))
    assert list(cnt) == [1, 0, 0, 0, 0] and list(st) == [1] and diag[0][0][0] < 10
    # the rotation is the point's own reference frame's: the same pixels with a rotated keyframe give a different parallax
    kfs = {REF_ID: (Ry(0.05), (0.0, 0.0, 0.0), True)}
    L = one(P, kfs, (0.5, -0.3, 8.0))
    _, _, _, _, d2 = run(P, kfs, L)
    assert d2[0][0][0] > 10


def test_depth_bounds_reject_each_gate_on_its_own():
    cases = [  # (focal, point depth in the keyframe, current position, which gate) -> near / far bound of the reference / current gate
        (INTR, 0.8, (0.3, 0, -0.4), "ref near"),
        (INTR, 1.2, (0.3, 0, 0.4), "cur near"),
        (FAR, 600.5, (2, 0, 1), "ref far"),
        (FAR, 599.5, (2, 0, -1), "cur far"),
    ]
    for intr, z0, tc, what in cases:
        P = params(tc, intr=intr, std=5.0)
        _, _, cnt, st, diag = run(P, KF, one(P, KF, (0.01, 0.02, z0)))
        assert list(cnt) == [0, 0, 1, 0, 0] and list(st) == [0], what
        zs = [q for q, thr in diag[0] if thr in (1.0, 600.0)]
        if what.startswith("ref"):
            assert len(zs) == 2 and not (1 < zs[0] < 600), what  # decided by the first gate's depth
        else:
            assert len(zs) == 4 and 1 < zs[0] < 600 and not (1 < zs[2] < 600), what


def test_depth_is_clamped_above_200():
    P = params((2, 0, 0), intr=FAR)
    _, new, cnt, _, _ = run(P, KF, one(P, KF, (0.3, 0.1, 300.0)))
    assert list(cnt) == [0, 1, 0, 0, 0]
    assert new["depth"][0] == 10.0 and abs(new["pw"][0][2] - 300.0) <= 1e-3


def reproj_errors(P, L):
    _, _, _, _, diag = run(dict(P, reprojection_error_std=1e9), KF, L)
    errs = [q for q, thr in diag[0] if thr == 1e9]
    return errs


def test_each_reprojection_gate_rejects_on_its_own():
    # the DLT shares the residual between the views by their depths: the closer view keeps the larger pixel error
    found = {}
    for which, tc in (("cur", (1, 0, 2)), ("ref", (1, 0, -4))):
        P = params(tc)
        L = one(P, KF, (0.5, -0.3, 4.0), noise=(0, 1.5, 0, 0))
        e0, e1 = reproj_errors(P, L)
        assert (e0 > 1.5 * e1) if which == "ref" else (e1 > 1.5 * e0), (which, e0, e1)
        found[which] = (P, L, e0, e1)
    for which, (P, L, e0, e1) in found.items():
        std = 0.5 * (e0 + e1)
        _, _, cnt, _, diag = run(dict(P, reprojection_error_std=std), KF, L)
        assert list(cnt) == [0, 0, 1, 0, 0], which
        errs = [q for q, thr in diag[0] if thr == std]
        assert len(errs) == (1 if which == "ref" else 2), which
        _, _, cnt, _, _ = run(dict(P, reprojection_error_std=max(e0, e1)), KF, L)  # <= std passes
        assert list(cnt) == [0, 1, 0, 0, 0], which


def float_double_cases(P, kfs, n, seed):
    """one-point lists near the left image edge, where world2pixel and the measurement straddle a power of two and the float difference of
    camera.cc:156 rounds; yields (lists, std) with std = the larger float error, which a double difference would exceed"""
    cam = cam_dict(P["intrinsic"], P["distortion"])
    rng = np.random.default_rng(seed)
    for _ in range(n):
        z = rng.uniform(3, 9)
        u, v = rng.uniform(0.2, 2.5), rng.uniform(0.2, 2.5)
        pw = np.array([(u - 320.0) / 400.0 * z, (v - 240.0) / 400.0 * z, z])
        L = one(P, kfs, pw, noise=tuple(rng.uniform(-1.2, 1.2, 4)))
        _, new, cnt, _, diag = tri.triangulation(dict(P, reprojection_error_std=1e9), kfs, L)
        if cnt[1] != 1:
            continue
        ef = [q for q, thr in diag[0] if thr == 1e9]
        ed = []
        for (R, t), pp in (((I3, (0.0, 0.0, 0.0)), L["ref_out_xy"]), ((P["R_cur"], P["t_cur"]), L["cur_xy"])):
            px = cref.cam2pixel(cam, np.array([tri.world2cam(new["pw"][0], R, t)]))[0]
            q = cref.undistort_points(cam, pp)[0]
            ed.append(np.hypot(float(px[0]) - float(q[0]), float(px[1]) - float(q[1])))
        if max(ed) > max(ef):
            yield L, max(ef)


def test_reprojection_difference_is_taken_in_float():
    P = params((1, 0, 0))
    hits = 0
    for L, std in float_double_cases(P, KF, 300, 3):
        _, _, cnt, _, _ = run(dict(P, reprojection_error_std=std), KF, L)
        assert list(cnt) == [0, 1, 0, 0, 0]  # admitted at the float error; the double error exceeds std
        _, _, cnt, _, _ = run(dict(P, reprojection_error_std=np.nextafter(std, 0)), KF, L)
        assert list(cnt) == [0, 0, 1, 0, 0]
        hits += 1
    assert hits >= 3, hits


def test_stable_compaction_and_counts_over_a_mixed_list():
    P = params((1, 0, 0), window_normal=True)
    kfs = dict(KF)
    parts = [one(P, kfs, (0.5, -0.3, 8.0)), one(P, kfs, (0.5, -0.3, 8.0), fid=12), one(P, kfs, (0.5, -0.3, 8.0), fid=5),
             one(dict(P, t_cur=np.array([0.1, 0, 0])), kfs, (0.1, 0.1, 8.0)), one(P, kfs, (0.2, 0.1, 6.0)), one(P, kfs, (0.1, 0.3, 0.5))]
    L = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    lo, new, cnt, st, _ = run(P, kfs, L)
    assert list(st) == [2, 1, 0, 1, 2, 0]
    assert list(cnt) == [2, 2, 1, 1, 1]
    assert list(lo["src"]) == [1, 3] and list(new["src"]) == [0, 4]
    assert list(lo["ref_frame_id_out"]) == [CUR_ID, REF_ID]


def test_missing_frame_reports_minus_two():
    P = params((1, 0, 0))
    lo, new, cnt, _, _ = run(P, KF, one(P, KF, (0.5, -0.3, 8.0), fid=7))
    assert cnt[0] == -2 and len(new["pw"]) == 0


def test_noise_free_scenes_recover_ground_truth():
    rng = np.random.default_rng(11)
    total = 0
    for trial in range(5):
        kfs = {REF_ID - j: (Ry(0.02 * j), (-0.5 * j, 0.1 * j, 0.0), True) for j in range(4)}
        P = params((1.5, 0.2, 0.3), R_cur=Ry(-0.05), std=1.0)
        n = 120
        fids = rng.integers(REF_ID - 3, REF_ID + 1, n)
        pw = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(5, 12, n)], 1)
        rows = [one(P, kfs, pw[k], fid=int(fids[k]), R0=kfs[int(fids[k])][0], t0=kfs[int(fids[k])][1]) for k in range(n)]
        L = {k: np.concatenate([r[k] for r in rows]) for k in rows[0]}
        _, new, cnt, st, _ = run(P, kfs, L)
        assert cnt[1] >= n // 2, (trial, cnt)
        truth = pw[new["src"]]
        rel = np.linalg.norm(new["pw"] - truth, axis=1) / np.linalg.norm(truth, axis=1)
        assert rel.max() <= 1e-6, (trial, rel.max())
        total += int(cnt[1])
    assert total >= 300
