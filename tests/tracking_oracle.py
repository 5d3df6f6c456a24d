"""CPU restatement of Tracking::trackMappoint (IG/tracking/tracking.cc:351-455) and Tracking::trackReferenceFrame (:457-574) for one stream,
in the output layout of icg_klt_track_frame (TEST INFRASTRUCTURE ONLY).

The forward + backward LK and its gate (:385-403, :487-506) come from a callable `lk_fb(prev_img, cur_img, prev_pts, init_pts) -> (fwd, gated
status)`: the C oracle (oracle_api.track_fb) or live cv2 (`cv2_lk_fb`).  The camera model is oracle/camera_ref.py, the RANSAC
oracle/fundamental_ref.py (or live cv2.findFundamentalMat).  Products of 3 x 3 matrices are the fixed-order sums of csrc/geom_core.cuh; both
parallax sums run in list order (the reference iterates an std::unordered_map, frame.h:80)."""
import numpy as np

from oracle import camera_ref as cref
from oracle import fundamental_ref as fref


def cam_dict(intrinsic, distortion):
    i, d = list(map(float, intrinsic)), list(map(float, distortion))
    return dict(fx=i[0], fy=i[1], cx=i[2], cy=i[3], skew=i[4] if len(i) == 5 else 0.0, k1=d[0], k2=d[1], p1=d[2], p2=d[3],
                k3=d[4] if len(d) == 5 else 0.0)


def rt_mul(A, B):
    """A^T B with M(i,j) = A(0,i) B(0,j) + A(1,i) B(1,j) + A(2,i) B(2,j), summed left to right"""
    A, B = np.asarray(A, np.float64).reshape(3, 3), np.asarray(B, np.float64).reshape(3, 3)
    M = np.zeros((3, 3))
    for i in range(3):
        for j in range(3):
            M[i, j] = A[0, i] * B[0, j] + A[1, i] * B[1, j] + A[2, i] * B[2, j]
    return M


def mat_vec(M, x, y, z):
    return M[0, 0] * x + M[0, 1] * y + M[0, 2] * z, M[1, 0] * x + M[1, 1] * y + M[1, 2] * z, M[2, 0] * x + M[2, 1] * y + M[2, 2] * z


def world2pixel(cam, pw, R, t):
    """Camera::world2pixel (camera.cc:141-147) with the fixed-order R^T (pw - t)"""
    R = np.asarray(R, np.float64).reshape(3, 3)
    d = np.asarray(pw, np.float64).reshape(-1, 3) - np.asarray(t, np.float64).reshape(1, 3)
    x = R[0, 0] * d[:, 0] + R[1, 0] * d[:, 1] + R[2, 0] * d[:, 2]
    y = R[0, 1] * d[:, 0] + R[1, 1] * d[:, 1] + R[2, 1] * d[:, 2]
    z = R[0, 2] * d[:, 0] + R[1, 2] * d[:, 1] + R[2, 2] * d[:, 2]
    return cref.cam2pixel(cam, np.stack([x, y, z], 1))


def predict_map(cam, pw, R_cur, t_cur, ops=cref):
    """pts2d_matched = distortPoints(world2pixel(pw, pose_cur)) (:367, :378)"""
    w2p = world2pixel if ops is cref else ops.world2pixel
    return ops.distort_points(cam, w2p(cam, pw, R_cur, t_cur))


def predict_ref(cam, new_xy, R_pre, R_cur, ops=cref):
    """undistort(new) -> pixel2cam -> R_cur^T R_pre . -> distortCameraPoint (:465-479)"""
    if len(new_xy) == 0:
        return np.zeros((0, 2), np.float32)
    pc = ops.pixel2cam(cam, ops.undistort_points(cam, new_xy))
    X, Y, Z = mat_vec(rt_mul(R_cur, R_pre), pc[:, 0], pc[:, 1], pc[:, 2])
    return ops.distort_camera_point(cam, np.stack([X, Y, Z], 1))


def velocity(cam, cur_undis, prev_undis, dt, ops=cref):
    """(pixel2cam(cur_undis) - pixel2cam(prev_undis)) / dt (:434, :531), x and y"""
    if len(cur_undis) == 0:
        return np.zeros((0, 2))
    a, b = ops.pixel2cam(cam, cur_undis), ops.pixel2cam(cam, prev_undis)
    return np.stack([(a[:, 0] - b[:, 0]) / dt, (a[:, 1] - b[:, 1]) / dt], 1)


def key_point_parallax(cam, Rc1c0, pp0, pp1, ops=cref):
    """Tracking::keyPointParallax (:861-871): |(R1^T R0 pc0).xy - pc1.xy| * (fx + fy) * 0.5"""
    a, b = ops.pixel2cam(cam, pp0), ops.pixel2cam(cam, pp1)
    px, py, _ = mat_vec(Rc1c0, a[:, 0], a[:, 1], a[:, 2])
    dx, dy = px - b[:, 0], py - b[:, 1]
    return np.sqrt(dx * dx + dy * dy) * ((cam["fx"] + cam["fy"]) * 0.5)


def mean_in_order(vals):
    s = 0.0
    for v in vals:  # list order, one double accumulator (parallaxFromReference*, :875-903, :909-919)
        s += float(v)
    return s / len(vals) if len(vals) else 0.0


def ransac_oracle(p1, p2, thr):
    m = fref.find_fm_ransac(p1, p2, thr, 0.99)
    return np.zeros(len(p1), bool) if m is None else np.asarray(m, bool)


def track_frame(lk_fb, prev_img, cur_img, P, map_lists=None, ref_lists=None, ransac=ransac_oracle, ops=cref):
    """Both steps for one stream (camera model from `ops`: oracle/camera_ref.py or an object with its interface).  P: dict(intrinsic, distortion, R_pre, R_cur, R_ref, t_cur, dt, ref_id, fm_threshold); the lists as
    KltTracker.track_frame takes them.  Returns (map_out, ref_out, n_out[2], parallax[2], parallax_n[2]) in KltTracker.track_frame's layout."""
    cam = cam_dict(P["intrinsic"], P["distortion"])
    Rcr = rt_mul(P["R_cur"], P["R_ref"])
    n_out, par, par_n = np.zeros(2, np.int32), np.zeros(2), np.zeros(2, np.int32)
    # ---- map list (trackMappoint)
    mo = {}
    m = map_lists or {}
    nm = len(m["prev_xy"]) if "prev_xy" in m else 0
    if nm == 0:
        par_n[0] = -1  # :372-375
    else:
        prev = np.asarray(m["prev_xy"], np.float32).reshape(-1, 2)
        fwd, st = lk_fb(prev_img, cur_img, prev, predict_map(cam, m["pw"], P["R_cur"], P["t_cur"], ops))
        keep = np.asarray(st) != 0
        fu = ops.undistort_points(cam, fwd)
        mo = dict(fwd_xy=fwd, fwd_undis_xy=fu, keep=keep.astype(np.uint8), cur_xy=fwd[keep], cur_undis_xy=fu[keep], src=np.nonzero(keep)[0].astype(np.int32))
        mo["velocity"] = velocity(cam, fu[keep], np.asarray(m["prev_undis_xy"], np.float32)[keep], P["dt"], ops)
        rk = np.asarray(m["ref_kp_xy"], np.float32).reshape(-1, 2)[keep]
        has = ~np.isnan(rk).any(axis=1)
        n_out[0] = keep.sum()
        par[0] = mean_in_order(key_point_parallax(cam, Rcr, rk[has], fu[keep][has], ops)) if has.any() else 0.0
        par_n[0] = has.sum()  # 0 when the gate emptied the list (:416-417)
    # ---- reference list (trackReferenceFrame)
    ro = {}
    r = ref_lists or {}
    nr = len(r["new_xy"]) if "new_xy" in r else 0
    if nr == 0:
        par_n[1] = -1  # :459-462
        return mo, ro, n_out, par, par_n
    new = np.asarray(r["new_xy"], np.float32).reshape(-1, 2)
    fwd, st = lk_fb(prev_img, cur_img, new, predict_ref(cam, new, P["R_pre"], P["R_cur"], ops))
    keep = np.asarray(st) != 0
    fu = ops.undistort_points(cam, fwd)
    ro = dict(fwd_xy=fwd, fwd_undis_xy=fu)
    if not keep.any():  # :513-517
        par_n[1] = -1
        ro.update(keep=keep.astype(np.uint8), cur_xy=fwd[:0], cur_undis_xy=fu[:0], velocity=np.zeros((0, 2)), ref_out_xy=fwd[:0],
                  ref_frame_id_out=np.zeros(0, np.int64), velocity_ref_out=np.zeros((0, 2)), src=np.zeros(0, np.int32))
        return mo, ro, n_out, par, par_n
    src = np.nonzero(keep)[0].astype(np.int32)
    nu = ops.undistort_points(cam, new[keep])
    cu = fu[keep]
    vel = velocity(cam, cu, nu, P["dt"], ops)
    fid = np.asarray(r["ref_frame_id"], np.int64)[keep]
    vref = np.asarray(r["velocity_ref"], np.float64).reshape(-1, 2)[keep].copy()
    newer = fid > P["ref_id"]  # :536-538
    vref[newer] = vel[newer]
    refp = np.asarray(r["ref_xy"], np.float32).reshape(-1, 2)[keep]
    same = fid == P["ref_id"]  # :911-915, before the RANSAC
    par_n[1] = same.sum()
    par[1] = mean_in_order(key_point_parallax(cam, Rcr, ops.undistort_points(cam, refp[same]), cu[same], ops)) if same.any() else 0.0
    inl = np.ones(len(src), bool)
    if len(src) >= 15:  # :546-555
        inl = ransac(nu, cu, P["fm_threshold"])
    k2 = keep.copy()
    k2[src[~inl]] = False
    ro.update(keep=k2.astype(np.uint8), cur_xy=fwd[keep][inl], cur_undis_xy=cu[inl], velocity=vel[inl], ref_out_xy=refp[inl],
              ref_frame_id_out=fid[inl], velocity_ref_out=vref[inl], src=src[inl])
    n_out[1] = inl.sum()
    return mo, ro, n_out, par, par_n


def cv2_lk_fb(cv2):
    """forward + backward cv2.calcOpticalFlowPyrLK with the reference's arguments and gate (:385-403), isOnBorder on a W x H frame"""
    def fb(a, b, p, init):
        crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.01)
        p = np.asarray(p, np.float32).reshape(-1, 1, 2)
        fwd, st, _ = cv2.calcOpticalFlowPyrLK(a, b, p, np.asarray(init, np.float32).reshape(-1, 1, 2).copy(), winSize=(21, 21), maxLevel=3,
                                              criteria=crit, flags=cv2.OPTFLOW_USE_INITIAL_FLOW)
        bwd, st2, _ = cv2.calcOpticalFlowPyrLK(b, a, fwd, p.copy(), winSize=(21, 21), maxLevel=3, criteria=crit, flags=cv2.OPTFLOW_USE_INITIAL_FLOW)
        fwd, bwd, p = fwd.reshape(-1, 2), bwd.reshape(-1, 2), p.reshape(-1, 2)
        H, W = a.shape
        fx, fy = fwd[:, 0].astype(np.float64), fwd[:, 1].astype(np.float64)
        border = (fx < 5.0) | (fy < 5.0) | (fx > W - 5.0) | (fy > H - 5.0)
        d = (bwd - p).astype(np.float64)
        dist = np.sqrt(d[:, 0] ** 2 + d[:, 1] ** 2)
        return fwd, ((st.reshape(-1) != 0) & (st2.reshape(-1) != 0) & ~border & (dist < 0.5)).astype(np.uint8)
    return fb


def cv2_ransac(cv2):
    def r(p1, p2, thr):
        _, st = cv2.findFundamentalMat(np.asarray(p1, np.float32), np.asarray(p2, np.float32), cv2.FM_RANSAC, thr, 0.99)
        return np.zeros(len(p1), bool) if st is None else st.reshape(-1) != 0
    return r
