"""CPU restatement of Tracking::triangulation (IG/tracking/tracking.cc:690-798) for one stream, in the layout of KltTracker.triangulate
(TEST INFRASTRUCTURE ONLY).

The camera model comes from `ops` (oracle/camera_ref.py by default, or an object with its interface, e.g. the library's icg_camera_* host
entry points) and the 4 x 4 solve from `tri(T0, T1, pc0, pc1) -> pw` (oracle/fundamental_ref.triangulate_point, numpy SVD, by default).
Products of 3 x 3 matrices and world2cam are the fixed-order sums of csrc/geom_core.cuh.  Besides the reference's outputs, every point
reports the quantities that decided it, with their thresholds, so that a test can tell a knife-edge decision from a real difference."""
import numpy as np

from oracle import camera_ref as cref
from oracle import fundamental_ref as fref
from tests.tracking_oracle import cam_dict, key_point_parallax, rt_mul

TRACK_MIN_PARALLAX = 10.0                  # tracking.h:114
NEAREST, FARTHEST, DEFAULT_DEPTH = 1.0, 200.0, 10.0  # mappoint.h:51-53


def world2cam(pw, R, t):
    """Camera::world2cam (camera.cc:145-147): R^T (pw - t), fixed-order sums"""
    R = np.asarray(R, np.float64).reshape(3, 3)
    d0, d1, d2 = (float(pw[k]) - float(t[k]) for k in range(3))
    return (R[0, 0] * d0 + R[1, 0] * d1 + R[2, 0] * d2, R[0, 1] * d0 + R[1, 1] * d1 + R[2, 1] * d2, R[0, 2] * d0 + R[1, 2] * d1 + R[2, 2] * d2)


def pose_tcw(R, t):
    """Tracking::pose2Tcw (:851-859), top 3 rows: [R^T | -R^T t], -R^T t as the fixed-order sum of world2cam"""
    R, t = np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64).reshape(3)
    T = np.zeros((3, 4))
    for i in range(3):
        T[i, :3] = R[:, i]
        T[i, 3] = -(R[0, i] * t[0] + R[1, i] * t[1] + R[2, i] * t[2])
    return T


def _world2pixel(cam, pw, R, t, ops):
    if ops is cref:  # fixed-order world2cam, cam2pixel in float
        return cref.cam2pixel(cam, np.array([world2cam(pw, R, t)]))[0]
    return ops.world2pixel(cam, np.asarray(pw, np.float64).reshape(1, 3), np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64))[0]


def good_to_track(cam, pp, R, t, pw, std, ops=cref, diag=None):
    """Tracking::isGoodToTrack(pp, pose, pw, 1.0, 3.0) (:813-829): 1 < z < 600, then |world2pixel(pw) - pp| <= std with the differences in
    float (camera.cc:153-157)"""
    z = world2cam(pw, R, t)[2]
    if diag is not None:
        diag += [(z, NEAREST), (z, FARTHEST * 3.0)]
    if not (z > NEAREST and z < FARTHEST * 3.0):
        return False
    px = _world2pixel(cam, pw, R, t, ops)
    ex, ey = float(np.float32(px[0]) - np.float32(pp[0])), float(np.float32(px[1]) - np.float32(pp[1]))
    err = np.sqrt(ex * ex + ey * ey)
    if diag is not None:
        diag.append((err, std))
    return not (err > std * 1.0)


def triangulation(P, keyframes, lists, ops=cref, tri=fref.triangulate_point):
    """P: dict(intrinsic, distortion, R_cur, t_cur, cur_id, ref_id, window_normal, reprojection_error_std[, triangulate]); keyframes: dict
    id -> (R, t, in_map); lists: dict(ref_out_xy, ref_frame_id_out, cur_xy, velocity_ref_out, velocity) as KltTracker.triangulate takes it.
    Returns (list_out, new, counts[5], status, diag): list_out / new / counts as KltTracker.triangulate; status per input point (0 dropped,
    1 kept, 2 new map point); diag per input point = the (quantity, threshold) pairs that were evaluated, in order."""
    cam = cam_dict(P["intrinsic"], P["distortion"])
    lists = lists or {}
    n = len(lists["cur_xy"]) if "cur_xy" in lists else 0
    refp = np.asarray(lists.get("ref_out_xy", np.zeros((0, 2))), np.float32).reshape(n, 2).copy()
    fid = np.asarray(lists.get("ref_frame_id_out", np.zeros(0)), np.int64).reshape(n).copy()
    cur = np.asarray(lists.get("cur_xy", np.zeros((0, 2))), np.float32).reshape(n, 2)
    vref = np.asarray(lists.get("velocity_ref_out", np.zeros((0, 2))), np.float64).reshape(n, 2)
    vcur = np.asarray(lists.get("velocity", np.zeros((0, 2))), np.float64).reshape(n, 2)
    empty_out = dict(ref_out_xy=refp, ref_frame_id_out=fid, cur_xy=cur, velocity_ref_out=vref, src=np.arange(n, dtype=np.int32))
    if not P.get("triangulate", True) or n == 0:  # :692-694
        return empty_out, _new([]), np.array([-1, 0, 0, 0, 0], np.int32), np.ones(n, np.int32), [[] for _ in range(n)]
    missing = [f for f in fid if f <= P["ref_id"] and int(f) not in keyframes]
    if missing:
        return empty_out, _new([]), np.array([-2, 0, 0, 0, 0], np.int32), np.ones(n, np.int32), [[] for _ in range(n)]
    ru = ops.undistort_points(cam, refp)  # :708-713
    cu = ops.undistort_points(cam, cur)
    T1 = pose_tcw(P["R_cur"], P["t_cur"])
    status, diag, new = np.zeros(n, np.int32), [], []
    n_succ = n_out = n_reset = n_time = 0
    for k in range(n):
        d = []
        diag.append(d)
        if fid[k] > P["ref_id"]:  # :723-730
            refp[k], fid[k] = cur[k], P["cur_id"]
            status[k] = 1
            n_reset += 1
            continue
        R0, t0, in_map = keyframes[int(fid[k])]
        if P["window_normal"] and not in_map:  # :733-737
            n_time += 1
            continue
        par = float(key_point_parallax(cam, rt_mul(P["R_cur"], R0), ru[k:k + 1], cu[k:k + 1], ops)[0])  # :740-745
        d.append((par, TRACK_MIN_PARALLAX))
        if par < TRACK_MIN_PARALLAX:
            status[k] = 1
            continue
        pc0, pc1 = ops.pixel2cam(cam, ru[k:k + 1])[0], ops.pixel2cam(cam, cu[k:k + 1])[0]
        pw = np.asarray(tri(pose_tcw(R0, t0), T1, pc0[:2], pc1[:2]), np.float64).reshape(3)  # :747-753
        std = P["reprojection_error_std"]
        if not (good_to_track(cam, ru[k], R0, t0, pw, std, ops, d) and good_to_track(cam, cu[k], P["R_cur"], P["t_cur"], pw, std, ops, d)):
            n_out += 1  # :756-760
            continue
        depth = world2cam(pw, R0, t0)[2]  # :764-765
        if depth < NEAREST or depth > FARTHEST:  # mappoint.cc:39-42
            depth = DEFAULT_DEPTH
        status[k] = 2
        n_succ += 1
        new.append(dict(pw=pw, depth=depth, ref_undis_xy=ru[k], ref_xy=refp[k], cur_undis_xy=cu[k], cur_xy=cur[k], velocity_cur=vcur[k],
                        velocity_ref=vref[k], ref_frame_id=fid[k], src=k))
    keep = status == 1  # :788-791
    lo = dict(ref_out_xy=refp[keep], ref_frame_id_out=fid[keep], cur_xy=cur[keep], velocity_ref_out=vref[keep], src=np.nonzero(keep)[0].astype(np.int32))
    return lo, _new(new), np.array([keep.sum(), n_succ, n_out, n_reset, n_time], np.int32), status, diag


def _new(rows):
    spec = {"pw": (np.float64, 3), "depth": (np.float64, 1), "ref_undis_xy": (np.float32, 2), "ref_xy": (np.float32, 2), "cur_undis_xy": (np.float32, 2),
            "cur_xy": (np.float32, 2), "velocity_cur": (np.float64, 2), "velocity_ref": (np.float64, 2), "ref_frame_id": (np.int64, 1), "src": (np.int32, 1)}
    out = {}
    for k, (dt, c) in spec.items():
        a = np.array([r[k] for r in rows], dt).reshape(len(rows), c)
        out[k] = a.reshape(-1) if c == 1 else a
    return out


def knife_edge(diag_k, rel=1e-9):
    """True when one of the point's deciding quantities lies within `rel` (relative) of its threshold"""
    return any(abs(q - t) <= rel * max(abs(t), 1.0) for q, t in diag_k)


class AbiOps:
    """the oracle/camera_ref.py interface on the library's host entry points (icg_camera_*), for the composition of existing ABI calls"""

    @staticmethod
    def _c(cam):
        from ic_gvins_b200.camera import Camera
        return Camera([cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["skew"]], [cam["k1"], cam["k2"], cam["p1"], cam["p2"], cam["k3"]])

    def undistort_points(self, cam, px):
        return self._c(cam).undistortPoints(px) if len(px) else np.zeros((0, 2), np.float32)

    def pixel2cam(self, cam, px):
        return self._c(cam).pixel2cam(px) if len(px) else np.zeros((0, 3))

    def world2pixel(self, cam, pw, R, t):
        return self._c(cam).world2pixel(pw, R, t) if len(pw) else np.zeros((0, 2), np.float32)


def abi_triangulate(T0, T1, pc0, pc1):
    """icg_triangulate_points on one pair"""
    from ic_gvins_b200.camera import triangulatePoints
    return triangulatePoints(np.asarray(T0).reshape(1, 3, 4), np.asarray(T1).reshape(3, 4), np.asarray(pc0).reshape(1, 2), np.asarray(pc1).reshape(1, 2))[0]
