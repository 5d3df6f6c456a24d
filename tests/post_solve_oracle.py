"""numpy restatement of the post-solve map update and outlier culling of GVINS::gvinsOptimization (IG/ic_gvins.cc:1232-1236):
updateParametersFromOptimizer (:1299-1389) and gvinsOutlierCulling (:1035-1128), plus the factor set gvinsMarginalization builds from the
culled map (:1558-1609).  Scalar Python floats in the kernel's operation order (csrc/ba_cull.cu: fixed-order sums, no FMA), so that the
device agrees to the last bit on the arithmetic and exactly on every decision away from knife edges."""
from __future__ import annotations

import math

import numpy as np


def quat_to_rot(x, y, z, w):
    """Eigen::Quaterniond::toRotationMatrix, row-major 3 x 3 as a flat list"""
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [1.0 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1.0 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1.0 - (txx + tyy)]


def unit_quat_to_rot(q):
    x, y, z, w = (float(v) for v in q)
    n = math.sqrt(x * x + y * y + z * z + w * w)
    return quat_to_rot(x / n, y / n, z / n, w / n)


def quat_vec_norm(M):
    """|Quaterniond(M).vec()| (Eigen's matrix -> quaternion branches)"""
    q = [0.0, 0.0, 0.0, 0.0]
    t = M[0] + M[4] + M[8]
    if t > 0.0:
        t = math.sqrt(t + 1.0)
        q[3] = 0.5 * t
        t = 0.5 / t
        q[0], q[1], q[2] = (M[7] - M[5]) * t, (M[2] - M[6]) * t, (M[3] - M[1]) * t
    else:
        i = 0
        if M[4] > M[0]:
            i = 1
        if M[8] > M[4 * i]:
            i = 2
        j = (i + 1) % 3
        k = (j + 1) % 3
        t = math.sqrt(M[4 * i] - M[4 * j] - M[4 * k] + 1.0)
        q[i] = 0.5 * t
        t = 0.5 / t
        q[3] = (M[3 * k + j] - M[3 * j + k]) * t
        q[j] = (M[3 * j + i] + M[3 * i + j]) * t
        q[k] = (M[3 * k + i] + M[3 * i + k]) * t
    return math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2])


def _f32(v):
    return np.float32(v)


def pixel2cam(cam, u, v):
    y = (float(v) - cam["cy"]) / cam["fy"]
    x = (float(u) - cam["cx"] - cam["skew"] * y) / cam["fx"]
    return x, y


def cam2pixel(cam, x, y, z):
    return _f32((cam["fx"] * x + cam["skew"] * y) / z + cam["cx"]), _f32(cam["fy"] * y / z + cam["cy"])


def world2cam(P, pw):
    d0, d1, d2 = pw[0] - P[9], pw[1] - P[10], pw[2] - P[11]
    return (P[0] * d0 + P[3] * d1 + P[6] * d2, P[1] * d0 + P[4] * d1 + P[7] * d2, P[2] * d0 + P[5] * d1 + P[8] * d2)


def good_to_track(cam, kp, P, pw, std, scale=3.0, depth_scale=1.0):
    """Tracking::isGoodToTrack(kp, pose, pw, scale, depth_scale) -> (passes, error or None)"""
    x, y, z = world2cam(P, pw)
    if not (z > 1.0 and z < 200.0 * depth_scale):
        return False, None
    pu, pv = cam2pixel(cam, x, y, z)
    ex, ey = float(_f32(pu - _f32(kp[0]))), float(_f32(pv - _f32(kp[1])))
    err = math.sqrt(ex * ex + ey * ey)
    return (not (err > std * scale)), err


def update_and_cull(prob, cam, std, ci):
    """One window.  prob: pose (K x 7: p, q_xyzw), ext (8), invdepth (L), K, L.  cam: dict of fx, fy, cx, cy, skew.  ci: the
    icg_ba_cull_window inputs (R_bc, t_bc, td_bc, estimate_ext, estimate_td, lm_ref_node, lm_ref_kp, obs_off, obs_node, obs_kp)."""
    K, L = int(prob["K"]), int(prob["L"])
    ext = [float(v) for v in np.asarray(prob["ext"], np.float64)]
    pose = np.asarray(prob["pose"], np.float64).reshape(-1, 7)
    rho = np.asarray(prob["invdepth"], np.float64)
    Rbc = [float(v) for v in np.asarray(ci["R_bc"], np.float64).reshape(-1)]
    tbc = [float(v) for v in np.asarray(ci["t_bc"], np.float64).reshape(-1)]
    accepted = -1
    if ci.get("estimate_ext", 1):
        R = unit_quat_to_rot(ext[3:7])
        d0, d1, d2 = ext[0] - tbc[0], ext[1] - tbc[1], ext[2] - tbc[2]
        dt = math.sqrt(d0 * d0 + d1 * d1 + d2 * d2)
        M = [R[3 * i] * Rbc[3 * j] + R[3 * i + 1] * Rbc[3 * j + 1] + R[3 * i + 2] * Rbc[3 * j + 2] for i in range(3) for j in range(3)]
        dr = quat_vec_norm(M) * (180.0 / math.pi)
        accepted = 0 if (dt > 1.0) or (dr > 5.0) else 1
        if accepted:
            Rbc, tbc = R, ext[:3]
    td = ext[7] if ci.get("estimate_td", 1) else float(ci.get("td_bc", 0.0))
    cam_pose = np.zeros((K, 12))
    P = []
    for k in range(K):
        Rq = unit_quat_to_rot(pose[k, 3:7])
        row = [Rq[3 * i] * Rbc[j] + Rq[3 * i + 1] * Rbc[3 + j] + Rq[3 * i + 2] * Rbc[6 + j] for i in range(3) for j in range(3)]
        row += [float(pose[k, i]) + (Rq[3 * i] * tbc[0] + Rq[3 * i + 1] * tbc[1] + Rq[3 * i + 2] * tbc[2]) for i in range(3)]
        P.append(row)
        cam_pose[k] = row
    off = np.asarray(ci["obs_off"], np.int64)
    ref_node = np.asarray(ci["lm_ref_node"], np.int64)
    ref_kp = np.asarray(ci["lm_ref_kp"], np.float32).reshape(-1, 2)
    obs_node = np.asarray(ci["obs_node"], np.int64)
    obs_kp = np.asarray(ci["obs_kp"], np.float32).reshape(-1, 2)
    n_obs = int(off[L]) if L > 0 else 0
    lm_pw, lm_depth = np.zeros((L, 3)), np.zeros(L)
    lm_outlier, obs_outlier = np.zeros(L, np.uint8), np.zeros(n_obs, np.uint8)
    counts = [0, 0, 0, 0, 0]
    with np.errstate(all="ignore"):
        for l in range(L):
            Pr = P[int(ref_node[l])]
            x, y = pixel2cam(cam, ref_kp[l, 0], ref_kp[l, 1])
            depth = float(np.float64(1.0) / np.float64(rho[l]))  # 1 / 0 = inf, as in C
            c0, c1, c2 = x * depth, y * depth, 1.0 * depth
            pw = [(Pr[3 * i] * c0 + Pr[3 * i + 1] * c1 + Pr[3 * i + 2] * c2) + Pr[9 + i] for i in range(3)]
            lm_pw[l], lm_depth[l] = pw, depth
            errs_sum, n_good, reason = 0.0, 0, 0
            for o in range(int(off[l]), int(off[l + 1])):
                k = int(obs_node[o])
                good, err = good_to_track(cam, obs_kp[o], P[k], pw, std)
                if good:
                    errs_sum += err
                    n_good += 1
                else:
                    obs_outlier[o] = 1
                    if k == int(ref_node[l]):
                        reason |= 1
                        counts[0] += 1
                        counts[2] += 1
                        break
                    counts[1] += 1
            if n_good < 2:
                reason |= 2
                counts[0] += 1
                counts[3] += 1
            elif errs_sum / float(n_good) > std:
                reason |= 4
                counts[0] += 1
                counts[4] += 1
            lm_outlier[l] = reason
    return dict(R_bc_out=np.array(Rbc).reshape(3, 3), t_bc_out=np.array(tbc), td_bc_out=td, ext_accepted=accepted, cam_pose=cam_pose, lm_pw=lm_pw,
                lm_depth=lm_depth, lm_outlier=lm_outlier, obs_outlier=obs_outlier, counts=np.array(counts, np.int32))


def culled_factor_mask(prob, ci, res, node_in_map):
    """gvinsMarginalization's reprojection factors after the culling (:1558-1609), per factor row: the landmark is not a culling outlier,
    neither the observation nor the landmark's reference observation is a feature outlier, and the observing keyframe is in the map.
    The chi-square activity plays no part."""
    F, L = int(prob["F"]), int(prob["L"])
    mask = np.ones(F, np.uint8)
    lm_bad = np.asarray(res["lm_outlier"]) != 0
    off = np.asarray(ci["obs_off"])
    for l in range(L):
        for o in range(int(off[l]), int(off[l + 1])):
            if not res["obs_outlier"][o]:
                continue
            if ci["obs_node"][o] == ci["lm_ref_node"][l]:
                lm_bad[l] = True
            if ci["obs_factor"][o] >= 0:
                mask[ci["obs_factor"][o]] = 0
    f_lm, f_obs = np.asarray(prob["f_lm"]), np.asarray(prob["f_obs"])
    nim = np.asarray(node_in_map, bool)
    mask[lm_bad[f_lm] | ~nim[f_obs]] = 0
    return mask
