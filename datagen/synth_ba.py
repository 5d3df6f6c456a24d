"""Synthetic sliding-window problems for hot path B (SURVEY.md section 8d, cfg 3 / cfg 4).  Input generator only.

K nodes at 0.5 s spacing (dt_node) on a planar arc (5 m/s, yaw rate 5 deg/s), IMU at 200 Hz with the noise model of
config/gvins.yaml:26-31, GNSS on every 2nd node, L landmarks at depth U(5, 60) m with reference frame j mod 5 observed in
frames r+1 .. min(K-1, r+3+(j mod 6)), pixel noise 0.5 px / f=787, reprojection std 1.5/787, extrinsic of
config/gvins.yaml:78-79 (free), td = 0 (free).  Initial guess = truth (+) N(0; 0.1 m, 0.5 deg, 0.1 m/s), rho (1+N(0,0.1)).

`preintegrate(state16, iewn, gravity, noise5, imu[n,7]) -> (blob[480], pn[n-1,4], end_state10)` is injected so that the
generator can run on the product's host-side preintegration (bench) or on the oracle's (tests).
"""
from __future__ import annotations

import math

import numpy as np

WIE = 7.2921151467e-5
D2R = math.pi / 180.0
F_PIX = 787.0
ANTLEVER = np.array([-0.37, 0.008, 0.353])
Q_B_C = np.array([0.497766, 0.502679, 0.501396, 0.498141])  # xyzw
T_B_C = np.array([0.074, -0.030, 0.128])
NOISE5 = np.array([0.1 * D2R / 60.0, 0.1 / 60.0, 50.0 * D2R / 3600.0, 50.0 * 1e-5, 3600.0])  # arw, vrw, gb, ab, corr
GRAVITY = np.array([0.0, 0.0, 9.7936])
LAT = 30.5 * D2R
IEWN = np.array([WIE * math.cos(LAT), 0.0, -WIE * math.sin(LAT)])


# ---------------------------------------------------------------------------------------------- quaternion helpers (xyzw)
def q_mul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def q_mat(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def q_from_rotvec(rv):
    a = np.linalg.norm(rv)
    if a == 0:
        return np.array([0.0, 0.0, 0.0, 1.0])
    ax = rv / a
    return np.concatenate([math.sin(a / 2) * ax, [math.cos(a / 2)]])


def q_yaw(psi):
    return np.array([0.0, 0.0, math.sin(psi / 2), math.cos(psi / 2)])


# ---------------------------------------------------------------------------------------------- trajectory + IMU
def trajectory(t, speed=5.0, yaw_rate=5.0 * D2R, heave=True):
    """Planar arc at `speed` (m/s) and `yaw_rate` (rad/s), a straight line when yaw_rate is 0; heave adds the 0.02 m vertical oscillation.
    speed = yaw_rate = 0 with heave=False is a vehicle standing still."""
    psi = 0.3 + yaw_rate * t
    z = (0.02 * math.sin(0.5 * t), 0.01 * math.cos(0.5 * t), -0.005 * math.sin(0.5 * t)) if heave else (0.0, 0.0, 0.0)
    if yaw_rate == 0:
        p = np.array([speed * t * math.cos(psi), speed * t * math.sin(psi), z[0]])
        return p, np.array([speed * math.cos(psi), speed * math.sin(psi), z[1]]), np.array([0.0, 0.0, z[2]]), psi
    r = speed / yaw_rate
    p = np.array([r * (math.sin(psi) - math.sin(0.3)), -r * (math.cos(psi) - math.cos(0.3)), z[0]])
    v = np.array([speed * math.cos(psi), speed * math.sin(psi), z[1]])
    a = np.array([-speed * yaw_rate * math.sin(psi), speed * yaw_rate * math.cos(psi), z[2]])
    return p, v, a, psi


def imu_samples(t0, t1, rate, rng, bg, ba, yaw_rate=5.0 * D2R, earth=True, speed=5.0, heave=True, noise_scale=1.0):
    """(n, 7) rows: dt, dtheta[3], dvel[3]; row 0 is the sample AT t0 (imu0 of the preintegration).
    noise_scale multiplies the white noise; 0 gives noise-free increments.  The same random numbers are drawn whatever its value, and the
    default (1) generates the same arrays as before the keyword existed."""
    n = int(round((t1 - t0) * rate))
    dt = 1.0 / rate
    out = np.zeros((n + 1, 7))
    arw, vrw = NOISE5[0] * noise_scale, NOISE5[1] * noise_scale
    for i in range(n + 1):
        tm = t0 + (i - 0.5) * dt  # mid-point of the sampling interval ending at t0 + i dt
        p, v, a, psi = trajectory(tm, speed, yaw_rate, heave)
        R = q_mat(q_yaw(psi))
        iewn = IEWN if earth else np.zeros(3)  # earth = False: the PreintegrationNormal world (no Earth rotation / Coriolis)
        w_b = np.array([0.0, 0.0, yaw_rate]) + R.T @ iewn
        f_b = R.T @ (a - GRAVITY + 2.0 * np.cross(iewn, v))
        out[i, 0] = dt
        out[i, 1:4] = (w_b + bg) * dt + rng.normal(0, arw * math.sqrt(dt), 3)
        out[i, 4:7] = (f_b + ba) * dt + rng.normal(0, vrw * math.sqrt(dt), 3)
    return out


# ---------------------------------------------------------------------------------------------- problem
def make_window(preintegrate, K=10, L=300, seed=2024, full_visibility=False, perturb=True, with_marg=False, pixel_noise=0.5, with_priors=False,
                gnss_every=2, earth=True, n_ref=5, dt_node=0.5, speed=5.0, yaw_rate=5.0 * D2R, heave=True):
    """n_ref: landmark j is anchored in node j mod n_ref (j mod (K - 1) when K <= n_ref).  A larger n_ref spreads the landmarks over more
    nodes, so fewer of them are marginalized with node 0.  The anchor itself draws no random numbers: the default (5) generates the same
    arrays as before the keyword existed.
    dt_node: time between consecutive nodes (s).  Shorter spacing keeps landmarks in view over more nodes: long tracks.  The default (0.5)
    generates the same arrays as before the keyword existed.
    speed (m/s), yaw_rate (rad/s), heave: the trajectory (see trajectory()); speed = yaw_rate = 0, heave=False is a vehicle standing still,
    whose landmarks are seen with no parallax.  They draw no random numbers: the defaults generate the same arrays as before they existed."""
    rng = np.random.Generator(np.random.PCG64(seed))
    dtk, rate = dt_node, 200.0
    times = np.arange(K) * dtk
    bg_true = rng.normal(0, 20.0 * D2R / 3600.0, 3)
    ba_true = rng.normal(0, 20.0 * 1e-5, 3)
    pose_t = np.zeros((K, 7))
    mix_t = np.zeros((K, 9))
    for k, t in enumerate(times):
        p, v, _, psi = trajectory(t, speed, yaw_rate, heave)
        pose_t[k, :3] = p
        pose_t[k, 3:] = q_yaw(psi)
        mix_t[k, :3], mix_t[k, 3:6], mix_t[k, 6:9] = v, bg_true, ba_true
    ext_t = np.concatenate([T_B_C, Q_B_C / np.linalg.norm(Q_B_C), [0.0]])

    # ---- landmarks and reprojection factors
    Rbc = q_mat(ext_t[3:7])
    f_lm, f_ref, f_obs, f_const = [], [], [], []
    invdepth_t = np.zeros(L)

    def to_cam(k, pw):
        Rk = q_mat(pose_t[k, 3:])
        pb = Rk.T @ (pw - pose_t[k, :3])
        return Rbc.T @ (pb - ext_t[:3])

    for j in range(L):
        r = j % n_ref if K > n_ref else j % max(1, K - 1)
        depth = rng.uniform(5.0, 60.0)
        uv = np.array([rng.uniform(-0.7, 0.7), rng.uniform(-0.3, 0.3), 1.0])
        pc0 = uv * depth
        pw = q_mat(pose_t[r, 3:]) @ (Rbc @ pc0 + ext_t[:3]) + pose_t[r, :3]
        invdepth_t[j] = 1.0 / depth
        last = K - 1 if full_visibility else min(K - 1, r + 3 + (j % 6))
        pts0 = uv + np.array([rng.normal(0, pixel_noise / F_PIX), rng.normal(0, pixel_noise / F_PIX), 0.0])
        for o in range(r + 1, last + 1):
            pc1 = to_cam(o, pw)
            if pc1[2] < 2.0 or abs(pc1[0] / pc1[2]) > 0.85 or abs(pc1[1] / pc1[2]) > 0.65:
                continue  # outside the field of view (1280x560 at f = 787 -> +-0.81 x +-0.36; keep a margin)
            pts1 = np.array([pc1[0] / pc1[2] + rng.normal(0, pixel_noise / F_PIX), pc1[1] / pc1[2] + rng.normal(0, pixel_noise / F_PIX), 1.0])
            vel0 = np.array([rng.normal(0, 0.05), rng.normal(0, 0.02), 0.0])
            vel1 = np.array([rng.normal(0, 0.05), rng.normal(0, 0.02), 0.0])
            f_lm.append(j), f_ref.append(r), f_obs.append(o)
            f_const.append(np.concatenate([pts0, pts1, vel0, vel1, [0.0, 0.0]]))
    F = len(f_lm)

    # ---- IMU preintegration between consecutive nodes (linearised at slightly wrong biases, as in operation)
    blobs = np.zeros((K - 1, 480))
    pn_all, pn_off = [], [0]
    bg_lin = bg_true + rng.normal(0, 5.0 * D2R / 3600.0, 3)
    ba_lin = ba_true + rng.normal(0, 5.0 * 1e-5, 3)
    for k in range(K - 1):
        imu = imu_samples(times[k], times[k + 1], rate, rng, bg_true, ba_true, yaw_rate=yaw_rate, earth=earth, speed=speed, heave=heave)
        state16 = np.concatenate([pose_t[k], mix_t[k, :3], bg_lin, ba_lin])
        blob, pn, _ = preintegrate(state16, IEWN if earth else None, GRAVITY, NOISE5, imu)
        blobs[k] = blob
        pn_all.append(pn)
        pn_off.append(pn_off[-1] + pn.shape[0])
    pn_all = np.concatenate(pn_all, axis=0) if len(pn_all) else np.zeros((0, 4))

    # ---- GNSS on every 2nd node
    gnss_node = np.arange(0, K, gnss_every, dtype=np.int32)
    gnss_std = np.tile(np.array([0.05, 0.05, 0.1]), (len(gnss_node), 1))
    gnss_blh = np.zeros((len(gnss_node), 3))
    for i, k in enumerate(gnss_node):
        gnss_blh[i] = pose_t[k, :3] + q_mat(pose_t[k, 3:]) @ ANTLEVER + rng.normal(0, 1, 3) * gnss_std[i]

    # ---- initial guess
    pose0, mix0, ext0, rho0 = pose_t.copy(), mix_t.copy(), ext_t.copy(), invdepth_t.copy()
    if perturb:
        for k in range(K):
            pose0[k, :3] += rng.normal(0, 0.1, 3)
            q = q_mul(pose0[k, 3:], q_from_rotvec(rng.normal(0, 0.5 * D2R, 3)))
            pose0[k, 3:] = q / np.linalg.norm(q)
            mix0[k, :3] += rng.normal(0, 0.1, 3)
            mix0[k, 3:6] = bg_lin
            mix0[k, 6:9] = ba_lin
        rho0 = rho0 * (1.0 + rng.normal(0, 0.1, L))
        ext0[:3] += rng.normal(0, 0.01, 3)
        q = q_mul(ext0[3:7], q_from_rotvec(rng.normal(0, 0.2 * D2R, 3)))
        ext0[3:7] = q / np.linalg.norm(q)
        ext0[7] = 0.002

    prob = dict(
        K=K, L=L, F=F, pose=pose0.reshape(-1).copy(), mix=mix0.reshape(-1).copy(), ext=ext0.copy(), invdepth=rho0.copy(),
        ext_const=0, td_const=0,
        f_lm=np.array(f_lm, np.int32), f_ref=np.array(f_ref, np.int32), f_obs=np.array(f_obs, np.int32),
        f_const=np.array(f_const, np.float64).reshape(-1), f_active=np.ones(F, np.uint8),
        reproj_std=1.5 / F_PIX, reproj_huber=1,
        n_imu=K - 1, imu_blob=blobs.reshape(-1).copy(), pn=pn_all.reshape(-1).copy(), pn_off=np.array(pn_off, np.int32),
        has_imu_error=1, has_pose_prior=0, pose_prior=np.zeros(7), pose_prior_std=np.ones(6), has_mix_prior=0,
        mix_prior=np.zeros(9), mix_prior_std=np.ones(9),
        n_gnss=len(gnss_node), gnss_node=gnss_node, gnss_blh=gnss_blh.reshape(-1).copy(), gnss_std=gnss_std.reshape(-1).copy(),
        lever=ANTLEVER.copy(), gnss_huber=1,
        marg_r=0, marg_nblocks=0, marg_block_type=np.zeros(0, np.int32), marg_block_node=np.zeros(0, np.int32),
        marg_x0=np.zeros(0), marg_J0=np.zeros(0), marg_e0=np.zeros(0),
    )
    if with_marg:
        # a synthetic linear-Gaussian prior on node 0 / node 1 / extrinsic / td around the (perturbed) initial values:
        # J0 upper-triangular random well-conditioned, e0 small -- exercises MarginalizationFactor (not a physical prior)
        types = np.array([0, 1, 0, 1, 2, 3], np.int32)
        nodes = np.array([0, 0, 1, 1, 0, 0], np.int32)
        lsz = {0: 6, 1: 9, 2: 6, 3: 1}
        r = int(sum(lsz[int(t)] for t in types))
        A = np.triu(rng.normal(0, 1.0, (r, r)))
        A[np.arange(r), np.arange(r)] = np.abs(A[np.arange(r), np.arange(r)]) + 3.0
        scale = np.concatenate([[10.0] * 6, [5.0] * 3, [2000.0] * 3, [500.0] * 3, [10.0] * 6, [5.0] * 3, [2000.0] * 3, [500.0] * 3, [50.0] * 6, [100.0]])
        J0 = A * scale[None, :]
        x0 = np.concatenate([pose_t[0], mix_t[0], pose_t[1], mix_t[1], ext_t[:7], [0.0]])
        prob.update(marg_r=r, marg_nblocks=len(types), marg_block_type=types, marg_block_node=nodes, marg_x0=x0,
                    marg_J0=J0.reshape(-1).copy(), marg_e0=rng.normal(0, 0.1, r))
    if with_priors:
        # first-window priors as GVINS::constructPrior builds them (IG/ic_gvins.cc:720-760): the initial pose / mix of node 0 with their stds
        pp = pose_t[0].copy()
        pp[:3] += rng.normal(0, 0.05, 3)
        q = q_mul(pp[3:], q_from_rotvec(rng.normal(0, 0.2 * D2R, 3)))
        pp[3:] = q / np.linalg.norm(q)
        mp = mix_t[0].copy()
        mp[:3] += rng.normal(0, 0.05, 3)
        prob.update(has_pose_prior=1, pose_prior=pp, pose_prior_std=np.array([0.1, 0.1, 0.2, 0.5 * D2R, 0.5 * D2R, 1.0 * D2R]),
                    has_mix_prior=1, mix_prior=mp,
                    mix_prior_std=np.array([0.1, 0.1, 0.1] + [100.0 * D2R / 3600.0] * 3 + [100.0 * 1e-5] * 3))
    truth = dict(pose=pose_t, mix=mix_t, ext=ext_t, invdepth=invdepth_t)
    return prob, truth
