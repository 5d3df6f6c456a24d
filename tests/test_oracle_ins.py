"""CPU: the INS window restatement (tests/ins_oracle.cpp) pinned by hand cases for every branch of getInsWindowIndex, isNeedInterpolation,
imuInterpolation, redoInsMechanization, statePoseInterpolation and runFusion's window step, by an mpmath restatement of insMechanization over
1000-sample windows in both forms, and by the synthetic trajectory the IMU samples were drawn from."""
import math

import mpmath
import numpy as np
import pytest

from datagen import synth_ba
from tests import ins_oracle as io
from tests import preint_mp as pm

NORMAL = {"with_earth": False, "gravity": synth_ba.GRAVITY}
EARTH = {"with_earth": True, "gravity": synth_ba.GRAVITY, "iewn": synth_ba.IEWN}
BG, BA = np.array([2e-4, -1e-4, 3e-4]), np.array([0.02, -0.01, 0.015])
pytestmark = pytest.mark.skipif(not io.HAVE_CXX, reason="no host C++ compiler for the INS restatement")
POSE_B_C = np.concatenate([synth_ba.q_mat(synth_ba.Q_B_C).reshape(9), synth_ba.T_B_C])


def rows8(t0, t1, rate, earth=True, seed=3, noise_scale=1.0, **kw):
    """synth_ba.imu_samples with the sample time in front: (n, 8) rows (time, dt, dtheta, dvel), row 0 AT t0"""
    imu = synth_ba.imu_samples(t0, t1, rate, np.random.default_rng(seed), BG, BA, earth=earth, noise_scale=noise_scale, **kw)
    return np.concatenate([(t0 + np.arange(imu.shape[0]) / rate)[:, None], imu], axis=1)


def state_at(t, bg=BG, ba=BA):
    p, v, _, psi = synth_ba.trajectory(t)
    return np.concatenate([[t], p, synth_ba.q_yaw(psi), v, bg, ba])


def normalised(state17):
    """stateFromData's q.normalize(), in the oracle's order of the squares (w, x, y, z)"""
    s = np.array(state17, np.float64)
    x, y, z, w = s[4:8]
    n = math.sqrt(w * w + x * x + y * y + z * z)
    s[4:8] = [x / n, y / n, z / n, w / n]
    return s


def mechanized(rows, cfg, state17, capacity=4000):
    """an oracle window over rows, mechanized from state17 placed just after row 0 (isNeedInterpolation -1) and kept whole (reserved large)"""
    o = io.OracleIns(1, capacity)
    assert o.push([rows[:2]], cfg) == 0
    st = np.array(state17, np.float64)
    st[0] = rows[0, 0] + 0.5e-4
    assert o.redo(st[None], cfg, reserved=10 ** 6)[0] == 1
    assert o.push([rows[2:]], cfg) == 0
    return o


# ---------------------------------------------------------------------------------------------- getInsWindowIndex / isNeedInterpolation
def test_window_index_cases():
    t = 10.0 + np.arange(7) * 0.005
    assert io.window_index(t, 9.0) == 0            # before the front
    assert io.window_index(t, t[0]) == 1           # at the front
    assert io.window_index(t, t[3]) == 4           # exactly on a row: the first row after it
    assert io.window_index(t, t[3] + 1e-3) == 4    # between rows
    assert io.window_index(t, t[-1] - 1e-9) == 6
    assert io.window_index(t, t[-1]) == 0          # at the back
    assert io.window_index(t, 11.0) == 0           # after the back
    assert io.window_index(t[:1], t[0]) == 0       # one row: never inside
    assert io.window_index([], 1.0) == 0
    big = np.arange(65537) * 0.005                 # the largest window whose search ends within the reference's cap
    for k in (1, 2, 3, 1000, 32768, 65535):
        assert io.window_index(big, big[k - 1] + 1e-4) == k


def test_need_interpolation_cases():
    assert io.need_interpolation(1.0, 1.005, 1.0 + 0.5e-4) == -1
    assert io.need_interpolation(1.0, 1.005, 1.005 - 0.5e-4) == 1
    assert io.need_interpolation(1.0, 1.005, 1.0025) == 2
    assert io.need_interpolation(1.0, 1.005, 1.0) == 0       # exactly the earlier sample
    assert io.need_interpolation(1.0, 1.005, 1.005) == 0
    assert io.need_interpolation(1.0, 1.005, 0.9) == 0


def test_imu_interpolation_split():
    row = np.array([2.005, 0.005, 1e-3, -2e-3, 3e-3, 0.04, -0.05, 0.06])
    a, b = io.interpolate(row, 2.003)
    scale = (2.005 - 2.003) / 0.005
    assert a[0] == 2.003 and a[1] == 0.005 - (2.005 - 2.003)
    assert b[0] == 2.005 and b[1] == 2.005 - 2.003
    np.testing.assert_array_equal(a[2:], row[2:] * (1 - scale))
    np.testing.assert_array_equal(b[2:], row[2:] * scale)


# ---------------------------------------------------------------------------------------------- redoInsMechanization
def _seeded(cfg, n=12, capacity=1000):
    rows = rows8(20.0, 20.0 + (n - 1) / 200.0, 200.0, earth=cfg["with_earth"])
    o = io.OracleIns(1, capacity)
    assert o.push([rows], cfg) == 0
    return o, rows


@pytest.mark.parametrize("cfg", [NORMAL, EARTH], ids=["normal", "earth"])
def test_redo_cases(cfg):
    n, k = 12, 5
    for case in (-1, 1, 2, 0):
        o, rows = _seeded(cfg, n)
        old = o.window(0)[1]
        st = state_at(0.0)
        t = {-1: rows[k - 1, 0] + 0.3e-4, 1: rows[k, 0] - 0.3e-4, 2: rows[k - 1, 0] + 0.002, 0: rows[k - 1, 0]}[case]
        st[0] = t
        assert io.need_interpolation(rows[k - 1, 0], rows[k, 0], t) == case
        assert o.redo(st[None], cfg, reserved=100)[0] == 1
        imu, x = o.window(0)
        np.testing.assert_array_equal(imu, rows)
        np.testing.assert_array_equal(x[:k], old[:k])  # entries before index are never touched
        s = normalised(st)
        if case == -1:
            s = io.mechanize(cfg, rows[k - 1], rows[k], s)
            pre = rows[k]
            np.testing.assert_array_equal(x[k], s)
        elif case == 1:
            s[0] = rows[k, 0]
            pre = rows[k]
            np.testing.assert_array_equal(x[k], s)
        elif case == 2:
            a, b = io.interpolate(rows[k], t)
            s = io.mechanize(cfg, a, b, s)
            pre = b                                     # the scaled second part is imu_pre of the next step
            np.testing.assert_array_equal(x[k], s)
            assert not np.array_equal(io.mechanize(cfg, rows[k], rows[k + 1], s), io.mechanize(cfg, b, rows[k + 1], s))
        else:
            pre = rows[k]
            np.testing.assert_array_equal(x[k], old[k])  # the quirk: nothing stored at index
        for j in range(k + 1, n):
            s = io.mechanize(cfg, pre, rows[j], s)
            pre = rows[j]
            np.testing.assert_array_equal(x[j], s)


def test_redo_pruning_and_outside():
    for k, reserved in ((5, 2), (5, 5), (5, 7), (1, 0), (11, 2)):
        o, rows = _seeded(NORMAL, 12)
        st = state_at(0.0)
        st[0] = rows[k - 1, 0] + 0.002
        assert o.redo(st[None], NORMAL, reserved=reserved)[0] == 1
        imu, _ = o.window(0)
        drop = k - reserved if k >= reserved else 0
        np.testing.assert_array_equal(imu, rows[drop:])
    o, rows = _seeded(NORMAL, 12)
    before = o.window(0)
    for t in (rows[0, 0] - 1.0, rows[-1, 0], rows[-1, 0] + 1.0):
        st = state_at(0.0)
        st[0] = t
        assert o.redo(st[None], NORMAL)[0] == -1
        for a, b in zip(o.window(0), before):
            np.testing.assert_array_equal(a, b)
    assert o.camera_pose([rows[3, 0]], POSE_B_C)[1][0] == -1  # still not mechanized
    assert o.redo(state_at(0.0)[None], NORMAL, redo=[0])[0] == 0


def test_redo_normalises_q():
    o, rows = _seeded(NORMAL, 12)
    st = state_at(0.0)
    st[0] = rows[4, 0] - 0.3e-4  # case 1: the state is stored as given, with q normalised
    st[4:8] *= 3.0
    o.redo(st[None], NORMAL, reserved=100)
    x = o.window(0)[1][4]
    np.testing.assert_array_equal(x[4:8], normalised(st)[4:8])


# ---------------------------------------------------------------------------------------------- runFusion's window step
def test_push_initialization_keeps_newest_1000():
    rows = rows8(0.0, 1500 / 200.0, 200.0)
    o = io.OracleIns(1, 2000)
    assert o.push([rows[:700]], NORMAL) == 0
    assert o.push([rows[700:1400]], NORMAL) == 0
    imu, x = o.window(0)
    np.testing.assert_array_equal(imu, rows[400:1400])
    assert not x.any()


def test_push_rejects():
    rows = rows8(0.0, 0.1, 200.0)
    o = io.OracleIns(1, 1000)
    assert o.push([rows[:5]], NORMAL) == 0
    before = o.window(0)
    for bad in (rows[4:6], rows[3:4], np.stack([rows[5], rows[5]])):
        assert o.push([bad], NORMAL) == -1
        for a, b in zip(o.window(0), before):
            np.testing.assert_array_equal(a, b)
    long = rows8(0.0, 1100 / 200.0, 200.0)
    o = mechanized(long[:600], NORMAL, state_at(0.0), capacity=1000)
    assert o.push([long[600:1001]], NORMAL) == -1
    assert o.push([long[600:1000]], NORMAL) == 0


def test_push_mechanizes_from_last_row():
    rows = rows8(0.0, 0.2, 200.0)
    o = mechanized(rows, EARTH, state_at(0.0))
    imu, x = o.window(0)
    for k in range(2, rows.shape[0]):
        np.testing.assert_array_equal(x[k], io.mechanize(EARTH, rows[k - 1], rows[k], x[k - 1]))


# ---------------------------------------------------------------------------------------------- getCameraPoseFromInsWindow
def _pose_of(state17, pose_b_c):
    R = synth_ba.q_mat(state17[4:8])
    Rbc = pose_b_c[:9].reshape(3, 3)
    return np.concatenate([(R @ Rbc).reshape(9), state17[1:4] + R @ pose_b_c[9:]])


def test_camera_pose_cases():
    rows = rows8(0.0, 0.1, 200.0)
    o = mechanized(rows, EARTH, state_at(0.0))
    _, x = o.window(0)
    stamps = [rows[0, 0] - 0.01, rows[3, 0], rows[3, 0] + 0.0021, rows[-1, 0], rows[-1, 0] + 0.01]
    got = [o.camera_pose([t], POSE_B_C) for t in stamps]  # one stream, one stamp per call
    pose, found = np.concatenate([g[0] for g in got]), np.concatenate([g[1] for g in got])
    np.testing.assert_array_equal(found, [0, 1, 1, 0, 0])
    for k in (0, 3, 4):
        np.testing.assert_allclose(pose[k], _pose_of(x[-1], POSE_B_C), rtol=0, atol=1e-12)
    np.testing.assert_array_equal(pose[1], io.pose_interpolate(x[3], x[4], rows[3, 0], POSE_B_C))
    np.testing.assert_array_equal(pose[2], io.pose_interpolate(x[3], x[4], rows[3, 0] + 0.0021, POSE_B_C))
    # exactly on a row: scale uses the STATES' times, which equal the rows' here
    np.testing.assert_allclose(pose[1], _pose_of(x[3], POSE_B_C), rtol=0, atol=1e-12)


def test_pose_interpolation_identity_and_negative_w():
    s0 = state_at(1.0)
    s1 = s0.copy()
    s1[0], s1[1:4] = 1.01, s0[1:4] + np.array([0.1, -0.2, 0.3])
    out = io.pose_interpolate(s0, s1, 1.0025, POSE_B_C)  # dq exactly identity: angle 0, axis (1, 0, 0)
    ref = s0.copy()
    ref[1:4] = s0[1:4] + (s1[1:4] - s0[1:4]) * 0.25
    np.testing.assert_allclose(out, _pose_of(ref, POSE_B_C), rtol=0, atol=1e-14)
    # w < 0: q1 = -(q0 * small rotation); AngleAxis flips the axis so the interpolation takes the short way
    rv = np.array([0.01, -0.02, 0.03])
    q1 = -synth_ba.q_mul(s0[4:8], synth_ba.q_from_rotvec(rv))
    s1[4:8] = q1
    out = io.pose_interpolate(s0, s1, 1.0025, POSE_B_C)
    ref[4:8] = synth_ba.q_mul(s0[4:8], synth_ba.q_from_rotvec(0.25 * rv))
    np.testing.assert_allclose(out, _pose_of(ref, POSE_B_C), rtol=0, atol=1e-12)


# ---------------------------------------------------------------------------------------------- mpmath restatement over 1000 samples
def _mech_mp(cfg, rows, state17):
    """insMechanization chained over rows[1:], each from the previous row, at 40 digits (shared structure with tests/preint_mp.py)"""
    f = mpmath.mpf
    with mpmath.workdps(pm.DPS):
        x = [f(float(v)) for v in state17]
        p, v, bg, ba = x[1:4], x[8:11], x[11:14], x[14:17]
        q = (x[7], x[4], x[5], x[6])
        g = [f(float(c)) for c in cfg["gravity"]]
        iw = [f(float(c)) for c in cfg.get("iewn", (0, 0, 0))]
        one = f(1)
        R = [[f(float(c)) for c in r] for r in rows]
        out = []
        for k in range(1, len(R)):
            pr, cu = R[k - 1], R[k]
            dt = cu[1]
            pth, pvl = pm._sub(pr[2:5], pm._sc(pr[1], bg)), pm._sub(pr[5:8], pm._sc(pr[1], ba))
            cth, cvl = pm._sub(cu[2:5], pm._sc(dt, bg)), pm._sub(cu[5:8], pm._sc(dt, ba))
            dvfb = pm._add(pm._add(cvl, pm._sc(f(0.5), pm._cross(cth, cvl))), pm._sc(one / 12, pm._add(pm._cross(pth, cvl), pm._cross(pvl, cth))))
            dth = pm._add(cth, pm._sc(one / 12, pm._cross(pth, cth)))
            if cfg["with_earth"]:
                qnn = pm._rv2q(pm._sc(-dt, iw))
                Rn = pm._qmat(qnn)
                half = [[(Rn[i][j] + (1 if i == j else 0)) / 2 for j in range(3)] for i in range(3)]
                dvel = pm._add(pm._mv(half, pm._mv(pm._qmat(q), dvfb)), pm._sc(dt, pm._sub(g, pm._sc(f(2), pm._cross(iw, v)))))
                q = pm._qnorm(pm._qmul(pm._qmul(qnn, q), pm._rv2q(dth)))
            else:
                dvel = pm._add(pm._mv(pm._qmat(q), dvfb), pm._sc(dt, g))
                q = pm._qnorm(pm._qmul(q, pm._rv2q(dth)))
            p = pm._add(p, pm._add(pm._sc(dt, v), pm._sc(dt / 2, dvel)))
            v = pm._add(v, dvel)
            out.append([float(c) for c in (*p, q[1], q[2], q[3], q[0], *v)])
    return np.array(out)


# measured worst error over the two 1000-sample windows below, in units of each group's scale (|p|, 1, |v|): 1.4e-15 (p), 1.1e-15 (q),
# 2.5e-15 (v); the bounds are about 10x.  The rounding of each step is carried on by the chain, so the error grows with the window.
TOL_WINDOW = {"p": 2e-14, "q": 2e-14, "v": 3e-14}


@pytest.mark.parametrize("cfg", [NORMAL, EARTH], ids=["normal", "earth"])
def test_mechanization_1000_samples_vs_mpmath(cfg):
    rows = rows8(100.0, 100.0 + 999 / 200.0, 200.0, earth=cfg["with_earth"], seed=11)
    assert rows.shape[0] == 1000
    st = state_at(100.0)
    o = mechanized(rows, cfg, st)
    _, x = o.window(0)
    st = normalised(st)
    st[0] = rows[0, 0]
    np.testing.assert_array_equal(x[1], io.mechanize(cfg, rows[0], rows[1], st))
    ref = _mech_mp(cfg, rows, st)
    got = x[1:, 1:11]
    err = np.abs(got - ref)
    ep = (err[:, 0:3].max(axis=1) / np.linalg.norm(ref[:, 0:3], axis=1)).max()
    eq = err[:, 3:7].max()
    ev = (err[:, 7:10].max(axis=1) / np.linalg.norm(ref[:, 7:10], axis=1)).max()
    assert ep <= TOL_WINDOW["p"] and eq <= TOL_WINDOW["q"] and ev <= TOL_WINDOW["v"], (ep, eq, ev)


@pytest.mark.parametrize("cfg", [NORMAL, EARTH], ids=["normal", "earth"])
def test_mechanization_follows_trajectory(cfg):
    """noise-free samples of synth_ba's arc, known biases: the mechanized 5 s track stays within a few cm / mrad of the trajectory"""
    rows = rows8(50.0, 55.0, 200.0, earth=cfg["with_earth"], noise_scale=0.0)
    o = mechanized(rows, cfg, state_at(50.0))
    _, x = o.window(0)
    for k in range(100, rows.shape[0], 100):
        t = rows[k, 0]
        p, v, _, psi = synth_ba.trajectory(t)
        assert np.linalg.norm(x[k, 1:4] - p) < 0.05, (k, x[k, 1:4], p)
        assert np.linalg.norm(x[k, 8:11] - v) < 0.02
        dq = synth_ba.q_mul(np.array([-x[k, 4], -x[k, 5], -x[k, 6], x[k, 7]]), synth_ba.q_yaw(psi))
        assert 2 * np.linalg.norm(dq[:3]) < 2e-3
