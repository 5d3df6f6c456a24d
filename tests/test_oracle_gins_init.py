"""CPU: the restatement of gvinsInitialization (tests/gins_init_oracle.cpp) pinned by one hand case per branch -- a time of 0, 19 vs 20
rows, rows exactly at last_time / gnss_time, each zero-velocity threshold at its knife edge, zero velocity then motion, the dual-antenna
yaw, a displacement below 0.5 m, pitch from GNSS without levelling and a window that cannot serve the series -- and by an independent
mpmath computation of one case's levelling and initial state."""
import math

import mpmath
import numpy as np
import pytest

from datagen import synth_ba
from tests import gins_init_oracle as go
from tests.test_oracle_ins import rows8

pytestmark = pytest.mark.skipif(not go.HAVE_CXX, reason="no host C++ compiler for the INS restatement")
RATE, G = 200.0, 9.7936
GYR_BIAS_STD = synth_ba.NOISE5[2]
EARTH = {"with_earth": True, "gravity": synth_ba.GRAVITY}
NORMAL = {"with_earth": False, "gravity": synth_ba.GRAVITY}
BG_TRUE = np.array([3e-4, -2e-4, 1e-4])
F_B = np.array([0.05, -0.08, -G])  # a slightly tilted vehicle at rest


def moving(t0, t1, seed=1, earth=True):
    """rows (time, dt, dtheta, dvel) of a vehicle in motion: the synthetic arc plus white noise well above both zero-velocity thresholds"""
    r = rows8(t0, t1, RATE, earth=earth, seed=seed)
    rng = np.random.default_rng(100 + seed)
    r[:, 2:5] += rng.normal(0, 1e-4, (r.shape[0], 3))
    r[:, 5:8] += rng.normal(0, 2.5e-3, (r.shape[0], 3))
    return r


def still(t0, t1, seed=2, noise=(2e-7, 5e-5)):
    """rows of a vehicle at rest: constant bias and specific force, small white noise"""
    n = int(round((t1 - t0) * RATE)) + 1
    t = t0 + np.arange(n) / RATE
    rng = np.random.default_rng(seed)
    dth = BG_TRUE / RATE + rng.normal(0, noise[0], (n, 3))
    dv = F_B / RATE + rng.normal(0, noise[1], (n, 3))
    return np.concatenate([t[:, None], np.full((n, 1), 1 / RATE), dth, dv], axis=1)


def init(last, gnss, disp=(3.0, 4.0, -0.2), **kw):
    g = dict(gnss_time=gnss, gnss_blh=tuple(np.array([1.0, 2.0, 0.5]) + disp), last_time=last, last_blh=(1.0, 2.0, 0.5), gravity=G,
             imudatarate=RATE, origin_blh=(0.5, 2.0, 30.0), antlever=(0.1, 0.2, 0.3))
    g.update(kw)
    return g


def run(rows, g, cfg=EARTH, o=None, reserved=2):
    o = o or go.OracleGins(1)
    assert o.push([rows], cfg) == 0
    out, cfg_out = o.gins_initialize([g], [cfg], GYR_BIAS_STD, reserved=reserved)
    return o, out, cfg_out


def test_time_zero():
    r = moving(10.0, 13.0)
    for g in (init(0.0, 12.0), init(11.0, 0.0)):
        o, out, _ = run(r, g)
        assert out["status"][0] == -1


def test_19_vs_20_rows_and_ends_excluded():
    """last_time and gnss_time exactly on rows: those rows are excluded, so 21 rows apart leaves 19 / 22 apart leaves 20"""
    r = moving(10.0, 13.0)
    t = r[:, 0]
    o, out, _ = run(r, init(t[200], t[220]))
    assert out["status"][0] == -2
    o, out, _ = run(r, init(t[200], t[221]))
    assert out["status"][0] == 1
    # one ulp inside either end takes the end row in
    o, out, _ = run(r, init(np.nextafter(t[200], 0), t[220]))
    assert out["status"][0] == 1
    o, out, _ = run(r, init(t[200], np.nextafter(t[220], 99)))
    assert out["status"][0] == 1


def _std_rate(vals):
    """detectZeroVelocity's statistic on one column, in its order of operations"""
    n = len(vals)
    inv = 1.0 / float(n)
    a = 0.0
    for v in vals:
        a += v
    a *= inv
    s = 0.0
    for v in vals:
        s += (v - a) * (v - a)
    return math.sqrt(s * inv) * RATE


def _knife(col, thr, base):
    """the largest alternating amplitude d whose statistic is below thr (the next double's is not)"""
    def stat(d):
        vals = [base[0] + (d if k % 2 == 0 else -d) for k in range(len(base))]
        return _std_rate(vals), vals
    lo, hi = 0.0, thr / RATE * 4
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        if stat(mid)[0] < thr:
            lo = mid
        else:
            hi = mid
    d = lo
    while stat(np.nextafter(d, 1))[0] < thr:
        d = np.nextafter(d, 1)
    assert stat(d)[0] < thr <= stat(np.nextafter(d, 1))[0]
    return stat(d)[1], stat(np.nextafter(d, 1))[1]


@pytest.mark.parametrize("col,thr", [(2, 0.002), (4, 0.002), (5, 0.1), (7, 0.1)])
def test_zero_velocity_threshold_knife_edge(col, thr):
    r = still(10.0, 12.0, noise=(0.0, 0.0))
    inside = (r[:, 0] > 10.5) & (r[:, 0] < 11.5)
    below, above = _knife(col, thr, r[inside, col])
    for vals, zero in ((below, True), (above, False)):
        rr = r.copy()
        rr[inside, col] = vals
        o, out, _ = run(rr, init(10.5, 11.5))
        assert out["status"][0] == (-3 if zero else 1), (col, zero, out["status"])


def test_zero_velocity_then_motion_keeps_levelling():
    o = go.OracleGins(1)
    r0 = still(10.0, 12.0)
    o, out, _ = run(r0, init(10.5, 11.5), o=o)
    assert out["status"][0] == -3 and out["has_zero_velocity"][0] == 1
    sel = r0[(r0[:, 0] > 10.5) & (r0[:, 0] < 11.5)]
    avg = sel[:, 2:8].mean(axis=0)
    np.testing.assert_allclose(out["bg"][0], avg[:3] * RATE, rtol=1e-12)
    np.testing.assert_allclose(out["initatt"][0, :2], [-math.asin(avg[4] * RATE / G), math.asin(avg[3] * RATE / G)], rtol=1e-12)
    # nothing else changed: the window is still unmechanized
    assert not o.window(0)[1][:, 1:].any()
    roll, pitch = out["initatt"][0, :2].copy()
    r1 = moving(12.0 + 1 / RATE, 14.0)
    o, out, _ = run(r1, init(12.5, 13.5), o=o)
    assert out["status"][0] == 1
    assert out["initatt"][0, 0] == roll and out["initatt"][0, 1] == pitch
    assert out["initatt"][0, 2] == math.atan2(4.0, 3.0)
    np.testing.assert_array_equal(out["mix_prior_std"][0, 3:6], GYR_BIAS_STD * 3)
    np.testing.assert_array_equal(out["state17"][0, 11:14], out["bg"][0])


def test_dual_antenna_yaw():
    o, out, _ = run(moving(10.0, 13.0), init(11.0023, 12.0023, disp=(0.0, 0.0, 0.0), last_yaw_valid=1, last_yaw=-2.5))
    assert out["status"][0] == 1
    np.testing.assert_array_equal(out["initatt"][0], [0.0, 0.0, -2.5])
    assert out["mix_prior_std"][0, 3] == 7200 * (math.pi / 180.0) / 3600


def test_displacement_below_half_metre():
    r = moving(10.0, 13.0)
    o, out, _ = run(r, init(11.0023, 12.0023, last_blh=(0.0, 0.0, 0.0), gnss_blh=(np.nextafter(0.5, 0), 0.0, 0.0)))
    assert out["status"][0] == -4
    assert not o.window(0)[1][:, 1:].any()
    o, out, _ = run(r, init(11.0023, 12.0023, last_blh=(0.0, 0.0, 0.0), gnss_blh=(0.5, 0.0, 0.0)))
    assert out["status"][0] == 1


def test_pitch_from_gnss_without_levelling():
    o, out, cfg = run(moving(10.0, 13.0, earth=False), init(11.0023, 12.0023, disp=(3.0, 4.0, -1.0)), cfg=NORMAL)
    assert out["status"][0] == 1 and out["has_zero_velocity"][0] == 0
    np.testing.assert_array_equal(out["initatt"][0], [0.0, math.atan(1.0 / 5.0), math.atan2(4.0, 3.0)])
    assert cfg[0]["gravity"] == (0.0, 0.0, G) and cfg[0]["iewn"] == (0.0, 0.0, 0.0)


@pytest.mark.parametrize("case", ["gnss_after_back", "last_before_front", "reserved_0"])
def test_window_cannot_serve(case):
    """gnss_time at or after the window's back, last_time before its front, or a redo that keeps no row before last_time (reserved 0), so
    that getInsWindowIndex(last_time) is 0 on the window the redo leaves: status -5 and the window and slots as they were"""
    r = moving(10.0, 13.0)
    g, reserved = {"gnss_after_back": (init(12.5, 13.5), 2), "last_before_front": (init(9.5, 10.5), 2), "reserved_0": (init(11.0023, 12.0023), 0)}[case]
    o = go.OracleGins(1)
    assert o.push([r], EARTH) == 0
    before = o.window(0)
    slots = o.slot7.copy()
    out, _ = o.gins_initialize([g], [EARTH], GYR_BIAS_STD, reserved=reserved)
    assert out["status"][0] == -5, out["status"]
    after = o.window(0)
    np.testing.assert_array_equal(before[0], after[0]), np.testing.assert_array_equal(before[1], after[1])
    np.testing.assert_array_equal(slots, o.slot7)


def test_series_covers_the_interval():
    """both ends interpolated: the series' dt after its first row adds up to gnss_time - last_time, the last row's time is gnss_time"""
    o, out, _ = run(moving(10.0, 13.0), init(11.0023, 12.0023))
    s = out["series"][0]
    assert out["n_series"][0] == s.shape[0] == 202
    assert s[-1, 0] == 12.0023 and s[0, 0] == 11.0023
    assert abs(s[1:, 1].sum() - 1.0) < 1e-13


def test_levelling_and_initial_state_against_mpmath():
    """the zero-velocity levelling, euler2quaternion and p = last_blh - q antlever, at 40 digits"""
    mpmath.mp.dps = 40
    o = go.OracleGins(1)
    r0 = still(10.0, 12.0)
    o, out, _ = run(r0, init(10.5, 11.5), o=o)
    sel = r0[(r0[:, 0] > 10.5) & (r0[:, 0] < 11.5)]
    avg = [mpmath.fsum(mpmath.mpf(float(v)) for v in sel[:, c]) / len(sel) for c in range(2, 8)]
    roll, pitch = -mpmath.asin(avg[4] * RATE / G), mpmath.asin(avg[3] * RATE / G)
    assert abs(out["initatt"][0, 0] - roll) <= 1e-15 * abs(roll) + 1e-18
    assert abs(out["initatt"][0, 1] - pitch) <= 1e-15 * abs(pitch) + 1e-18
    for c in range(3):
        assert abs(out["bg"][0, c] - avg[c] * RATE) <= 1e-13 * abs(avg[c] * RATE)
    r1 = moving(12.0 + 1 / RATE, 14.0)
    g = init(12.5, 13.5)
    o, out, _ = run(r1, g, o=o)
    att = [mpmath.mpf(float(a)) for a in out["initatt"][0]]
    cr, sr, cp, sp, cy, sy = (f(a / 2) for a in att for f in (mpmath.cos, mpmath.sin))
    q = [cy * cp * sr - sy * sp * cr, cy * sp * cr + sy * cp * sr, sy * cp * cr - cy * sp * sr, cy * cp * cr + sy * sp * sr]  # x y z w
    np.testing.assert_allclose(out["state17"][0, 4:8], [float(v) for v in q], rtol=0, atol=4e-16)
    x, y, z, w = q
    R = mpmath.matrix([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                       [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                       [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    p = mpmath.matrix(g["last_blh"]) - R * mpmath.matrix(g["antlever"])
    np.testing.assert_allclose(out["state17"][0, 1:4], [float(v) for v in p], rtol=0, atol=4e-16)
    np.testing.assert_array_equal(out["pose_prior"][0], out["state17"][0, 1:8])
    np.testing.assert_array_equal(out["mix_prior"][0], out["state17"][0, 8:17])
