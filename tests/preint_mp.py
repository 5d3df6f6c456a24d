"""A high-precision restatement of the IMU preintegration, and the sweep of intervals the edge tests run it on.

`preintegrate(state16, iewn, gravity, noise5, imu)` follows PreintegrationEarth (iewn given) and PreintegrationNormal (iewn None) as
geom_core.cuh documents them (IG/preintegration/preintegration_earth.cc:205-338, preintegration_normal.cc:195-232): compensationBias, dvfb
with the coning and sculling terms, the qnn / dnn Earth corrections, cbb0, phi = I + F dt, G = gt noise gt^T and
covariance = phi C phi^T + 0.5 dt (phi G + G phi^T).  It runs in mpmath at DPS digits from the doubles it is given, with dense phi, gt and
G (a product skips the zero factors it finds, which changes no value), the Normal form with its own gt (gt(3, 3) = R(dq), gt(6, 0) = +I)
rather than the Earth form's.  Nothing is shared with the product's arithmetic.  Results are rounded to doubles once, at the end, and
cached per interval: the sweep is a Python loop of a few milliseconds per sample.

`sweep()` is every edge interval; `mp_sweep()` the few dozen of them short enough for the restatement."""
from __future__ import annotations

import math

import mpmath
import numpy as np

from datagen import synth_ba

DPS = 40
WIE = synth_ba.WIE
D2R = synth_ba.D2R


# ---------------------------------------------------------------------------------------------- mp arithmetic (vectors are lists of 3 mpf)
def _add(a, b):
    return [a[i] + b[i] for i in range(3)]


def _sub(a, b):
    return [a[i] - b[i] for i in range(3)]


def _sc(s, a):
    return [s * a[i] for i in range(3)]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _mv(M, v):
    return [M[i][0] * v[0] + M[i][1] * v[1] + M[i][2] * v[2] for i in range(3)]


def _qmul(a, b):  # (w, x, y, z), Hamilton
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return (aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
            aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx)


def _qinv(q):  # conjugate / squared norm (Eigen's inverse())
    n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]
    return (q[0] / n2, -q[1] / n2, -q[2] / n2, -q[3] / n2)


def _qnorm(q):
    n = mpmath.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    return tuple(c / n for c in q)


def _qmat(q):  # Eigen's toRotationMatrix(), which does not normalise
    w, x, y, z = q
    return [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
            [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
            [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]


def _rv2q(rv):  # Rotation::rotvec2quaternion: angle |rv|, axis rv / |rv| (rv itself when the angle is 0)
    a = mpmath.sqrt(rv[0] * rv[0] + rv[1] * rv[1] + rv[2] * rv[2])
    ax = [c / a for c in rv] if a > 0 else rv
    s, c = mpmath.sin(a / 2), mpmath.cos(a / 2)
    return (c, s * ax[0], s * ax[1], s * ax[2])


def _skew(v):
    z = mpmath.mpf(0)
    return [[z, -v[2], v[1]], [v[2], z, -v[0]], [-v[1], v[0], z]]


def _m3mul(A, B):
    return [[A[i][0] * B[0][j] + A[i][1] * B[1][j] + A[i][2] * B[2][j] for j in range(3)] for i in range(3)]


def _mm(A, B):
    """dense A B; the zero entries of A's rows are skipped, which leaves every value as it is"""
    nb = len(B[0])
    out = []
    for row in A:
        nz = [(k, a) for k, a in enumerate(row) if a]
        out.append([mpmath.fsum(a * B[k][j] for k, a in nz) for j in range(nb)])
    return out


def _t(A):
    return [list(r) for r in zip(*A)]


def _put(M, r0, c0, m):
    for i in range(3):
        for j in range(3):
            M[r0 + i][c0 + j] = m[i][j]


# ---------------------------------------------------------------------------------------------- the restatement
def _preintegrate_mp(state16, iewn, gravity, noise5, imu):
    f = mpmath.mpf
    z, one = f(0), f(1)
    ident = [[one if i == j else z for j in range(3)] for i in range(3)]
    st = [f(float(x)) for x in state16]
    cur_p, cur_v, bg, ba = st[0:3], st[7:10], st[10:13], st[13:16]
    cur_q = (st[6], st[3], st[4], st[5])
    q0, dq = cur_q, (one, z, z, z)
    earth = iewn is not None
    iw = [f(float(x)) for x in iewn] if earth else [z, z, z]
    grav = [f(float(x)) for x in gravity]
    arw, vrw, gbs, abs_, corr = (f(float(x)) for x in noise5)
    noise = [arw * arw] * 3 + [vrw * vrw] * 3 + [2 * gbs * gbs / corr] * 3 + [2 * abs_ * abs_ / corr] * 3
    dp, dv, s1 = [z, z, z], [z, z, z], [z, z, z]
    delta_time, s0 = z, z
    J = [[one if i == j else z for j in range(15)] for i in range(15)]
    C = [[z] * 15 for _ in range(15)]
    rows = [[f(float(x)) for x in r] for r in np.asarray(imu, np.float64)]
    for s in range(1, len(rows)):
        pr, cu = rows[s - 1], rows[s]
        dt = cu[0]
        pth, pvl = _sub(pr[1:4], _sc(pr[0], bg)), _sub(pr[4:7], _sc(pr[0], ba))  # compensationBias
        cth, cvl = _sub(cu[1:4], _sc(dt, bg)), _sub(cu[4:7], _sc(dt, ba))
        delta_time += dt
        dvfb = _add(_add(cvl, _sc(f(0.5), _cross(cth, cvl))), _sc(one / 12, _add(_cross(pth, cvl), _cross(pvl, cth))))
        dtheta = _add(cth, _sc(one / 12, _cross(pth, cth)))
        phi = [[z] * 15 for _ in range(15)]
        gt = [[z] * 12 for _ in range(15)]
        if earth:
            dv_cor_g = _sc(dt, _sub(grav, _sc(f(2), _cross(iw, cur_v))))
            qnn = _rv2q(_sc(-dt, iw))
            half = [[(ident[i][j] + m) / 2 for j, m in enumerate(r)] for i, r in enumerate(_qmat(qnn))]
            dvel = _add(_mv(half, _mv(_qmat(cur_q), dvfb)), dv_cor_g)
            cur_p = _add(_add(cur_p, _sc(dt, cur_v)), _sc(dt / 2, dvel))
            cur_v = _add(cur_v, dvel)
            s0 += dt
            s1 = _add(s1, _sc(dt, cur_p))
            cur_q = _qnorm(_qmul(_qmul(qnn, cur_q), _rv2q(dtheta)))
            dnn = _sc(-(delta_time - dt / 2), iw)
            dvel = _mv(_qmat(_qmul(_qmul(_qmul(_qinv(q0), _rv2q(dnn)), q0), dq)), dvfb)
            dp = _add(_add(dp, _sc(dt, dv)), _sc(dt / 2, dvel))
            dv = _add(dv, dvel)
            dq = _qnorm(_qmul(dq, _rv2q(dtheta)))
            cbb0 = [[-m for m in r] for r in _qmat(_qmul(_qmul(_qmul(_qinv(q0), _rv2q(_sc(-delta_time, iw))), q0), dq))]
            _put(phi, 3, 6, _m3mul(cbb0, _skew(cvl)))
            _put(phi, 3, 12, [[dt * m for m in r] for r in cbb0])
            _put(gt, 3, 3, cbb0)
            _put(gt, 6, 0, [[-m for m in r] for r in ident])
        else:
            dvel = _add(_mv(_qmat(cur_q), dvfb), _sc(dt, grav))
            cur_p = _add(_add(cur_p, _sc(dt, cur_v)), _sc(dt / 2, dvel))
            cur_v = _add(cur_v, dvel)
            cur_q = _qnorm(_qmul(cur_q, _rv2q(dtheta)))
            dvel = _mv(_qmat(dq), dvfb)
            dp = _add(_add(dp, _sc(dt, dv)), _sc(dt / 2, dvel))
            dv = _add(dv, dvel)
            dq = _qnorm(_qmul(dq, _rv2q(dtheta)))
            Rdq = _qmat(dq)
            _put(phi, 3, 6, [[-m for m in r] for r in _m3mul(Rdq, _skew(cvl))])
            _put(phi, 3, 12, [[-dt * m for m in r] for r in Rdq])
            _put(gt, 3, 3, Rdq)
            _put(gt, 6, 0, ident)
        _put(phi, 0, 0, ident)
        _put(phi, 0, 3, [[dt * m for m in r] for r in ident])
        _put(phi, 3, 3, ident)
        _put(phi, 6, 6, [[ident[i][j] - m for j, m in enumerate(r)] for i, r in enumerate(_skew(cth))])
        _put(phi, 6, 9, [[-dt * m for m in r] for r in ident])
        _put(phi, 9, 9, [[(1 - dt / corr) * m for m in r] for r in ident])
        _put(phi, 12, 12, [[(1 - dt / corr) * m for m in r] for r in ident])
        _put(gt, 9, 6, ident)
        _put(gt, 12, 9, ident)
        J = _mm(phi, J)
        G = _mm([[g * noise[k] for k, g in enumerate(r)] for r in gt], _t(gt))
        phiT = _t(phi)
        PC, PG, GPt = _mm(phi, C), _mm(phi, G), _mm(G, phiT)
        PCPt = _mm(PC, phiT)
        C = [[PCPt[i][j] + dt / 2 * (PG[i][j] + GPt[i][j]) for j in range(15)] for i in range(15)]
    head = [delta_time, *dp, *dv, dq[1], dq[2], dq[3], dq[0], *bg, *ba, *grav, *iw, s0, *s1]
    end = [*cur_p, cur_q[1], cur_q[2], cur_q[3], cur_q[0], *cur_v]
    dbl = lambda xs: np.array([float(x) for x in xs], np.float64)
    return dbl(head), dbl(x for r in J for x in r).reshape(15, 15), dbl(x for r in C for x in r).reshape(15, 15), dbl(end)


_CACHE = {}


def preintegrate(state16, iewn, gravity, noise5, imu):
    """(head[27], J (15, 15), covariance (15, 15), end state[10]) of the interval, each entry the double nearest the DPS-digit value"""
    arrs = [np.ascontiguousarray(x, np.float64) for x in (state16, gravity, noise5, imu)]
    key = tuple(a.tobytes() for a in arrs) + (None if iewn is None else np.ascontiguousarray(iewn, np.float64).tobytes(),)
    if key not in _CACHE:
        with mpmath.workdps(DPS):
            _CACHE[key] = _preintegrate_mp(state16, iewn, gravity, noise5, imu)
    return _CACHE[key]


# ---------------------------------------------------------------------------------------------- the sweep
def iewn_at(lat_deg):
    lat = lat_deg * D2R
    return np.array([WIE * math.cos(lat), 0.0, -WIE * math.sin(lat)])


NOISE5_CORR100 = np.concatenate([synth_ba.NOISE5[:4], [100.0]])
ROWS = (1, 2, 3, 4, 33, 101, 201, 1001, 2001)
RATES = (100.0, 200.0, 400.0)
TIMINGS = ("uniform", "frac_ends", "repeat", "jitter")
MOTIONS = ("stationary", "line", "arc", "turn", "big_bias")
FORMS = ("earth30", "earth0", "earth80", "normal")
TURN_RATE = 180.0 * D2R                                  # rad/s
TURN_SPEED = 2.0 * 9.80665 / TURN_RATE                   # 2 g lateral acceleration on that turn
BIG_BG, BIG_BA = np.array([2.0, -3.0, 1.5]) * D2R, np.array([0.3, -0.5, 0.2])  # rad/s, m/s^2 in the start state


class Case:
    """one interval: the arguments of a preintegration call, and what it was made of"""

    def __init__(self, name, state16, iewn, noise5, imu, **tags):
        self.name, self.state16, self.iewn, self.noise5, self.imu, self.tags = name, state16, iewn, noise5, imu, tags
        self.gravity = synth_ba.GRAVITY

    @property
    def args(self):
        return self.state16, self.iewn, self.gravity, self.noise5, self.imu

    def __repr__(self):
        return self.name


def retime(imu, timing, rng):
    """the timestamp edges on rows from imu_samples: each row's dt and increments scaled together"""
    imu = imu.copy()
    n = len(imu)
    if timing == "frac_ends" and n >= 2:  # a short first and last sample, as interpolation at node times leaves them
        imu[1] *= 0.3
        if n >= 3:
            imu[-1] *= 0.7
    elif timing == "repeat" and n >= 3:   # one record repeated mid-interval: the same increments again, at the same time (dt = 0)
        imu[n // 2] = imu[n // 2 - 1]
        imu[n // 2, 0] = 0.0
    elif timing == "jitter":
        imu *= 1.0 + rng.uniform(-0.05, 0.05, (n, 1))
    return imu


def make_case(n, rate, timing, motion, form, noise, seed):
    rng = np.random.default_rng(seed)
    t0 = 0.37 * (seed % 7)
    kw = dict(line=dict(yaw_rate=0.0), arc=dict(), turn=dict(yaw_rate=TURN_RATE, speed=TURN_SPEED), big_bias=dict(),
              stationary=dict(yaw_rate=0.0, speed=0.0, heave=False, noise_scale=0.0))[motion]
    if motion == "stationary":
        form = "normal"  # zero rotation rate, zero bias, no noise, no Earth rate: every dtheta is exactly 0
    bg_t = np.zeros(3) if motion == "stationary" else rng.normal(0, 20.0 * D2R / 3600.0, 3)
    ba_t = np.zeros(3) if motion == "stationary" else rng.normal(0, 20.0 * 1e-5, 3)
    imu = synth_ba.imu_samples(t0, t0 + (n - 1) / rate, rate, rng, bg_t, ba_t, earth=form != "normal", **kw)
    assert len(imu) == n
    imu = retime(imu, timing, rng)
    p, v, _, psi = synth_ba.trajectory(t0, kw.get("speed", 5.0), kw.get("yaw_rate", 5.0 * D2R), kw.get("heave", True))
    bg, ba = (BIG_BG, BIG_BA) if motion == "big_bias" else (bg_t, ba_t)
    st = np.concatenate([p, synth_ba.q_yaw(psi), v, bg, ba])
    iewn = None if form == "normal" else iewn_at({"earth30": 30.5, "earth0": 0.0, "earth80": 80.0}[form])
    nz = NOISE5_CORR100 if noise else synth_ba.NOISE5
    name = f"{n}r-{int(rate)}hz-{timing}-{motion}-{form}" + ("-corr100" if noise else "")
    return Case(name, st, iewn, nz, imu, n=n, rate=rate, timing=timing, motion=motion, form=form, corr100=bool(noise))


def sweep():
    """every row count at every rate, each with every motion; the timing, form and noise cycle across them so that each appears with
    each row count"""
    out = []
    i = 0
    for n in ROWS:
        for r, rate in enumerate(RATES):
            for m, motion in enumerate(MOTIONS):
                out.append(make_case(n, rate, TIMINGS[(r + m) % 4], motion, FORMS[(i + m) % 4], (r + m + i) % 2, 1000 + len(out)))
            i += 1
    return out


def mp_sweep():
    """the cases short enough for the restatement: up to 101 rows, plus one of 201 rows in each form"""
    cases = [c for c in sweep() if c.tags["n"] <= 101]
    for form in FORMS:
        cases.append(make_case(201, 200.0, "jitter", "turn", form, form == "earth80", 5000 + FORMS.index(form)))
    return cases
