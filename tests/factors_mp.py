"""A high-precision restatement of the window factors' Evaluate, each result with a first-order rounding bound, and the edge sweep the factor
tests run it on.

Written from the reference formulas (IG/ = ic_gvins/ic_gvins/): ReprojectionFactor (factors/reprojection_factor.h:55-147), GnssFactor
(gnss_factor.h:43-71), ImuPosePriorFactor (preintegration/imu_pose_prior_factor.h:42-68), ImuMixPriorFactor (imu_mix_prior_factor.h:40-75),
ImuErrorFactor (imu_error_factor.h:45-91), MarginalizationFactor (factors/marginalization_factor.h:47-101) and PreintegrationEarth /
PreintegrationNormal::evaluate + residualJacobianPose0/Mix0/Pose1/Mix1 (preintegration_earth.cc:37-164, preintegration_normal.cc:38-142).
The quaternion operations are the reference's own: inverse() is the conjugate over the squared norm, q * v is Eigen's _transformVector and
toRotationMatrix does not normalise, so a quaternion a few ulp off the unit sphere is evaluated as the reference evaluates it.  The IMU
whitening U = LLT(cov^-1).matrixL()^T is formed here from the blob's covariance.

Every value is an `X`: the DPS-digit value and a first-order (Wilkinson) running bound on the error a double evaluation of the same
operations makes, in units of eps = 2^-53.  Inputs are exact doubles (error 0); each +, -, *, / and sqrt adds |result| to the propagated
error, sin / cos add 2 |result| (one libm ulp).  A product that evaluates a different but equal expression (the row-by-row Jacobians of
ba_math.cuh, one reciprocal in place of several divisions) makes errors of the same order, which the tests' constant c covers.

`sweep_*()` build the edge points from datagen/synth_ba plus hand-made geometry; each point carries a `why`."""
from __future__ import annotations

import math

import mpmath
import numpy as np

from datagen import synth_ba

DPS = 40
EPS = 2.0 ** -53
mpf = mpmath.mpf


class X:
    """a DPS-digit value v with a first-order bound e (units of eps) on the error of its double evaluation"""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0):
        self.v, self.e = mpf(v), mpf(e)

    def __add__(s, o):
        o = _x(o)
        v = s.v + o.v
        return X(v, s.e + o.e + abs(v))

    __radd__ = __add__

    def __sub__(s, o):
        o = _x(o)
        v = s.v - o.v
        return X(v, s.e + o.e + abs(v))

    def __rsub__(s, o):
        return _x(o) - s

    def __mul__(s, o):
        o = _x(o)
        v = s.v * o.v
        return X(v, abs(o.v) * s.e + abs(s.v) * o.e + abs(v))

    __rmul__ = __mul__

    def __truediv__(s, o):
        o = _x(o)
        v = s.v / o.v
        return X(v, (s.e + abs(v) * o.e) / abs(o.v) + abs(v))

    def __rtruediv__(s, o):
        return _x(o) / s

    def __neg__(s):
        return X(-s.v, s.e)


def _x(a):
    return a if isinstance(a, X) else X(a)


def xsqrt(a):
    v = mpmath.sqrt(a.v)
    return X(v, (a.e / (2 * v) if v else 0) + abs(v))


def xsin(a):
    v = mpmath.sin(a.v)
    return X(v, abs(mpmath.cos(a.v)) * a.e + 2 * abs(v))


def xcos(a):
    v = mpmath.cos(a.v)
    return X(v, abs(mpmath.sin(a.v)) * a.e + 2 * abs(v))


def xs(arr):
    return [X(float(a)) for a in np.asarray(arr, np.float64).ravel()]


def vals(xl):
    """(values as doubles, bounds in units of eps) of a nested list of X"""
    a = np.array(xl, dtype=object)
    return np.vectorize(lambda x: float(x.v))(a).astype(np.float64), np.vectorize(lambda x: float(x.e))(a).astype(np.float64)


# ---------------------------------------------------------------------------------------------- vectors, matrices and quaternions of X
def add(a, b):
    return [a[i] + b[i] for i in range(len(a))]


def sub(a, b):
    return [a[i] - b[i] for i in range(len(a))]


def sc(s, a):
    return [s * x for x in a]


def cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def mv(M, v):
    return [M[i][0] * v[0] + M[i][1] * v[1] + M[i][2] * v[2] for i in range(len(M))]


def mm(A, B):
    return [[sum((A[i][k] * B[k][j] for k in range(1, len(B))), A[i][0] * B[0][j]) for j in range(len(B[0]))] for i in range(len(A))]


def tr(A):
    return [list(r) for r in zip(*A)]


def madd(A, B, s=1):
    return [[A[i][j] + s * B[i][j] for j in range(len(A[0]))] for i in range(len(A))]


def msc(s, A):
    return [[s * a for a in r] for r in A]


def skew(v):
    z = X(0)
    return [[z, -v[2], v[1]], [v[2], z, -v[0]], [-v[1], v[0], z]]


def ident(n=3):
    return [[X(1 if i == j else 0) for j in range(n)] for i in range(n)]


def qmul(a, b):  # (w, x, y, z), Hamilton
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return (aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
            aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx)


def qinv(q):  # Eigen inverse(): conjugate / squared norm
    n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]
    return (q[0] / n2, -q[1] / n2, -q[2] / n2, -q[3] / n2)


def qrot(q, v):  # Eigen q * v (_transformVector)
    uv = cross(q[1:], v)
    uv = add(uv, uv)
    return add(add(v, sc(q[0], uv)), cross(q[1:], uv))


def qmat(q):  # Eigen toRotationMatrix(), which does not normalise
    w, x, y, z = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz, txx, txy, txz, tyy, tyz, tzz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x, ty * y, tz * y, tz * z
    return [[1 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1 - (txx + tzz), tyz - twx], [txz - twy, tyz + twx, 1 - (txx + tyy)]]


def rv2q(rv):  # Rotation::rotvec2quaternion (rotation.h:72-76); Eigen's normalized() leaves a zero vector as it is
    a = xsqrt(rv[0] * rv[0] + rv[1] * rv[1] + rv[2] * rv[2])
    ax = [c / a for c in rv] if a.v > 0 else rv
    h = a * mpf(0.5)
    s = xsin(h)
    return (xcos(h), s * ax[0], s * ax[1], s * ax[2])


def qleft_br(q):  # Rotation::quaternionleft(q).bottomRightCorner<3, 3>() (rotation.h:103-110)
    return madd(msc(q[0], ident()), skew(q[1:]))


def qright_br(q):  # Rotation::quaternionright(q).bottomRightCorner<3, 3>() (rotation.h:112-119)
    return madd(msc(q[0], ident()), skew(q[1:]), -1)


def lr_br(a, b):  # (quaternionleft(a) quaternionright(b)).bottomRightCorner<3, 3>(): -a_v b_v^T + L_br(a) R_br(b)
    lr = mm(qleft_br(a), qright_br(b))
    return [[lr[i][j] - a[1 + i] * b[1 + j] for j in range(3)] for i in range(3)]


def pose_pq(x):
    return list(x[:3]), (x[6], x[3], x[4], x[5])


def pose_plus(x, d):
    """PoseParameterization::Plus (pose_parameterization.h:34-49) on plain mpf lists: p + dp, (q * rotvec2quaternion(dq)).normalized()"""
    q = (x[6], x[3], x[4], x[5])
    a = mpmath.sqrt(d[3] ** 2 + d[4] ** 2 + d[5] ** 2)
    ax = [c / a for c in d[3:6]] if a > 0 else d[3:6]
    s = mpmath.sin(a / 2)
    w, qx, qy, qz = (c.v for c in qmul(tuple(X(c) for c in q), (X(mpmath.cos(a / 2)), X(s * ax[0]), X(s * ax[1]), X(s * ax[2]))))
    n = mpmath.sqrt(w * w + qx * qx + qy * qy + qz * qz)
    return [x[0] + d[0], x[1] + d[1], x[2] + d[2], qx / n, qy / n, qz / n, w / n]


def _block(J, c0, M):
    for i in range(len(M)):
        for j in range(len(M[0])):
            J[i][c0 + j] = M[i][j]


def zeros(r, c):
    return [[X(0) for _ in range(c)] for _ in range(r)]


# ---------------------------------------------------------------------------------------------- the factors
def reprojection(pose0, pose1, ext, rho, td, c, std, frames=False):
    """ReprojectionFactor::Evaluate: r[2] and the global Jacobians [2x7, 2x7, 2x7, 2x1, 2x1] as the reference forms them (matrix products
    with reduce = sqrt_info [1/d 0 -x/d^2; 0 1/d -y/d^2]).  frames=True: the node-frame form's function instead (every rotation by
    toRotationMatrix(q), each inverse by its transpose), which off the unit sphere differs from the reference's"""
    p0, q0 = pose_pq(pose0)
    p1, q1 = pose_pq(pose1)
    tic, qic = pose_pq(ext)
    pts0, pts1, vel0, vel1, td0, td1 = c[0:3], c[3:6], c[6:9], c[9:12], c[12], c[13]
    pts_0_td = sub(pts0, sc(td - td0, vel0))
    pts_1_td = sub(pts1, sc(td - td1, vel1))
    pts_c_0 = [x / rho for x in pts_0_td]
    pts_b_0 = add(qrot(qic, pts_c_0), tic)
    pts_n = add(qrot(q0, pts_b_0), p0)
    if frames:
        pts_b_1 = mv(tr(qmat(q1)), sub(pts_n, p1))
        pts_1 = mv(tr(qmat(qic)), sub(pts_b_1, tic))
    else:
        pts_b_1 = qrot(qinv(q1), sub(pts_n, p1))
        pts_1 = qrot(qinv(qic), sub(pts_b_1, tic))
    d1 = pts_1[2]
    si = 1 / std
    r = [si * (pts_1[0] / d1 - pts_1_td[0]), si * (pts_1[1] / d1 - pts_1_td[1])]
    cb0n, cnb1, cbc = qmat(q0), tr(qmat(q1)), tr(qmat(qic))
    red = msc(si, [[1 / d1, X(0), -pts_1[0] / (d1 * d1)], [X(0), 1 / d1, -pts_1[1] / (d1 * d1)]])
    cc = mm(cbc, cnb1)
    tmp_r = mm(mm(cc, cb0n), tr(cbc))
    J = [zeros(2, 7) for _ in range(3)]
    _block(J[0], 0, mm(red, cc))
    _block(J[0], 3, mm(red, msc(-1, mm(mm(cc, cb0n), skew(pts_b_0)))))
    _block(J[1], 0, mm(red, msc(-1, cc)))
    _block(J[1], 3, mm(red, mm(cbc, skew(pts_b_1))))
    _block(J[2], 0, mm(red, mm(cbc, madd(mm(cnb1, cb0n), ident(), -1))))
    lever = sub(mv(cnb1, sub(add(mv(cb0n, tic), p0), p1)), tic)
    rot = madd(madd(msc(-1, mm(tmp_r, skew(pts_c_0))), skew(mv(tmp_r, pts_c_0))), skew(mv(cbc, lever)))
    _block(J[2], 3, mm(red, rot))
    jr = mv(red, mv(tmp_r, pts_0_td))
    jt = mv(red, mv(tmp_r, vel0))
    J.append([[-(jr[i] / (rho * rho))] for i in range(2)])
    J.append([[-(jt[i] / rho) + si * vel1[i]] for i in range(2)])
    return r, J, pts_1


def gnss(pose, blh, std3, lever):
    p, q = pose_pq(pose)
    R = qmat(q)
    e = sub(add(p, mv(R, lever)), blh)
    si = [1 / s for s in std3]
    r = [si[i] * e[i] for i in range(3)]
    J = zeros(3, 7)
    b = msc(-1, mm(R, skew(lever)))
    for i in range(3):
        J[i][i] = si[i] * X(1)
        for j in range(3):
            J[i][3 + j] = si[i] * b[i][j]
    return r, [J]


def pose_prior(pose, prior7, std6):
    si = [1 / s for s in std6]
    r = [si[k] * (pose[k] - prior7[k]) for k in range(3)]
    dq = qmul(qinv(pose_pq(pose)[1]), pose_pq(prior7)[1])
    r += [si[3 + k] * (2 * dq[1 + k]) for k in range(3)]
    J = zeros(6, 7)
    b = msc(-1, qright_br(dq))
    for i in range(3):
        J[i][i] = si[i] * X(1)
        for j in range(3):
            J[3 + i][3 + j] = si[3 + i] * b[i][j]
    return r, [J]


def mix_prior(mix, prior9, std9):
    J = zeros(9, 9)
    for k in range(9):
        J[k][k] = 1 / std9[k]
    return [(mix[k] - prior9[k]) / std9[k] for k in range(9)], [J]


GB_STD, AB_STD = 7200 / 3600.0 * math.pi / 180.0, 2.0e4 * 1.0e-5  # imu_error_factor.h, as doubles


def imu_error(mix):
    J = zeros(6, 9)
    for k in range(3):
        J[k][3 + k], J[3 + k][6 + k] = 1 / X(GB_STD), 1 / X(AB_STD)
    return [mix[3 + k] / X(GB_STD) for k in range(3)] + [mix[6 + k] / X(AB_STD) for k in range(3)], [J]


def marginalization(block_type, params, x0, J0, e0):
    """e = e0 + J0 dx; a pose block's dx is (p - p0, 2 vec(q0^-1 q)), negated when dq.w < 0 (an exact zero, of either sign, is not
    negative: the restatement has no signed zero, and Eigen's dq.w() < 0 is false for -0.0).  J = the block's columns of J0."""
    gs, ls = {0: 7, 1: 9, 2: 7, 3: 1}, {0: 6, 1: 9, 2: 6, 3: 1}
    rr = len(e0)
    dx, xo = [], 0
    for t, x in zip(block_type, params):
        g = gs[int(t)]
        xl = x0[xo:xo + g]
        if g == 7:
            dq = qmul(qinv(pose_pq(xl)[1]), pose_pq(x)[1])
            a = [2 * v for v in dq[1:]]
            if dq[0].v < 0:
                a = [-v for v in a]
            dx += sub(x[:3], xl[:3]) + a
        else:
            dx += sub(x, xl)
        xo += g
    r = [sum((J0[i][k] * dx[k] for k in range(1, rr)), J0[i][0] * dx[0]) + e0[i] for i in range(rr)]
    Js, col = [], 0
    for t in block_type:
        g, l = gs[int(t)], ls[int(t)]
        Js.append([[J0[i][col + c] if c < l else X(0) for c in range(g)] for i in range(rr)])
        col += l
    return r, Js


def sqrt_information(cov):
    """U = LLT(cov^-1).matrixL()^T in DPS digits (the bounds of U are not tracked: each U_ij enters the tests' bound with the error a
    double Gauss-Jordan inverse and Cholesky leave, measured against this U, see test_factor_edges.IMU_U_REL)"""
    with mpmath.workdps(DPS + 20):
        A = mpmath.matrix([[mpf(float(v)) for v in row] for row in np.asarray(cov, np.float64).reshape(15, 15)])
        Ai = A ** -1
        Ai = (Ai + Ai.T) / 2
        L = mpmath.cholesky(Ai)
        return [[X(L[j, i]) if j >= i else X(0) for j in range(15)] for i in range(15)]


def imu(blob, pn, pose0, mix0, pose1, mix1, U=None):
    """the IMU factor: (whitened r[15], whitened global Jacobians [15x7, 15x9, 15x7, 15x9], raw r, raw local 15x30 J).  pn: the
    (dt, pn[3]) rows of PreintegrationEarth::evaluate's position-compensation loop (empty in the Normal form)."""
    b = blob
    normal = float(b[477].v) != 0.0
    p0, q0 = pose_pq(pose0)
    p1, q1 = pose_pq(pose1)
    v0, bg0, ba0, v1, bg1, ba1 = mix0[0:3], mix0[3:6], mix0[6:9], mix1[0:3], mix1[3:6], mix1[6:9]
    Jc = [b[27 + 15 * i:27 + 15 * i + 15] for i in range(15)]
    blk = lambda r0, c0: [[Jc[r0 + i][c0 + j] for j in range(3)] for i in range(3)]
    dp_dbg, dp_dba, dv_dbg, dv_dba, dq_dbg = blk(0, 9), blk(0, 12), blk(3, 9), blk(3, 12), blk(6, 9)
    dbg, dba = sub(bg0, b[11:14]), sub(ba0, b[14:17])
    grav, iewn, dt = b[17:20], b[20:23], b[0]
    dq = (b[10], b[7], b[8], b[9])
    corrected_p = add(add(b[1:4], mv(dp_dba, dba)), mv(dp_dbg, dbg))
    corrected_v = add(add(b[4:7], mv(dv_dba, dba)), mv(dv_dbg, dbg))
    corrected_q = qmul(dq, rv2q(mv(dq_dbg, dbg)))
    qnb0 = qinv(q0)
    cnb0 = qmat(qnb0)
    half_g_dt2 = sc(mpf(0.5), sc(dt, sc(dt, grav)))
    if normal:
        dpn = sub(sub(sub(p1, p0), sc(dt, v0)), half_g_dt2)
        dvn = sub(sub(v1, v0), sc(dt, grav))
        rp, rv = sub(qrot(qnb0, dpn), corrected_p), sub(qrot(qnb0, dvn), corrected_v)
        rq = [2 * c for c in qmul(qmul(qinv(corrected_q), qnb0), q1)[1:]]
    else:
        isk = skew(iewn)
        # p_cor = 2 iewn_skew sum_i (pn_i - p0) dt_i (:55-59); the product sums it as S1 - p0 S0 from the blob, whose rounding (each of the
        # n sums of S0 / S1 and the cancellation against p0 S0) is added to the bound
        acc = [X(0)] * 3
        for row in pn:
            acc = add(acc, sc(row[0], sub(row[1:4], p0)))
        n = max(1, len(pn))
        acc = [X(a.v, a.e + n * (abs(b[24 + k].v) + abs(p0[k].v) * abs(b[23].v))) for k, a in enumerate(acc)]
        p_cor = sc(2, mv(isk, acc))
        v_cor = sc(2, mv(isk, sub(p1, p0)))
        qnn = rv2q([-(dt * w) for w in iewn])
        dpn = add(sub(sub(sub(p1, p0), sc(dt, v0)), half_g_dt2), p_cor)
        dvn = add(sub(sub(v1, v0), sc(dt, grav)), v_cor)
        qb0b1 = qmul(qmul(qinv(q1), qnn), q0)
        rp, rv = sub(mv(cnb0, dpn), corrected_p), sub(mv(cnb0, dvn), corrected_v)
        rq = [2 * c for c in qmul(qb0b1, corrected_q)[1:]]
    raw = rp + rv + rq + sub(bg1, bg0) + sub(ba1, ba0)
    J = zeros(15, 30)
    neg = lambda M: msc(-1, M)
    I3 = ident()

    def _block3(r0, c0, M):
        for i in range(3):
            for j in range(3):
                J[r0 + i][c0 + j] = M[i][j]

    if normal:  # preintegration_normal.cc:77-140
        q10 = qmul(qinv(q1), q0)
        _block3(0, 0, neg(cnb0))
        _block3(0, 3, skew(qrot(qnb0, dpn)))
        _block3(3, 3, skew(qrot(qnb0, dvn)))
        _block3(6, 3, neg(lr_br(q10, corrected_q)))
        _block3(0, 6, neg(msc(dt, cnb0)))
        _block3(6, 9, neg(mm(qleft_br(qmul(q10, dq)), dq_dbg)))
        _block3(0, 15, cnb0)
        _block3(6, 18, qleft_br(qmul(qmul(qinv(corrected_q), qnb0), q1)))
    else:  # preintegration_earth.cc:92-164
        ci = mm(cnb0, isk)
        _block3(0, 0, madd(neg(cnb0), msc(2 * dt, ci), -1))
        _block3(0, 3, skew(mv(cnb0, dpn)))
        _block3(3, 0, msc(-2, ci))
        _block3(3, 3, skew(mv(cnb0, dvn)))
        _block3(6, 3, lr_br(qb0b1, corrected_q))
        _block3(0, 6, neg(msc(dt, cnb0)))
        _block3(6, 9, mm(qleft_br(qmul(qb0b1, dq)), dq_dbg))
        _block3(0, 15, cnb0)
        _block3(3, 15, msc(2, ci))
        _block3(6, 18, neg(qright_br(qmul(qb0b1, corrected_q))))
    _block3(0, 9, neg(dp_dbg))
    _block3(0, 12, neg(dp_dba))
    _block3(3, 6, neg(cnb0))
    _block3(3, 9, neg(dv_dbg))
    _block3(3, 12, neg(dv_dba))
    _block3(9, 9, neg(I3))
    _block3(12, 12, neg(I3))
    _block3(3, 21, cnb0)
    _block3(9, 24, I3)
    _block3(12, 27, I3)
    if U is None:
        U = sqrt_information([float(c.v) for c in b[252:477]])
    rw = [sum((U[i][k] * raw[k] for k in range(i + 1, 15)), U[i][i] * raw[i]) for i in range(15)]
    Jw = [[sum((U[i][k] * J[k][c] for k in range(i + 1, 15)), U[i][i] * J[i][c]) for c in range(30)] for i in range(15)]
    Js = []
    for c0, l, g in ((0, 6, 7), (6, 9, 9), (15, 6, 7), (21, 9, 9)):
        Js.append([[Jw[i][c0 + c] if c < l else X(0) for c in range(g)] for i in range(15)])
    return rw, Js, raw, J, U


def apply_loss(r, Js, huber):
    """the loss as the solver applies it to one residual block (Ceres: HuberLoss(1.0)::Evaluate, loss_function.cc, and the Corrector,
    corrector.cc; the reference's own copy IG/factors/residual_block_info.h:59-87).  huber False: cost = 0.5 |r|^2, r and J unchanged.
    Otherwise rho = (s, 1, 0) for s = |r|^2 <= 1 and (2 sqrt(s) - 1, 1 / sqrt(s), -rho' / (2 s)) above; cost = 0.5 rho; with rho'' <= 0
    (always, for Huber) or s = 0 the residuals and Jacobians scale by sqrt(rho'), else alpha = 1 - sqrt(1 + 2 s rho'' / rho'),
    r *= sqrt(rho') / (1 - alpha) and J = sqrt(rho') (J - alpha / s r r^T J).  The branch is taken on the DPS-digit s: one ulp from the
    knee a double evaluation may take the other one, which moves no value by more than an ulp (Huber is C^1 there)."""
    sq = sum((x * x for x in r[1:]), r[0] * r[0])
    if not huber:
        return r, Js, X(0.5) * sq
    if sq.v > 1:
        rt = xsqrt(sq)
        rho = (2 * rt - 1, 1 / rt)
        rho = rho + (-(rho[1] / (2 * sq)),)
    else:
        rho = (sq, X(1), X(0))
    cost = X(0.5) * rho[0]
    s1 = xsqrt(rho[1])
    if sq.v == 0 or rho[2].v <= 0:
        return [s1 * x for x in r], [[[s1 * v for v in row] for row in J] for J in Js], cost
    alpha = 1 - xsqrt(1 + 2 * sq * rho[2] / rho[1])
    a = alpha / sq
    out = []
    for J in Js:
        rtj = [sum((r[k] * J[k][c] for k in range(1, len(r))), r[0] * J[0][c]) for c in range(len(J[0]))]
        out.append([[s1 * (J[k][c] - a * r[k] * rtj[c]) for c in range(len(J[0]))] for k in range(len(r))])
    return [s1 / (1 - alpha) * x for x in r], out, cost


# ---------------------------------------------------------------------------------------------- central differences in DPS digits
H = mpf("1e-15")


def central_pose(fun, x, k):
    """d fun / d delta_k through PoseParameterization::Plus, at step H (truncation ~ H^2, cancellation ~ 10^-DPS / H: both < 1e-24)"""
    d = [mpf(0)] * 6
    d[k] = H
    fp = fun(pose_plus(x, d))
    d[k] = -H
    fm = fun(pose_plus(x, d))
    return [(a - b) / (2 * H) for a, b in zip(fp, fm)]


def central_vec(fun, x, k):
    xp, xm = list(x), list(x)
    xp[k] += H
    xm[k] -= H
    return [(a - b) / (2 * H) for a, b in zip(fun(xp), fun(xm))]


def values_of(f):
    """wrap a restatement taking X arguments into a function of plain mpf lists returning the residual values"""
    def g(*args):
        return [r.v for r in f(*[[X(a) for a in arg] if isinstance(arg, list) else X(arg) for arg in args])[0]]
    return g


# ---------------------------------------------------------------------------------------------- the edge sweep
class Point:
    def __init__(self, why, **kw):
        self.why = why
        self.__dict__.update(kw)

    def __repr__(self):
        return self.why


def _qaxis(axis, ang):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    return np.concatenate([math.sin(ang / 2) * a, [math.cos(ang / 2)]])


def _place_observer(pose0, ext, c, rho, q1, target):
    """the observer position p1 that puts the landmark of factor constants c at camera coordinates `target` of a body with attitude q1"""
    Rbc, R0 = synth_ba.q_mat(ext[3:7]), synth_ba.q_mat(pose0[3:7])
    pts_c_0 = (c[0:3] - (0.0 - c[12]) * c[6:9]) / rho
    pn = R0 @ (Rbc @ pts_c_0 + ext[:3]) + pose0[:3]
    return pn - synth_ba.q_mat(q1) @ (Rbc @ np.asarray(target, float) + ext[:3])


def _off_unit(q, k):
    """q with every component moved k ulp outward (k > 0) or inward: |q|^2 about 2 k ulp from 1"""
    return np.array([np.nextafter(v, math.copysign(np.inf, v) * np.sign(k)) if k else v for v in q]) if abs(k) == 1 else \
        _off_unit(_off_unit(q, int(np.sign(k))), k - int(np.sign(k)))


def window(preintegrate, **kw):
    return synth_ba.make_window(preintegrate, **kw)


def sweep_reprojection(prob):
    """(pose0, pose1, ext, rho, td, c14, std) points from one synthetic window plus hand-made geometry"""
    pose = prob["pose"].reshape(-1, 7)
    ext, std = prob["ext"][:7].copy(), prob["reproj_std"]
    fc = prob["f_const"].reshape(-1, 14)
    pts = []

    def add_pt(why, i, j, c, rho, td=None, e=None, p0=None, p1=None):
        pts.append(Point(why, args=(pose[i].copy() if p0 is None else p0, pose[j].copy() if p1 is None else p1, ext.copy() if e is None else e,
                                    float(rho), float(prob["ext"][7] if td is None else td), np.asarray(c, float).copy(), std)))

    for f in (0, 3, 50, 111, prob["F"] - 1):
        add_pt(f"synthetic factor {f}: ordinary depth, td = the window's td, td_i = 0", prob["f_ref"][f], prob["f_obs"][f], fc[f],
               prob["invdepth"][prob["f_lm"][f]])
    f = 7
    i, j, rho = prob["f_ref"][f], prob["f_obs"][f], prob["invdepth"][prob["f_lm"][f]]
    c = fc[f].copy()
    c[12], c[13] = -0.031, 0.017
    cz = c.copy()
    cz[6:12] = 0.0
    add_pt("td 0.05 s from distinct td_0 / td_1, zero pixel velocities (the td terms vanish)", i, j, cz, rho, td=0.05)
    cv = c.copy()
    cv[6:9], cv[9:12] = [1.7, -0.9, 0.0], [-1.3, 2.1, 0.0]
    add_pt("td 0.05 s from distinct td_0 / td_1, pixel velocities ~2 normalised units / s", i, j, cv, rho, td=0.05)
    add_pt("the same with td = td_1 exactly (only the td_0 term moves pts_0)", i, j, cv, rho, td=c[13])
    add_pt("inverse depth 1e-4: a landmark 10 km away", i, j, fc[f], 1e-4)
    add_pt("inverse depth 2: a landmark 0.5 m away", i, j, fc[f], 2.0)
    K = prob["K"]
    add_pt("reference node = the first window node, observer = the last", 0, K - 1, fc[f], rho)
    add_pt("reference node = the last window node, observer = the first", K - 1, 0, fc[f], rho)
    for z in (1e-3, 1e-6):
        p1 = pose[j].copy()
        p1[:3] = _place_observer(pose[i], ext, fc[f], rho, pose[j][3:7], [0.4 * z, -0.2 * z, z])
        add_pt(f"observing depth {z:g} m: the projection divides by a near-zero depth", i, j, fc[f], rho, p1=p1)
    for ang, why in ((math.pi - 1e-6, "pi - 1e-6"), (math.pi, "pi (w = cos(pi / 2) ~ 6e-17)")):
        q1 = synth_ba.q_mul(pose[i][3:7], _qaxis([0.3, -0.8, 0.5], ang))
        p1 = np.concatenate([_place_observer(pose[i], ext, fc[f], rho, q1, [0.1, -0.05, 8.0]), q1])
        add_pt(f"relative attitude {why} about a skew axis", i, j, fc[f], rho, p1=p1)
    for ang in (math.pi - 1e-7, math.pi):
        e = ext.copy()
        e[3:7] = _qaxis([1.0, 1.0, 0.2], ang)
        add_pt(f"extrinsic rotation {ang:.9f} rad (near pi)", i, j, fc[f], rho, e=e)
    for k in (1, 2, 4, -1, -3):
        q0, q1, qe = (_off_unit(x[3:7], k) for x in (pose[i], pose[j], ext))
        add_pt(f"all three quaternions {k:+d} ulp per component off the unit sphere", i, j, fc[f], rho,
               p0=np.concatenate([pose[i][:3], q0]), p1=np.concatenate([pose[j][:3], q1]), e=np.concatenate([ext[:3], qe]))
    far = np.array([3.2e6, -4.1e6, 2.5e6])
    add_pt("both poses 6e6 m from the origin (ECEF-sized positions)", i, j, fc[f], rho,
           p0=np.concatenate([pose[i][:3] + far, pose[i][3:7]]), p1=np.concatenate([pose[j][:3] + far, pose[j][3:7]]))
    return pts


def sweep_gnss(prob):
    pose = prob["pose"].reshape(-1, 7)
    lever = np.asarray(prob["lever"], float)
    pts = []
    for g in range(prob["n_gnss"]):
        nd = int(prob["gnss_node"][g])
        blh, sd = prob["gnss_blh"][3 * g:3 * g + 3].copy(), prob["gnss_std"][3 * g:3 * g + 3].copy()
        pts.append(Point(f"synthetic fix {g}, the antenna lever arm", args=(pose[nd].copy(), blh, sd, lever.copy())))
    nd, blh = int(prob["gnss_node"][1]), prob["gnss_blh"][3:6].copy()
    pts.append(Point("zero lever arm: the rotation Jacobian block is exactly zero", args=(pose[nd].copy(), blh, np.array([0.05, 0.05, 0.1]), np.zeros(3))))
    pts.append(Point("standard deviations 1e-3 / 10 / 1e-3 m (1e4 apart)", args=(pose[nd].copy(), blh, np.array([1e-3, 10.0, 1e-3]), lever.copy())))
    p = pose[nd].copy()
    p[3:7] = _qaxis([0.2, 0.9, -0.4], math.pi - 1e-8)
    pts.append(Point("attitude near pi, a 2 m lever arm", args=(p, blh, np.array([0.05, 0.05, 0.1]), np.array([1.5, -1.2, 0.4]))))
    far = pose[nd].copy()
    far[:3] += [3.2e6, -4.1e6, 2.5e6]
    pts.append(Point("a pose and fix 6e6 m from the origin", args=(far, blh + [3.2e6, -4.1e6, 2.5e6], np.array([0.05, 0.05, 0.1]), lever.copy())))
    return pts


KNEE_SQ = {"exactly 1": 1.0, "one ulp above 1": float(np.nextafter(1.0, 2.0)), "one ulp below 1": float(np.nextafter(1.0, 0.0))}


def sweep_gnss_knee():
    """GNSS factors whose squared residual norm, as the product sums it (r0 r0 + r1 r1 + r2 r2 in doubles), is exactly 1, one ulp above and
    one ulp below: the identity attitude, a zero lever arm, blh = 0 and std = 1, so r = p exactly; plus r = 0 (the corrector's s = 0 branch)
    and |r|^2 = 0.25, 2 and 1e6 (below, above and far above the knee)"""
    pts = []
    for why, e in (("exactly 1", (1.0, 0.0, 0.0)), ("one ulp above 1", (1.0, 2.0 ** -26, 0.0)),
                   ("one ulp below 1", (1.0 - 2.0 ** -52, math.sqrt(2.0 ** -53 * 3), 0.0)),
                   ("zero", (0.0, 0.0, 0.0)), ("0.25 (below)", (0.5, 0.0, 0.0)), ("2 (above)", (1.0, 1.0, 0.0)),
                   ("1e6 (far above)", (600.0, 800.0, 0.0))):
        pose = np.array([e[0], e[1], e[2], 0.0, 0.0, 0.0, 1.0])
        pts.append(Point(f"squared norm {why}", args=(pose, np.zeros(3), np.ones(3), np.zeros(3)), target=KNEE_SQ.get(why)))
    return pts


def huber_reprojection_points(prob):
    """synthetic factors whose std is rescaled so that |r|^2 sits within a few ulp of the knee, at 1e-2 and at 1e4 of it"""
    pts = []
    for p in sweep_reprojection(prob)[:5]:
        r = reprojection(*[xs(a) if np.ndim(a) else X(a) for a in p.args])[0]
        n = float(mpmath.sqrt(r[0].v ** 2 + r[1].v ** 2)) * p.args[6]  # |r| at std = 1
        for k, why in ((1.0, "at the knee"), (10.0, "|r|^2 = 1e-2"), (0.01, "|r|^2 = 1e4")):
            a = list(p.args)
            a[6] = n * k
            pts.append(Point(f"{p.why[:20]}, std rescaled: {why}", args=tuple(a)))
    return pts


def sweep_pose_prior(prob):
    pose = prob["pose"].reshape(-1, 7)
    prior, sd = np.asarray(prob["pose_prior"], float), np.asarray(prob["pose_prior_std"], float)
    pts = [Point("the first window's prior", args=(pose[0].copy(), prior.copy(), sd.copy())),
           Point("standard deviations 1e4 apart across axes", args=(pose[0].copy(), prior.copy(), np.array([1e-3, 10.0, 0.1, 1e-6, 1e-2, 1e-4])))]
    p = pose[0].copy()
    p[3:7] = synth_ba.q_mul(prior[3:7], _qaxis([0.5, 0.5, -0.7], math.pi - 1e-6))
    pts.append(Point("pose rotated by pi - 1e-6 from the prior (dq.w ~ 5e-7)", args=(p, prior.copy(), sd.copy())))
    p = pose[0].copy()
    p[3:7] = _off_unit(p[3:7], 3)
    pts.append(Point("pose quaternion 3 ulp per component off the unit sphere", args=(p, prior.copy(), sd.copy())))
    return pts


def sweep_mix(prob):
    mix = prob["mix"].reshape(-1, 9)
    sd = np.asarray(prob["mix_prior_std"], float)
    return [Point("the first window's mix prior", args=(mix[0].copy(), np.asarray(prob["mix_prior"], float).copy(), sd.copy())),
            Point("standard deviations 1e-6 .. 1e2", args=(mix[0].copy(), np.asarray(prob["mix_prior"], float).copy(), np.logspace(-6, 2, 9)))]


def sweep_marginalization(prob, rng):
    """every block type mixed in one factor, and pose blocks whose dq.w is +0, -0 and one ulp either side of 0"""
    pose, mix = prob["pose"].reshape(-1, 7), prob["mix"].reshape(-1, 9)
    types = np.array([0, 1, 0, 1, 2, 3], np.int32)
    ext = prob["ext"]
    base = [pose[0].copy(), mix[0].copy(), pose[1].copy(), mix[1].copy(), ext[:7].copy(), ext[7:8].copy()]
    x0 = np.concatenate([b + (rng.normal(0, 1e-3, b.shape) if len(b) != 7 else 0) for b in base])
    for o in (0, 16):
        x0[o + 3:o + 7] = synth_ba.q_mul(base[0 if o == 0 else 2][3:7], synth_ba.q_from_rotvec(rng.normal(0, 1e-3, 3)))
    r = 6 + 9 + 6 + 9 + 6 + 1
    J0 = np.triu(rng.normal(0, 1, (r, r))) * np.concatenate([[10.0] * 6, [5.0] * 9, [10.0] * 6, [5.0] * 9, [50.0] * 6, [100.0]])[None, :]
    e0 = rng.normal(0, 0.1, r)
    pts = [Point("every block type (pose, mix, pose, mix, extrinsic, td) in one factor", args=(types, [b.copy() for b in base], x0, J0, e0))]
    # x0 of block 0 = the identity attitude: dq = q itself, so dq.w is q.w as given
    x0i = x0.copy()
    x0i[3:7] = [0.0, 0.0, 0.0, 1.0]
    tiny = 5e-324
    for w, xyz, why in ((0.0, (1.0, 0.0, 0.0), "dq.w = +0 exactly (a half turn): no sign fix"),
                        (-0.0, (-1.0, -0.0, -0.0), "dq.w = -0.0 exactly: -0.0 < 0 is false, no sign fix"),
                        (tiny, (0.6, 0.8, 0.0), "dq.w one denormal ulp above 0: no sign fix"),
                        (-tiny, (0.6, 0.8, 0.0), "dq.w one denormal ulp below 0: the sign fix flips 2 vec(dq)")):
        p = [b.copy() for b in base]
        p[0][3:7] = [xyz[0], xyz[1], xyz[2], w]
        pts.append(Point(why, args=(types, p, x0i.copy(), J0, e0), dqw=w))
    return pts


def interval(preintegrate, n, form, lat_deg=30.5, far=False, dbias=1.0, seed=0):
    """one IMU factor: n rows at 200 Hz, its blob and pn, and the two states it connects (perturbed like a solve's iterate).  dbias
    scales the bias deviation from the linearisation point; far moves both states 6e6 m from the origin.  preintegrate None returns the
    preintegration's arguments (state16, iewn, gravity, noise5, imu) instead."""
    rng = np.random.default_rng(seed)
    earth = form == "earth"
    t0, t1 = 0.4, 0.4 + (n - 1) / 200.0
    bg_t, ba_t = rng.normal(0, 20.0 * synth_ba.D2R / 3600.0, 3), rng.normal(0, 2e-4, 3)
    imu = synth_ba.imu_samples(t0, t1, 200.0, rng, bg_t, ba_t, earth=earth)
    p, v, _, psi = synth_ba.trajectory(t0)
    p1, v1, _, psi1 = synth_ba.trajectory(t1)
    off = np.array([3.2e6, -4.1e6, 2.5e6]) if far else np.zeros(3)
    st = np.concatenate([p + off, synth_ba.q_yaw(psi), v, bg_t, ba_t])
    lat = lat_deg * synth_ba.D2R
    iewn = np.array([synth_ba.WIE * math.cos(lat), 0.0, -synth_ba.WIE * math.sin(lat)]) if earth else None
    if preintegrate is None:
        return st, iewn, synth_ba.GRAVITY, synth_ba.NOISE5, imu
    blob, pn, _ = preintegrate(st, iewn, synth_ba.GRAVITY, synth_ba.NOISE5, imu)
    pose0 = np.concatenate([p + off + rng.normal(0, 0.05, 3), synth_ba.q_mul(synth_ba.q_yaw(psi), synth_ba.q_from_rotvec(rng.normal(0, 0.005, 3)))])
    pose1 = np.concatenate([p1 + off + rng.normal(0, 0.05, 3), synth_ba.q_mul(synth_ba.q_yaw(psi1), synth_ba.q_from_rotvec(rng.normal(0, 0.005, 3)))])
    dev = dbias * np.concatenate([rng.normal(0, 5.0 * synth_ba.D2R / 3600.0, 3), rng.normal(0, 5e-5, 3)])
    mix0 = np.concatenate([v + rng.normal(0, 0.05, 3), bg_t + dev[:3], ba_t + dev[3:]])
    mix1 = np.concatenate([v1 + rng.normal(0, 0.05, 3), bg_t + dev[:3] * 0.9, ba_t + dev[3:] * 1.1])
    return blob, pn, pose0, mix0, pose1, mix1


IMU_POINTS = [  # (why, n, form, lat, far, dbias)
    ("4 rows, Earth form at 30.5 deg: the shortest interval whose covariance is positive definite (after 3 rows it is indefinite in exact"
     " arithmetic, so LLT(cov^-1) does not exist: the restatement's Cholesky and icg_ba_imu_evaluate both refuse it)", 4, "earth", 30.5,
     False, 1.0),
    ("the 0.5 s default, Earth form at latitude 0", 101, "earth", 0.0, False, 1.0),
    ("the 0.5 s default, Earth form at latitude 80 deg", 101, "earth", 80.0, False, 1.0),
    ("the 0.5 s default, Normal form", 101, "normal", 0.0, False, 1.0),
    ("10 s (2001 rows), Earth form at 30.5 deg", 2001, "earth", 30.5, False, 1.0),
    ("10 s, Normal form", 2001, "normal", 0.0, False, 1.0),
    ("bias deviations 1e-3 of the default (small)", 101, "earth", 30.5, False, 1e-3),
    ("bias deviations 100x the default (large: dq_dbg dbg ~ 0.01 rad)", 101, "earth", 30.5, False, 100.0),
    ("states 6e6 m from the origin, Earth form", 101, "earth", 30.5, True, 1.0),
    ("states 6e6 m from the origin, Normal form", 101, "normal", 0.0, True, 1.0),
]
