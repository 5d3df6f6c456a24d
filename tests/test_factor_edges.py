"""CPU: every window factor's residual and Jacobians, entry by entry, against a high-precision restatement (tests/factors_mp.py), at the
edges of the sweep there: td far from the per-feature td_i with zero and large pixel velocities, inverse depths 1e-4 and 2, an observing
depth of 1e-3 / 1e-6 m, the reference node first and last in the window, relative and extrinsic rotations at pi, quaternions a few ulp off
the unit sphere, states 6e6 m from the origin; IMU intervals of 4 rows, 0.5 s and 10 s in the Earth form at latitudes 0 / 30.5 / 80 deg and
the Normal form, with small and large bias deviations; GNSS with and without a lever arm and standard deviations 1e4 apart.

Bounds: each entry's error against the restatement must stay within c eps E, where E is the restatement's first-order (Wilkinson) running
bound for that entry (factors_mp.X).  For a whitened IMU entry the bound is c eps (sum_k |U_ik| (E_k + 16 |x_k|) + sum_{k >= i} ||U_:k|| |x_k|)
with x the unwhitened residual or Jacobian column: the rounding of the unwhitened entries, of the whitening sum, and of U itself, whose
double Gauss-Jordan inverse and Cholesky leave errors of the size of eps times U's column norms.  Worst ratios measured (error / (eps E))
over the sweep, for oracle/ba_ref.cpp and for the device evaluators (tests/test_factor_edges_gpu.py, H100 80GB HBM3), and the constants
chosen (about 10x the worst):
  reprojection        oracle: r 0.074, J_i 0.11, J_j 0.13, J_ext 0.30, J_rho 0.053, J_td 0.092;
                      device: quaternion form 0.39, frame form 0.25, icg_ba_residual_costs 0.52                   -> C_REPROJ = 3
  GNSS, pose prior,   oracle 0.25; device 0.79 (mix prior and ImuErrorFactor included), marginalization 0.033      -> C_SMALL = 8
  IMU                 oracle: r 0.61, J_pose0 0.96, J_mix0 0.69, J_pose1 2.5, J_mix1 2.5; device 2.5               -> C_IMU = 25
  with the loss       oracle per factor: reprojection 0.12, GNSS (knee points included) 0.61; per-factor costs without the loss:
                      oracle 0.026 / 0.50, device 0.027 / 0.52 (reprojection / GNSS); window initial cost, losses on and off:
                      oracle 0.011, device 0.0074
Entries whose bound is exactly zero (structural zeros, the copied 1 / std) must match exactly.

The restatement's analytic Jacobians are held to mpmath central differences through PoseParameterization::Plus wherever the reference's
Jacobian is exact: reprojection, GNSS, the pose prior, the mix prior, ImuErrorFactor, the marginalization factor's non-rotation columns, and
the IMU factor's unwhitened blocks except these first-order ones, checked only against the analytic restatement:
  IMU_INEXACT   attitude rows (6..8) x {pose0 rotation, pose1 rotation, mix0 gyro bias}; the marginalization factor's rotation columns are J0
                itself, the derivative only where dq is the identity."""
import mpmath
import numpy as np
import pytest

from tests import factors_mp as fm
from tests import oracle_api as oa

C_REPROJ, C_SMALL, C_IMU = 3.0, 8.0, 25.0
FD_DPS = 60
FRAME_GAP = {"+1": 0.0260, "+2": 0.0471, "+4": 0.0892, "-1": 0.0162, "-3": 0.0584}  # ulp per component: exact gap / (eps E)
IMU_INEXACT = [(slice(6, 9), slice(3, 6)), (slice(6, 9), slice(18, 21)), (slice(6, 9), slice(9, 12))]  # rows x columns of the local 15 x 30


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def prob(olib):
    return fm.window(lambda *a: oa.preintegrate(olib, *a), K=10, L=60, seed=11, with_priors=True)[0]


@pytest.fixture(autouse=True)
def _dps():
    with mpmath.workdps(fm.DPS):
        yield


def ratio(got, ref, c):
    """the worst |got - ref| / (eps E) of one block; entries with E = 0 must be equal"""
    v, e = fm.vals(ref) if not isinstance(ref, tuple) else ref
    got = np.asarray(got, float).reshape(v.shape)
    d = np.abs(got - v)
    assert not d[e == 0].any(), "an exact entry differs"
    return float((d[e > 0] / (fm.EPS * e[e > 0])).max()) if (e > 0).any() else 0.0


def check(got_r, got_J, ref_r, ref_J, c, what):
    ws = [ratio(got_r, ref_r, c)] + [ratio(g, r, c) for g, r in zip(got_J, ref_J)]
    assert max(ws) <= c, (what, ws)
    return ws


def reproj_ref(a):
    r, J, _ = fm.reprojection(fm.xs(a[0]), fm.xs(a[1]), fm.xs(a[2]), fm.X(a[3]), fm.X(a[4]), fm.xs(a[5]), fm.X(a[6]))
    return r, J


def imu_ref(blob, pn, p0, m0, p1, m1):
    """the whitened residual and global Jacobians with the whitening bound of the module docstring, as (values, E) pairs"""
    rw, Js, raw, Jraw, U = fm.imu(fm.xs(blob), [fm.xs(r) for r in pn], fm.xs(p0), fm.xs(m0), fm.xs(p1), fm.xs(m1))
    Uv = fm.vals(U)[0]
    A, u = np.abs(Uv), np.triu(np.tile(np.sqrt((Uv ** 2).sum(0)), (15, 1)))
    rv, re = fm.vals(raw)
    Jv, Je = fm.vals(Jraw)
    out_r = (fm.vals(rw)[0], A @ (re + 16 * np.abs(rv)) + u @ np.abs(rv))
    out_J = []
    for b, (c0, l, g) in enumerate(((0, 6, 7), (6, 9, 9), (15, 6, 7), (21, 9, 9))):
        e = np.zeros((15, g))
        e[:, :l] = A @ (Je[:, c0:c0 + l] + 16 * np.abs(Jv[:, c0:c0 + l])) + u @ np.abs(Jv[:, c0:c0 + l])
        out_J.append((fm.vals(Js[b])[0], e))
    return out_r, out_J


@pytest.fixture(scope="module")
def imu_points(olib):
    prep = lambda *a: oa.preintegrate(olib, *a)
    return [(why, fm.interval(prep, n, form, lat, far, db, seed=n + int(lat))) for why, n, form, lat, far, db in fm.IMU_POINTS]


# ---------------------------------------------------------------------------------------------- the oracle against the restatement
def test_reprojection(olib, prob):
    for p in fm.sweep_reprojection(prob):
        r, J = oa.reproj_eval(olib, *p.args)
        check(r, J, *reproj_ref(p.args), C_REPROJ, p)


def frame_gap(p):
    """the exact gap of the node-frame form's residual to the reference's, per entry, in units of eps E (the bound's scale)"""
    a = [fm.xs(x) if np.ndim(x) else fm.X(x) for x in p.args]
    rq, rf = fm.reprojection(*a)[0], fm.reprojection(*a, frames=True)[0]
    return max(float(abs(f.v - q.v) / (fm.EPS * q.e)) for f, q in zip(rf, rq))


def test_frame_form_gap_off_the_unit_sphere(prob):
    """The reference rotates by q^-1 = conj(q) / |q|^2, the frame form by R(q)^T: 2 (|q|^2 - 1) (R^T - I) v apart.  On the unit sphere
    (to DPS digits) the two functions agree; for the sweep's quaternions 1 to 4 ulp per component off it the exact gap is FRAME_GAP
    (units of eps E, worst over the residual entries): far below C_REPROJ, so the frame-form tests cannot tell node_frame from one that
    normalises the quaternion first.  Doubles that Plus normalised are themselves ~1 ulp off the sphere: the other sweep points show
    exact gaps of 2e-7 to 0.03."""
    for p in fm.sweep_reprojection(prob):
        g = frame_gap(p)
        if "ulp per component" in p.why:
            assert abs(g - FRAME_GAP[p.why.split()[3]]) <= 0.02 * g, (p, g)
        else:
            assert g <= 0.03, (p, g)


def test_gnss(olib, prob):
    for p in fm.sweep_gnss(prob):
        r, J = np.zeros(3), np.zeros((3, 7))
        a = [np.ascontiguousarray(x, float) for x in p.args]
        olib.icgo_gnss_eval(*[oa._p(x) for x in a], oa._p(r), oa._p(J))
        check(r, [J], *fm.gnss(*[fm.xs(x) for x in a]), C_SMALL, p)


def test_pose_prior(olib, prob):
    for p in fm.sweep_pose_prior(prob):
        r, J = np.zeros(6), np.zeros((6, 7))
        a = [np.ascontiguousarray(x, float) for x in p.args]
        olib.icgo_pose_prior_eval(*[oa._p(x) for x in a], oa._p(r), oa._p(J))
        check(r, [J], *fm.pose_prior(*[fm.xs(x) for x in a]), C_SMALL, p)


def test_imu(olib, imu_points):
    for why, (blob, pn, p0, m0, p1, m1) in imu_points:
        r, J = oa.imu_eval(olib, blob, pn, p0, m0, p1, m1)
        check(r, J, *imu_ref(blob, pn, p0, m0, p1, m1), C_IMU, why)


def test_three_row_interval_has_no_square_root_information(olib):
    """After 2 propagation steps the covariance is indefinite in exact arithmetic, so LLT(cov^-1) does not exist.  Shown on the
    preintegration restatement (tests/preint_mp.py): its covariance rounded to doubles has an eigenvalue below -eps ||C||_F, and rounding
    moves no eigenvalue by more than ||C - round(C)||_2 <= eps / 2 ||C||_F (Weyl), so the exact covariance has a negative one too.  One
    more row (4 rows) makes it positive definite.  The restatement's Cholesky refuses the product's 3-row blob."""
    from tests import preint_mp as pm
    for n, pd in ((3, False), (4, True)):
        _, _, Cv, _ = pm.preintegrate(*fm.interval(None, n, "earth", seed=n + 30))
        with mpmath.workdps(60):
            lam = min(mpmath.eigsy(mpmath.matrix(Cv.tolist()))[0])
        fro = float(np.sqrt((Cv ** 2).sum()))
        assert (lam > fm.EPS * fro) if pd else (lam < -2 * fm.EPS * fro), (n, float(lam), fro)
    blob, *_ = fm.interval(lambda *a: oa.preintegrate(olib, *a), 3, "earth", seed=33)
    with pytest.raises(ValueError, match="positive-definite"):
        fm.sqrt_information(blob[252:477])


def residual_cost_ratios(rc, gc, prob):
    """(worst reprojection, worst GNSS) ratio of per-factor costs 0.5 |r|^2 (no loss) to the restatement"""
    pose, fc = prob["pose"].reshape(-1, 7), prob["f_const"].reshape(-1, 14)
    wr = wg = 0.0
    for f in range(prob["F"]):
        a = (pose[prob["f_ref"][f]], pose[prob["f_obs"][f]], prob["ext"][:7], prob["invdepth"][prob["f_lm"][f]], prob["ext"][7], fc[f], prob["reproj_std"])
        wr = max(wr, ratio([rc[f]], [fm.apply_loss(reproj_ref(a)[0], [], False)[2]], 0))
    for g in range(prob["n_gnss"]):
        nd = int(prob["gnss_node"][g])
        r, _ = fm.gnss(fm.xs(pose[nd]), fm.xs(prob["gnss_blh"][3 * g:3 * g + 3]), fm.xs(prob["gnss_std"][3 * g:3 * g + 3]), fm.xs(prob["lever"]))
        wg = max(wg, ratio([gc[g]], [fm.apply_loss(r, [], False)[2]], 0))
    return wr, wg


def test_residual_costs(olib, prob):
    """icgo_ba_residual_costs (EvaluateResidualBlock without the loss, ic_gvins.cc:1251,1278) per factor of a whole window"""
    wr, wg = residual_cost_ratios(*oa.ba_residual_costs(olib, prob), prob)
    assert wr <= C_REPROJ and wg <= C_SMALL, (wr, wg)


# ---------------------------------------------------------------------------------------------- the loss the solver applies
def loss_ref(r, J, huber):
    rc, Jc, cost = fm.apply_loss(r, J, huber)
    return rc, Jc, cost


def test_huber_per_factor(olib, prob):
    """evaluate_block's loss (icgo_*_eval_loss) against the restated HuberLoss + Corrector, with the loss on and off: GNSS at a squared
    norm of exactly 1, one ulp either side, 0 and 1e6; the GNSS sweep; reprojection factors rescaled to the knee, below and far above it"""
    for p in fm.sweep_gnss_knee():
        if p.target is not None:
            r = np.asarray(p.args[0][:3])
            assert r[0] * r[0] + r[1] * r[1] + r[2] * r[2] == p.target, p  # the product's own sum lands on the knee point
    for p in fm.sweep_gnss_knee() + fm.sweep_gnss(prob):
        for hub in (0, 1):
            r, J, cost = oa.gnss_eval_loss(olib, *p.args, hub)
            rr, JJ = fm.gnss(*[fm.xs(x) for x in p.args])
            rc, Jc, cc = loss_ref(rr, JJ, hub)
            check(r, [J], rc, Jc, C_SMALL, (p, hub))
            assert ratio([cost], [cc], C_SMALL) <= C_SMALL, (p, hub)
    for p in fm.huber_reprojection_points(prob):
        for hub in (0, 1):
            r, J, cost = oa.reproj_eval_loss(olib, *p.args, hub)
            rc, Jc, cc = loss_ref(*reproj_ref(p.args), hub)
            check(r, J, rc, Jc, C_REPROJ, (p, hub))
            assert ratio([cost], [cc], C_REPROJ) <= C_REPROJ, (p, hub)


def window_cost(prob):
    """the window's total cost as the solver's initial cost sums it (ic_gvins.cc's factors: GNSS, IMU, ImuErrorFactor, the priors and the
    reprojection factors, each with its loss), restated, with its bound"""
    pose, mix = prob["pose"].reshape(-1, 7), prob["mix"].reshape(-1, 9)
    fc, off, pn = prob["f_const"].reshape(-1, 14), prob["pn_off"], prob["pn"].reshape(-1, 4)
    terms = []
    for g in range(prob["n_gnss"]):
        nd = int(prob["gnss_node"][g])
        r, J = fm.gnss(fm.xs(pose[nd]), fm.xs(prob["gnss_blh"][3 * g:3 * g + 3]), fm.xs(prob["gnss_std"][3 * g:3 * g + 3]), fm.xs(prob["lever"]))
        terms.append(fm.apply_loss(r, J, prob["gnss_huber"])[2])
    for k in range(prob["n_imu"]):
        (v, e), _ = imu_ref(prob["imu_blob"][480 * k:480 * (k + 1)], pn[off[k]:off[k + 1]], pose[k], mix[k], pose[k + 1], mix[k + 1])
        terms.append(fm.apply_loss([fm.X(a, b) for a, b in zip(v, e)], [], False)[2])
    if prob["has_imu_error"]:
        terms.append(fm.apply_loss(fm.imu_error(fm.xs(mix[prob["n_imu"]]))[0], [], False)[2])
    if prob["has_pose_prior"]:
        terms.append(fm.apply_loss(fm.pose_prior(fm.xs(pose[0]), fm.xs(prob["pose_prior"]), fm.xs(prob["pose_prior_std"]))[0], [], False)[2])
    if prob["has_mix_prior"]:
        terms.append(fm.apply_loss(fm.mix_prior(fm.xs(mix[0]), fm.xs(prob["mix_prior"]), fm.xs(prob["mix_prior_std"]))[0], [], False)[2])
    for f in range(prob["F"]):
        a = (pose[prob["f_ref"][f]], pose[prob["f_obs"][f]], prob["ext"][:7], prob["invdepth"][prob["f_lm"][f]], prob["ext"][7], fc[f], prob["reproj_std"])
        terms.append(fm.apply_loss(reproj_ref(a)[0], [], prob["reproj_huber"])[2])
    return sum(terms[1:], terms[0])


HUBER_WINDOWS = [(1, 1), (1, 0), (0, 1), (0, 0)]  # (reproj_huber, gnss_huber)


def huber_window(prob, reproj_huber, gnss_huber):
    """the sweep window with the loss flags set; its GNSS std is tripled so that its fixes sit on both sides of the knee (|r|^2 from 0.13
    to 3.6)"""
    import copy
    p = copy.deepcopy(prob)
    p["reproj_huber"], p["gnss_huber"] = reproj_huber, gnss_huber
    p["gnss_std"] = p["gnss_std"] * 3.0
    return p


def test_huber_through_the_window_cost(olib, prob):
    """the oracle's initial cost (evaluate_all over evaluate_block) against the restated total, with each loss on and off"""
    p = huber_window(prob, 1, 1)
    pose = p["pose"].reshape(-1, 7)
    sq = [float(sum(x.v ** 2 for x in fm.gnss(fm.xs(pose[int(p["gnss_node"][g])]), fm.xs(p["gnss_blh"][3 * g:3 * g + 3]),
                                                 fm.xs(p["gnss_std"][3 * g:3 * g + 3]), fm.xs(p["lever"]))[0])) for g in range(p["n_gnss"])]
    assert min(sq) < 1 < max(sq), sq
    for flags in HUBER_WINDOWS:
        p = huber_window(prob, *flags)
        ref = window_cost(p)
        s = oa.ba_solve(olib, p, 1)
        assert abs(s["initial_cost"] - float(ref.v)) <= C_SMALL * fm.EPS * float(ref.e), (flags, s["initial_cost"], float(ref.v))


# ---------------------------------------------------------------------------------------------- the restatement's Jacobians
# Evaluated at points whose quaternions are normalised in DPS digits: the reference's analytic Jacobians assume a unit quaternion (q^-1 v
# = R(q)^T v), and a double quaternion's |q|^2 - 1 of ~1e-16 moves the true derivative by that much relative.
def unit(x):
    x = [mpmath.mpf(v) for v in x]
    n = mpmath.sqrt(x[3] ** 2 + x[4] ** 2 + x[5] ** 2 + x[6] ** 2)
    return x[:3] + [v / n for v in x[3:7]]


def mp_of(J):
    return [[v.v for v in r] for r in J]


def fd_close(Jfd, Jan, what):
    """central differences against the analytic formula, both in FD_DPS digits: they agree to ~1e-24 relative when the formula is the
    derivative, a wrong entry is off by O(1)"""
    for rf, ra in zip(Jfd, Jan):
        tol = mpmath.mpf("1e-20") * max(max(abs(v) for v in ra), 1)
        assert all(abs(f - a) <= tol for f, a in zip(rf, ra)), (what, [float(f - a) for f, a in zip(rf, ra)])


@pytest.fixture
def fd_dps():
    """60 digits: the differences cancel intermediates up to 1e8 times the residual (positions 6e6 m from the origin over a 0.05 m std),
    which at 40 digits would leave 1e-40 1e8 / H ~ 1e-17 in the quotient"""
    with mpmath.workdps(FD_DPS):
        yield


def T(cols):
    return [list(r) for r in zip(*cols)]


def test_reprojection_jacobians_are_derivatives(prob, fd_dps):
    fun = fm.values_of(fm.reprojection)
    for p in fm.sweep_reprojection(prob)[::3]:
        a = [unit(x) if i < 3 else (list(map(mpmath.mpf, x)) if np.ndim(x) else mpmath.mpf(x)) for i, x in enumerate(p.args)]
        _, J, _ = fm.reprojection(*[[fm.X(c) for c in x] if isinstance(x, list) else fm.X(x) for x in a])
        for w in range(3):
            g = lambda x, w=w: fun(*[x if i == w else a[i] for i in range(7)])
            fd_close(T([fm.central_pose(g, a[w], k) for k in range(6)]), [r[:6] for r in mp_of(J[w])], (p, w))
            assert all(r[6].v == 0 for r in J[w])
        for w in (3, 4):
            g = lambda x, w=w: fun(*[x[0] if i == w else a[i] for i in range(7)])
            fd_close(T([fm.central_vec(g, [a[w]], 0)]), mp_of(J[w]), (p, w))


def test_small_factor_jacobians_are_derivatives(prob, fd_dps):
    for f, pts in ((fm.gnss, fm.sweep_gnss(prob)), (fm.pose_prior, fm.sweep_pose_prior(prob))):
        fun = fm.values_of(f)
        for p in pts:
            a = [unit(p.args[0])] + [list(map(mpmath.mpf, x)) for x in p.args[1:]]
            J = f(*[[fm.X(c) for c in x] for x in a])[1][0]
            g = lambda x: fun(x, *a[1:])
            fd_close(T([fm.central_pose(g, a[0], k) for k in range(6)]), [r[:6] for r in mp_of(J)], p)
    for p in fm.sweep_mix(prob):
        a = [list(map(mpmath.mpf, x)) for x in p.args]
        for f, args in ((fm.mix_prior, a), (fm.imu_error, a[:1])):
            fun = fm.values_of(f)
            J = f(*[[fm.X(c) for c in x] for x in args])[1][0]
            g = lambda x, f=f, args=args: fun(x, *args[1:])
            fd_close(T([fm.central_vec(g, args[0], k) for k in range(9)]), mp_of(J), p)


def test_marginalization_jacobians_and_sign_fix(prob, fd_dps):
    rng = np.random.default_rng(5)
    pts = fm.sweep_marginalization(prob, rng)
    types, params, x0, J0, e0 = pts[0].args
    X0, XJ, Xe = fm.xs(x0), [fm.xs(r) for r in J0], fm.xs(e0)
    r, Js = fm.marginalization(types, [fm.xs(p) for p in params], X0, XJ, Xe)
    col = 0
    for b, (t, p) in enumerate(zip(types, params)):
        l = {0: 6, 1: 9, 2: 6, 3: 1}[int(t)]
        g = lambda x, b=b: [v.v for v in fm.marginalization(types, [[fm.X(c) for c in x] if i == b else fm.xs(q) for i, q in enumerate(params)],
                                                           X0, XJ, Xe)[0]]
        xm = list(map(mpmath.mpf, p))
        cols = range(3) if l == 6 else range(l)  # rotation columns: J0, not the derivative away from dq = identity (module docstring)
        Jfd = T([fm.central_pose(g, xm, k) if l == 6 else fm.central_vec(g, xm, k) for k in cols])
        fd_close(Jfd, [[mpmath.mpf(J0[i, col + k]) for k in cols] for i in range(len(e0))], (t, b))
        assert np.array_equal(fm.vals(Js[b])[0][:, :l], J0[:, col:col + l])
        col += l
    for p in pts[1:]:  # the dq.w edges: the sign fix flips 2 vec(dq) only for a negative w
        types, params, x0, J0, e0 = p.args
        dx = fm.vals(fm.marginalization(types, [fm.xs(q) for q in params], fm.xs(x0), [fm.xs(np.eye(len(e0))[i]) for i in range(len(e0))],
                                        fm.xs(np.zeros(len(e0))))[0])[0]
        sign = -1.0 if p.dqw < 0 else 1.0
        assert np.array_equal(dx[3:6], sign * 2.0 * np.asarray(params[0][3:6])), p


def test_imu_jacobians_are_derivatives(olib, imu_points, fd_dps):
    """the unwhitened local 15 x 30 Jacobian against central differences of the unwhitened residual, except IMU_INEXACT"""
    for why, (blob, pn, p0, m0, p1, m1) in imu_points[:6]:
        st = [list(map(mpmath.mpf, x)) for x in (p0, m0, p1, m1)]
        B, P = fm.xs(blob), [fm.xs(r) for r in pn]
        U = [[fm.X(1 if i == j else 0) for j in range(15)] for i in range(15)]

        def raw(which, x):
            args = [[fm.X(c) for c in (x if i == which else st[i])] for i in range(4)]
            return [v.v for v in fm.imu(B, P, *args, U=U)[2]]

        Jan = fm.vals(fm.imu(B, P, *[fm.xs(x) for x in (p0, m0, p1, m1)], U=U)[3])[0]
        cols = []
        for which, c0, l in ((0, 0, 6), (1, 6, 9), (2, 15, 6), (3, 21, 9)):
            f = lambda x, which=which: raw(which, x)
            cols += [fm.central_pose(f, st[which], k) if l == 6 else fm.central_vec(f, st[which], k) for k in range(l)]
        Jfd = np.array([[float(v) for v in c] for c in cols]).T
        mask = np.ones((15, 30), bool)
        for rs, cs in IMU_INEXACT:
            mask[rs, cs] = False
        sc = np.maximum(np.abs(Jan).max(axis=1, keepdims=True), 1.0)
        bad = (np.abs(Jfd - Jan) > 1e-15 * sc) & mask
        assert not bad.any(), (why, np.argwhere(bad))
        # the first-order blocks differ from the derivative by O(|attitude residual|), not by a wrong formula
        for rs, cs in IMU_INEXACT:
            assert np.abs(Jfd[rs, cs] - Jan[rs, cs]).max() <= 0.05 * np.abs(Jan[rs, cs]).max() + 1e-12, (why, rs, cs)


def test_the_sweep_reaches_every_edge(prob):
    whys = " | ".join(p.why for p in fm.sweep_reprojection(prob))
    for key in ("zero pixel velocities", "~2 normalised", "td = td_1", "1e-4", "inverse depth 2", "first window node", "last window node",
                "depth 0.001", "depth 1e-06", "relative attitude pi", "extrinsic rotation", "ulp per component", "6e6 m"):
        assert key in whys, key
    assert any(p.args[3][:3].any() == False for p in fm.sweep_gnss(prob))  # noqa: E712  (a zero lever arm)
    signs = [np.copysign(1.0, p.dqw) for p in fm.sweep_marginalization(prob, np.random.default_rng(5))[1:]]
    assert signs == [1.0, -1.0, 1.0, -1.0]
    assert {n for _, n, *_ in fm.IMU_POINTS} >= {4, 101, 2001} and {f for _, _, f, *_ in fm.IMU_POINTS} == {"earth", "normal"}
