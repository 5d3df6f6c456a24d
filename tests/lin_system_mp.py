"""A high-precision assembly of a window's normal equations and reduced camera system, each entry with a first-order rounding bound: the
reference the linearisation read-out (WindowSolver.peek_linearization) is held to, entry by entry.

Built on tests/factors_mp.py.  Every factor is evaluated there in DPS digits with its Wilkinson bound, the loss applied by fm.apply_loss,
and the result rounded to doubles: the factor's whitened, loss-corrected local Jacobian and residual in the window's column layout
[pose 6K | extrinsic 6 | td 1 | mix 9K], plus j_rho for a reprojection factor.  A factor's bound is its restatement bound times the
constant the factor tests hold the device evaluators to (C_REPROJ, C_IMU, C_SMALL of tests/test_factor_edges.py), plus one unit for the
rounding to doubles.

The sums are exactly rounded sums of error-free products: every product a b is split into p + e exactly (Dekker's TwoProduct) and the
terms are summed by Ogita-Rump-Oishi's Sum2, as if in twice the working precision and then rounded.  So the reference carries no error
beyond the rounding of its factor values, which the bounds include.

Bounds, in units of eps = 2^-53, of an entry S = sum_k a_k b_k (a Gram entry, a J^T r entry, a Schur term with a = phi_l w_l):
    E(S) = sum_k (|a_k| E(b_k) + |b_k| E(a_k)) + m sum_k |a_k b_k|,
the propagated factor bounds plus gamma_m for a sum of m terms in any order.  m counts every rounding the kernel's sum can make: the
products, the partial sums of ba_lin_vis's runs, the gather over pairs, the cluster split of ba_schur_dmma.  phi_l = s_l^2 / (s_l^2 h_l +
D_l^2) is evaluated in factors_mp.X arithmetic from h_l and its bound.  An entry passes when |device - reference| <= C eps E with one C
per kernel (C_LIN_VIS, C_LIN_CAM, C_SCHUR); entries whose bound is exactly zero must match exactly."""
from __future__ import annotations

import math

import mpmath
import numpy as np

from tests import factors_mp as fm
from tests.test_factor_edges import C_IMU, C_REPROJ, C_SMALL, imu_ref

C_LIN_VIS, C_LIN_CAM, C_SCHUR = 1.0, 1.0, 1.0
EPS = fm.EPS
MIN_DIAG, MAX_DIAG = 1e-6, 1e32  # LevenbergMarquardtStrategy's clamp of the LM diagonal (ba_lm.cuh lm_d2)


# ---------------------------------------------------------------------------------------------- exact sums of exact products
def two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = 134217729.0 * a  # 2^27 + 1
    h = c - (c - a)
    return h, a - h


def two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


class Sum2:
    """elementwise Sum2 over added arrays (and error-free products)"""

    def __init__(self, shape):
        self.s, self.c = np.zeros(shape), np.zeros(shape)

    def add(self, x):
        self.s, e = two_sum(self.s, x)
        self.c += e

    def add_prod(self, a, b):
        p, e = two_prod(a, b)
        self.add(p)
        self.c += e

    def value(self):
        return self.s + self.c


def gram(V, E, m):
    """(V^T V exactly rounded, its bound) for rows V (n x c) with bounds E (units of eps); m: the roundings the kernel's sum may make"""
    n, c = V.shape
    acc = Sum2((c, c))
    for k in range(n):
        acc.add_prod(V[k][:, None], V[k][None, :])
    A = np.abs(V)
    return acc.value(), A.T @ E + E.T @ A + m * (A.T @ A)


# ---------------------------------------------------------------------------------------------- the factors
def _ve(xl, c):
    """values and bounds of a nested list of X: the restatement bound times c, plus the rounding to doubles"""
    v, e = fm.vals(xl)
    return v, c * e + np.abs(v)


class VisFactor:
    """one reprojection factor: rows X = [J_ref pose 6 | J_obs pose 6 | J_ext 6 | J_td | r] (2 x 20) and j_rho (2), loss applied"""

    def __init__(self, f, l, ref, obs, X, XE, jr, jrE, cost, costE, sq):
        self.f, self.l, self.ref, self.obs = f, l, ref, obs
        self.X, self.XE, self.jr, self.jrE, self.cost, self.costE, self.sq = X, XE, jr, jrE, cost, costE, sq


class CamFactor:
    """one camera-only factor: its columns of the window, local Jacobian (m x n) and residual (m), with bounds"""

    def __init__(self, kind, cols, J, JE, r, rE):
        self.kind, self.cols, self.J, self.JE, self.r, self.rE = kind, np.asarray(cols), J, JE, r, rE


_CACHE: dict = {}


def _reproj_x(args, huber):
    """(r, [Ji, Jj, Je, Jrho, Jtd], cost, |r|^2) of one factor with its loss, in X; memoised on the arguments' bytes"""
    key = (b"".join(np.ascontiguousarray(a, float).tobytes() for a in args), huber)
    if key not in _CACHE:
        with mpmath.workdps(fm.DPS):
            r, J, _ = fm.reprojection(fm.xs(args[0]), fm.xs(args[1]), fm.xs(args[2]), fm.X(args[3]), fm.X(args[4]), fm.xs(args[5]), fm.X(args[6]))
            sq = float(sum(x.v * x.v for x in r))
            rc, Jc, cost = fm.apply_loss(r, J, huber)
        _CACHE[key] = (rc, Jc, cost, sq)
    return _CACHE[key]


def vis_factor(prob, f, huber=None):
    pose, fc = prob["pose"].reshape(-1, 7), prob["f_const"].reshape(-1, 14)
    i, j, l = int(prob["f_ref"][f]), int(prob["f_obs"][f]), int(prob["f_lm"][f])
    args = (pose[i], pose[j], prob["ext"][:7], prob["invdepth"][l], prob["ext"][7], fc[f], prob["reproj_std"])
    rc, Jc, cost, sq = _reproj_x(args, bool(prob["reproj_huber"] if huber is None else huber))
    X, XE = np.zeros((2, 20)), np.zeros((2, 20))
    for b, c0 in ((0, 0), (1, 6), (2, 12)):
        v, e = _ve([row[:6] for row in Jc[b]], C_REPROJ)
        if b == 2 and prob["ext_const"]:
            v, e = 0 * v, 0 * e
        X[:, c0:c0 + 6], XE[:, c0:c0 + 6] = v, e
    v, e = _ve(Jc[4], C_REPROJ)
    if not prob["td_const"]:
        X[:, 18:19], XE[:, 18:19] = v, e
    X[:, 19], XE[:, 19] = _ve(rc, C_REPROJ)
    jr, jrE = _ve(Jc[3], C_REPROJ)
    cv, ce = _ve([cost], C_REPROJ)
    return VisFactor(f, l, i, j, X, XE, jr[:, 0], jrE[:, 0], cv[0], ce[0], sq)


def cam_factors(prob):
    """every camera-only factor of the window: IMU, GNSS, ImuErrorFactor, the pose and mix priors, the marginalization prior"""
    K = prob["K"]
    pose, mix = prob["pose"].reshape(-1, 7), prob["mix"].reshape(-1, 9)
    cp = lambda k: list(range(6 * k, 6 * k + 6))
    cm = lambda k: list(range(6 * K + 7 + 9 * k, 6 * K + 16 + 9 * k))
    out = []
    with mpmath.workdps(fm.DPS):
        off, pn = prob["pn_off"], prob["pn"].reshape(-1, 4)
        for k in range(prob["n_imu"]):
            (rv, re), Js = imu_ref(prob["imu_blob"][480 * k:480 * (k + 1)], pn[off[k]:off[k + 1]], pose[k], mix[k], pose[k + 1], mix[k + 1])
            J = np.concatenate([Js[0][0][:, :6], Js[1][0], Js[2][0][:, :6], Js[3][0]], axis=1)
            JE = np.concatenate([Js[0][1][:, :6], Js[1][1], Js[2][1][:, :6], Js[3][1]], axis=1)
            out.append(CamFactor(f"imu {k}", cp(k) + cm(k) + cp(k + 1) + cm(k + 1), J, C_IMU * JE + np.abs(J), rv, C_IMU * re + np.abs(rv)))
        for g in range(prob["n_gnss"]):
            nd = int(prob["gnss_node"][g])
            r, J = fm.gnss(fm.xs(pose[nd]), fm.xs(prob["gnss_blh"][3 * g:3 * g + 3]), fm.xs(prob["gnss_std"][3 * g:3 * g + 3]), fm.xs(prob["lever"]))
            r, J, _ = fm.apply_loss(r, J, bool(prob["gnss_huber"]))
            out.append(_cam(f"gnss {g}", cp(nd), [row[:6] for row in J[0]], r, C_SMALL))
        if prob["has_imu_error"]:
            r, J = fm.imu_error(fm.xs(mix[prob["n_imu"]]))
            out.append(_cam("imu error", cm(prob["n_imu"]), J[0], r, C_SMALL))
        if prob["has_pose_prior"]:
            r, J = fm.pose_prior(fm.xs(pose[0]), fm.xs(prob["pose_prior"]), fm.xs(prob["pose_prior_std"]))
            out.append(_cam("pose prior", cp(0), [row[:6] for row in J[0]], r, C_SMALL))
        if prob["has_mix_prior"]:
            r, J = fm.mix_prior(fm.xs(mix[0]), fm.xs(prob["mix_prior"]), fm.xs(prob["mix_prior_std"]))
            out.append(_cam("mix prior", cm(0), J[0], r, C_SMALL))
        if prob["marg_r"] > 0:
            out.append(_marg(prob, cp, cm))
    return out


def _cam(kind, cols, J, r, c):
    Jv, Je = _ve(J, c)
    rv, re = _ve(r, c)
    return CamFactor(kind, cols, Jv, Je, rv, re)


def _marg(prob, cp, cm):
    K, r = prob["K"], prob["marg_r"]
    pose, mix, ext = prob["pose"].reshape(-1, 7), prob["mix"].reshape(-1, 9), prob["ext"]
    types, nodes = prob["marg_block_type"], prob["marg_block_node"]
    params, cols = [], []
    for t, nd in zip(types, nodes):
        t, nd = int(t), int(nd)
        params.append(pose[nd] if t == 0 else mix[nd] if t == 1 else ext[:7] if t == 2 else ext[7:8])
        c = cp(nd) if t == 0 else cm(nd) if t == 1 else list(range(6 * K, 6 * K + 6)) if t == 2 else [6 * K + 6]
        if (t == 2 and prob["ext_const"]) or (t == 3 and prob["td_const"]):
            c = [-1] * len(c)
        cols += c
    J0 = prob["marg_J0"].reshape(r, r)
    res, _ = fm.marginalization(types, [fm.xs(p) for p in params], fm.xs(prob["marg_x0"]), [fm.xs(row) for row in J0], fm.xs(prob["marg_e0"]))
    rv, re = _ve(res, C_SMALL)
    keep = np.array(cols) >= 0
    J = J0[:, keep]
    # the handle forms H0 = J0^T J0 and b0 = J0^T e0 once, in doubles, and g = b0 + H0 dx: the roundings of that path are those of r = e0 +
    # J0 dx, which the bound of r carries, and of the two products, which m covers
    return CamFactor("marginalization", np.array(cols)[keep], J, np.zeros_like(J), rv, re)


# ---------------------------------------------------------------------------------------------- the assembly
def factors(prob):
    """(vision factors of the active reprojection factors, camera-only factors): the slow part, separate so that mutations reuse it"""
    vis = [vis_factor(prob, f) for f in range(prob["F"]) if prob["f_active"][f]]
    return vis, cam_factors(prob)


def tri20(a, b):
    return a * 20 - a * (a - 1) // 2 + (b - a)


TRI20 = np.array([[tri20(min(a, b), max(a, b)) for b in range(20)] for a in range(20)])
UPPER20 = np.triu(np.ones((20, 20), bool))


def vis_cols(K, ref, obs):
    """the window columns of a record's 20 columns: the 19 Jacobian columns, then the residual as column NCV (the augmented vision matrix)"""
    return np.array(list(range(6 * ref, 6 * ref + 6)) + list(range(6 * obs, 6 * obs + 6)) + list(range(6 * K, 6 * K + 7)) + [6 * K + 7])


def assemble(prob, vis, cam, radius, dup_rows=None, wrong_rows=None, no_d2=False):
    """the reference system of a window: a dict of (value, bound) pairs.  radius: the trust-region radius of the Schur complement.
    Mutations: dup_rows, a (reference, observing) pair whose first factor's rows are counted twice; wrong_rows, (pair, factor): the pair's
    Gram matrix takes that factor's records (of another pair) in place of its own first factor's; no_d2: phi_l without D_l^2."""
    K, L = prob["K"], prob["L"]
    NCV, N = 6 * K + 7, 15 * K + 7
    out = {}
    # ---- ba_lin_vis: per-pair Gram matrices
    pairs = {}
    for v in vis:
        pairs.setdefault((v.ref, v.obs), []).append(v)
    Mp = {}
    for key, fs in pairs.items():
        if wrong_rows is not None and key == wrong_rows[0]:
            fs = [wrong_rows[1]] + fs[1:]
        X = np.concatenate([v.X for v in fs] + ([fs[0].X] if key == dup_rows else []))
        XE = np.concatenate([v.XE for v in fs] + ([fs[0].XE] if key == dup_rows else []))
        G, E = gram(X, XE, 3 * len(X))
        Mp[key] = (G[UPPER20], E[UPPER20])
    out["Mp"] = Mp
    # ---- landmark terms and coupling rows
    AW, AWE = np.zeros((L, NCV + 1)), np.zeros((L, NCV + 1))
    hl, hlE, gl, glE = np.zeros(L), np.zeros(L), np.zeros(L), np.zeros(L)
    by_l = {}
    for v in vis:
        by_l.setdefault(v.l, []).append(v)
    for l, fs in by_l.items():
        W, WE = np.zeros((2 * len(fs), NCV + 2)), np.zeros((2 * len(fs), NCV + 2))
        for q, v in enumerate(fs):
            c = vis_cols(K, v.ref, v.obs)
            W[2 * q:2 * q + 2, c], WE[2 * q:2 * q + 2, c] = v.X, v.XE
            W[2 * q:2 * q + 2, NCV + 1], WE[2 * q:2 * q + 2, NCV + 1] = v.jr, v.jrE
        G, E = gram(W, WE, 2 * len(W))
        AW[l], AWE[l] = G[NCV + 1, :NCV + 1], E[NCV + 1, :NCV + 1]
        hl[l], hlE[l], gl[l], glE[l] = G[NCV + 1, NCV + 1], E[NCV + 1, NCV + 1], G[NCV + 1, NCV], E[NCV + 1, NCV]
    out.update(A_W=(AW, AWE), h_l=(hl, hlE), g_l=(gl, glE))
    out["costf"] = {v.f: (v.cost, v.costE) for v in vis}
    # ---- ba_lin_cam
    Hc, HcE, gc, gcE = Sum2((N, N)), np.zeros((N, N)), Sum2(N), np.zeros(N)
    nterm = np.zeros((N, N))
    for c in cam:
        A = np.concatenate([c.J, c.r[:, None]], axis=1)
        AE = np.concatenate([c.JE, c.rE[:, None]], axis=1)
        G, E = gram(A, AE, 0)
        n = len(c.cols)
        ix = np.ix_(c.cols, c.cols)
        Hc.add(_scatter((N, N), ix, G[:n, :n]))
        gc.add(_scatter(N, (c.cols,), G[:n, n]))
        HcE[ix] += E[:n, :n] + np.abs(G[:n, :n])     # + the rounding of this factor's exactly rounded contribution
        gcE[c.cols] += E[:n, n] + np.abs(G[:n, n])
        nterm[ix] += len(A) + 1
    Hc, gc = Hc.value(), gc.value()
    # gamma over the terms of an entry: every factor's products and one addition per factor (the reference's own cross-factor sum is exact)
    absum = Sum2((N, N))
    for c in cam:
        A = np.abs(np.concatenate([c.J, c.r[:, None]], axis=1))
        n = len(c.cols)
        S = A.T @ A
        absum.add(_scatter((N, N), np.ix_(c.cols, c.cols), S[:n, :n]))
    absum = absum.value()
    mcam = nterm.max() if nterm.any() else 0
    HcE += mcam * absum
    gabs = np.zeros(N)
    for c in cam:
        gabs[c.cols] += np.abs(c.J).T @ np.abs(c.r)
    gcE += mcam * gabs
    out.update(H_c=(Hc, HcE), g_c=(gc, gcE))
    # ---- the vision Gram matrix [H_vis g_vis] over all pairs (ba_schur_dmma's gather of Mp)
    rows = sum(len(v.X) for v in vis)
    V, VE = np.zeros((max(rows, 1), NCV + 1)), np.zeros((max(rows, 1), NCV + 1))
    q = 0
    for v in vis:
        c = vis_cols(K, v.ref, v.obs)
        V[q:q + 2, c], VE[q:q + 2, c] = v.X, v.XE
        q += 2
    Hv, HvE = gram(V, VE, 3 * rows + 2 * len(pairs))
    # ---- the Schur term sum_l phi_l w_l w_l^T (w_l augmented with g_l)
    scale, scaleE, phi, phiE = np.zeros(L), np.zeros(L), np.zeros(L), np.zeros(L)
    with mpmath.workdps(fm.DPS):
        for l in range(L):
            h = fm.X(hl[l], C_LIN_VIS * hlE[l])
            s = 1 / (1 + fm.xsqrt(h))
            s2 = s * s
            hs = s2 * h
            d2 = fm.X(0) if no_d2 else (hs if MIN_DIAG < hs.v < MAX_DIAG else fm.X(MIN_DIAG if hs.v <= MIN_DIAG else MAX_DIAG)) / fm.X(radius)
            p = s2 / (hs + d2) if (hs + d2).v else fm.X(0)  # only when D_l^2 is left out (a mutation) and h_l = 0
            scale[l], scaleE[l] = float(s.v), float(s.e) + abs(float(s.v))
            phi[l], phiE[l] = float(p.v), float(p.e) + abs(float(p.v))
    out["scale_l"] = (scale, scaleE)
    T, TE = Sum2((NCV + 1, NCV + 1)), np.zeros((NCV + 1, NCV + 1))
    Tabs = np.zeros((NCV + 1, NCV + 1))
    nl = 0
    for l in range(L):
        w, we = AW[l], C_LIN_VIS * AWE[l]
        if not w.any():
            continue
        nl += 1
        a, ae = two_prod(phi[l], w)   # phi w exactly as a + ae
        T.add_prod(a[:, None], w[None, :])
        T.add_prod(ae[:, None], w[None, :])
        pw = np.abs(phi[l] * w)
        TE += pw[:, None] * we[None, :] + (np.abs(phi[l]) * we)[:, None] * np.abs(w)[None, :] + phiE[l] * np.abs(np.outer(w, w))
        Tabs += np.outer(pw, np.abs(w))
    T = T.value()
    TE += (nl + 2 + 4) * Tabs   # the landmarks' products, phi w, the cluster's four split partials
    # ---- Hs = H_c + H_vis - T (vision rows, lower triangle) and visv
    Hs = Sum2((NCV, NCV))
    for M in (Hc[:NCV, :NCV], Hv[:NCV, :NCV], -T[:NCV, :NCV]):
        Hs.add(M)
    HsE = C_LIN_CAM * HcE[:NCV, :NCV] + C_LIN_VIS * HvE[:NCV, :NCV] + TE[:NCV, :NCV]
    HsE += 2 * (np.abs(Hc[:NCV, :NCV]) + np.abs(Hv[:NCV, :NCV]) + np.abs(T[:NCV, :NCV])) + 3 * np.abs(Hs.value())
    out["Hs"] = (np.tril(Hs.value()), np.tril(HsE))
    out["visv"] = (np.stack([np.diag(Hv)[:NCV], Hv[:NCV, NCV], T[:NCV, NCV]]),
                   np.stack([C_LIN_VIS * np.diag(HvE)[:NCV], C_LIN_VIS * HvE[:NCV, NCV], TE[:NCV, NCV]]))
    out["phi"], out["H_vis"] = (phi, phiE), (Hv, HvE)
    return out


def _scatter(shape, ix, vals):
    z = np.zeros(shape)
    z[ix] = vals
    return z


# ---------------------------------------------------------------------------------------------- the comparison
KERNEL_OF = {"Mp": "ba_lin_vis", "A_W": "ba_lin_vis", "h_l": "ba_lin_vis", "g_l": "ba_lin_vis", "costf": "ba_lin_vis", "scale_l": "ba_lin_vis",
             "H_c": "ba_lin_cam", "g_c": "ba_lin_cam", "Hs": "ba_schur_dmma", "visv": "ba_schur_dmma"}
CONST = {"ba_lin_vis": C_LIN_VIS, "ba_lin_cam": C_LIN_CAM, "ba_schur_dmma": C_SCHUR}


def ratio(got, val, bnd, c):
    """worst |got - val| / (c eps bnd); entries with a zero bound must match exactly (returned as inf when they do not)"""
    got, val, bnd = (np.asarray(x, float) for x in (got, val, bnd))
    d = np.abs(got - val)
    if (d[bnd == 0] > 0).any() or not np.isfinite(got).all():
        return math.inf
    return float((d[bnd > 0] / (c * EPS * bnd[bnd > 0])).max()) if (bnd > 0).any() else 0.0


def ratios(dev, ref):
    """worst error-to-bound ratio of every read-out array against the reference (dev: peek_linearization's dict)"""
    out = {}
    for name, kern in KERNEL_OF.items():
        c = CONST[kern]
        if name == "Mp":
            assert set(dev["Mp"]) == set(ref["Mp"]), (sorted(dev["Mp"]), sorted(ref["Mp"]))
            out[name] = max([ratio(dev["Mp"][k], *ref["Mp"][k], c) for k in ref["Mp"]], default=0.0)
        elif name == "costf":
            out[name] = max([ratio(dev["costf"][f], *ref["costf"][f], c) for f in ref["costf"]], default=0.0)
            inactive = [f for f in range(len(dev["costf"])) if f not in ref["costf"]]
            if np.any(dev["costf"][inactive] != 0):
                out[name] = math.inf
        elif name == "Hs":
            out[name] = ratio(np.tril(dev["Hs"]), *ref["Hs"], c)
        else:
            out[name] = ratio(dev[name], *ref[name], c)
    return out
