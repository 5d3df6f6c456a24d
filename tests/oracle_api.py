"""ctypes signatures + numpy wrappers for the CPU oracle (oracle/libicg_oracle.so).  Tests/bench only."""
import ctypes as C

import numpy as np

vp = C.c_void_p


def _p(a):
    return C.c_void_p(a.ctypes.data)


def declare(lib):
    lib.icgo_pyr_down.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, C.c_int]
    lib.icgo_pyr_down.restype = None
    lib.icgo_calc_optical_flow_pyr_lk.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int,
                                                  C.c_int, C.c_int, C.c_double, C.c_int, C.c_double]
    lib.icgo_calc_optical_flow_pyr_lk.restype = C.c_int
    lib.icgo_track_fb.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int,
                                  C.c_double, C.c_double, C.c_double]
    lib.icgo_track_fb.restype = None


def pyr_down(lib, img):
    H, W = img.shape
    out = np.zeros(((H + 1) // 2, (W + 1) // 2), np.uint8)
    img = np.ascontiguousarray(img)
    lib.icgo_pyr_down(_p(img), W, H, W, _p(out), out.shape[1])
    return out


def lk(lib, a, b, p, init, max_level=3, max_iter=30, eps=0.01, flags=4, want_err=True):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    H, W = a.shape
    p = np.ascontiguousarray(p, np.float32).reshape(-1, 2)
    q = np.array(init, np.float32).reshape(-1, 2).copy()
    n = p.shape[0]
    st = np.zeros(n, np.uint8)
    err = np.zeros(n, np.float32)
    lib.icgo_calc_optical_flow_pyr_lk(_p(a), _p(b), W, H, W, _p(p), _p(q), _p(st), _p(err) if want_err else None, n, 21,
                                      max_level, max_iter, eps, flags, 1e-4)
    return q, st, err


def track_fb(lib, a, b, p, init):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    H, W = a.shape
    p = np.ascontiguousarray(p, np.float32).reshape(-1, 2)
    q = np.array(init, np.float32).reshape(-1, 2).copy()
    n = p.shape[0]
    back = np.zeros((n, 2), np.float32)
    st = np.zeros(n, np.uint8)
    lib.icgo_track_fb(_p(a), _p(b), W, H, W, _p(p), _p(q), _p(back), _p(st), n, 21, 3, 30, 0.01, 0.5, 5.0)
    return q, back, st


# ------------------------------------------------------------------------------------------------ BA oracle
def declare_ba(lib):
    from ic_gvins_b200._lib import BaProblem, BaSummary
    lib.icgo_ba_solve.argtypes = [C.POINTER(BaProblem), vp, vp, C.c_int, C.c_int, C.POINTER(BaSummary)]
    lib.icgo_ba_residual_costs.argtypes = [C.POINTER(BaProblem), vp, vp]
    lib.icgo_preintegrate.argtypes = [vp, vp, vp, vp, vp, C.c_int, vp, vp, vp]
    lib.icgo_reproj_eval.argtypes = [vp, vp, vp, vp, vp, vp, C.c_double, vp, vp]
    lib.icgo_imu_eval.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, vp, vp]
    lib.icgo_gnss_eval.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.icgo_pose_prior_eval.argtypes = [vp, vp, vp, vp, vp]
    lib.icgo_reproj_eval_loss.argtypes = [vp, vp, vp, vp, vp, vp, C.c_double, C.c_int, vp, vp, vp]
    lib.icgo_gnss_eval_loss.argtypes = [vp, vp, vp, vp, C.c_int, vp, vp, vp]
    lib.icgo_pose_plus.argtypes = [vp, vp, vp]
    lib.icgo_pose_plus.restype = None
    lib.icgo_ba_marginalize.argtypes = [C.POINTER(BaProblem), vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.icgo_sym_eig.argtypes = [vp, C.c_int, vp, vp]
    lib.icgo_sym_eig.restype = None


def preintegrate(lib, state16, iewn, gravity, noise5, imu):
    imu = np.ascontiguousarray(imu, np.float64)
    n = imu.shape[0]
    blob = np.zeros(480)
    pn = np.zeros((n - 1, 4))
    end = np.zeros(10)
    a = [np.ascontiguousarray(x, np.float64) if x is not None else None for x in (state16, iewn, gravity, noise5)]
    # iewn None: PreintegrationNormal (iswithearth false); pn stays empty in that form
    lib.icgo_preintegrate(_p(a[0]), _p(a[1]) if a[1] is not None else None, _p(a[2]), _p(a[3]), _p(imu), n, _p(blob), _p(pn), _p(end))
    if iewn is None:
        pn = np.zeros((0, 4))
    return blob, pn, end


def ba_solve(lib, prob, max_iter, num_threads=1):
    from ic_gvins_b200._lib import BaSummary
    from ic_gvins_b200.ba import to_struct
    s = to_struct(prob)
    pn = np.ascontiguousarray(prob["pn"], np.float64)
    off = np.ascontiguousarray(prob["pn_off"], np.int32)
    summ = BaSummary()
    lib.icgo_ba_solve(C.byref(s), _p(pn), _p(off), max_iter, num_threads, C.byref(summ))
    return dict(iterations=summ.iterations, num_successful_steps=summ.num_successful_steps, termination=summ.termination,
                initial_cost=summ.initial_cost, final_cost=summ.final_cost, final_radius=summ.final_radius)


def ba_residual_costs(lib, prob):
    from ic_gvins_b200.ba import to_struct
    s = to_struct(prob)
    rc = np.zeros(prob["F"])
    gc = np.zeros(prob["n_gnss"])
    lib.icgo_ba_residual_costs(C.byref(s), _p(rc), _p(gc))
    return rc, gc


def ba_marginalize(lib, prob, num_marg=1):
    """MarginalizationInfo::marginalization on the window (oracle).  Returns a dict with the new prior in the layout
    icg_ba_problem.marg_* uses (node indices already shifted by num_marg) + the Schur complement (Hp, bp)."""
    from ic_gvins_b200.ba import to_struct
    s = to_struct(prob)
    pn = np.ascontiguousarray(prob["pn"], np.float64)
    off = np.ascontiguousarray(prob["pn_off"], np.int32)
    rmax = 15 * prob["K"] + 7
    m = np.zeros(1, np.int32); nb = np.zeros(1, np.int32)
    bt = np.zeros(2 * prob["K"] + 2, np.int32); bn = np.zeros(2 * prob["K"] + 2, np.int32)
    x0 = np.zeros(16 * prob["K"] + 8); J0 = np.zeros(rmax * rmax); e0 = np.zeros(rmax); Hp = np.zeros(rmax * rmax); bp = np.zeros(rmax)
    r = lib.icgo_ba_marginalize(C.byref(s), _p(pn), _p(off), num_marg, _p(m), _p(nb), _p(bt), _p(bn), _p(x0), _p(J0), _p(e0), _p(Hp), _p(bp))
    nb = int(nb[0])
    gs = {0: 7, 1: 9, 2: 7, 3: 1}
    nx = sum(gs[int(t)] for t in bt[:nb])
    return dict(m=int(m[0]), r=r, block_type=bt[:nb].copy(), block_node=bn[:nb].copy(), x0=x0[:nx].copy(),
                J0=J0[:r * r].reshape(r, r).copy(), e0=e0[:r].copy(), Hp=Hp[:r * r].reshape(r, r).copy(), bp=bp[:r].copy())


def sym_eig(lib, A):
    A = np.ascontiguousarray(A, np.float64)
    n = A.shape[0]
    ev = np.zeros(n); V = np.zeros((n, n))
    lib.icgo_sym_eig(_p(A), n, _p(ev), _p(V))
    return ev, V


def reproj_eval(lib, pose0, pose1, ext, rho, td, c14, std, want_jac=True):
    a = [np.ascontiguousarray(x, np.float64) for x in (pose0, pose1, ext, np.atleast_1d(rho), np.atleast_1d(td), c14)]
    r = np.zeros(2)
    Js = [np.zeros((2, 7)), np.zeros((2, 7)), np.zeros((2, 7)), np.zeros((2, 1)), np.zeros((2, 1))]
    jp = (vp * 5)(*[vp(j.ctypes.data) for j in Js])
    lib.icgo_reproj_eval(*[_p(x) for x in a], float(std), _p(r), jp if want_jac else None)
    return r, Js


def imu_eval(lib, blob, pn, pose0, mix0, pose1, mix1, want_jac=True):
    a = [np.ascontiguousarray(x, np.float64) for x in (blob, pn, pose0, mix0, pose1, mix1)]
    r = np.zeros(15)
    Js = [np.zeros((15, 7)), np.zeros((15, 9)), np.zeros((15, 7)), np.zeros((15, 9))]
    jp = (vp * 4)(*[vp(j.ctypes.data) for j in Js])
    lib.icgo_imu_eval(_p(a[0]), _p(a[1]), a[1].size // 4, _p(a[2]), _p(a[3]), _p(a[4]), _p(a[5]), _p(r), jp if want_jac else None)
    return r, Js


def reproj_eval_loss(lib, pose0, pose1, ext, rho, td, c14, std, huber):
    """ReprojectionFactor with the loss the solver applies (evaluate_block's apply_loss): corrected r, global Jacobians, cost"""
    a = [np.ascontiguousarray(x, np.float64) for x in (pose0, pose1, ext, np.atleast_1d(rho), np.atleast_1d(td), c14)]
    r, cost = np.zeros(2), np.zeros(1)
    Js = [np.zeros((2, 7)), np.zeros((2, 7)), np.zeros((2, 7)), np.zeros((2, 1)), np.zeros((2, 1))]
    jp = (vp * 5)(*[vp(j.ctypes.data) for j in Js])
    lib.icgo_reproj_eval_loss(*[_p(x) for x in a], float(std), int(huber), _p(r), jp, _p(cost))
    return r, Js, float(cost[0])


def gnss_eval_loss(lib, pose, blh, std3, lever, huber):
    a = [np.ascontiguousarray(x, np.float64) for x in (pose, blh, std3, lever)]
    r, J, cost = np.zeros(3), np.zeros((3, 7)), np.zeros(1)
    lib.icgo_gnss_eval_loss(*[_p(x) for x in a], int(huber), _p(r), _p(J), _p(cost))
    return r, J, float(cost[0])


def pose_plus(lib, x, d):
    x = np.ascontiguousarray(x, np.float64); d = np.ascontiguousarray(d, np.float64)
    out = np.zeros(7)
    lib.icgo_pose_plus(_p(x), _p(d), _p(out))
    return out


# ------------------------------------------------------------------------------------------------ detection oracle
def declare_detect(lib):
    lib.icgo_min_eig_roi.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    lib.icgo_min_eig_roi.restype = None
    lib.icgo_good_features_from_eig.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_double, C.c_double, vp]
    lib.icgo_good_features_from_eig.restype = C.c_int
    lib.icgo_corner_subpix_roi.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_double]
    lib.icgo_corner_subpix_roi.restype = None
    lib.icgo_rect_subpix.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, vp]
    lib.icgo_rect_subpix.restype = None
    lib.icgo_detect_block.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, vp]
    lib.icgo_detect_block.restype = C.c_int


def min_eig_roi(lib, img, roi):
    img = np.ascontiguousarray(img)
    H, W = img.shape
    x0, y0, w, h = roi
    eig = np.zeros((h, w), np.float32)
    lib.icgo_min_eig_roi(_p(img), W, H, W, x0, y0, w, h, _p(eig))
    return eig


def good_features(lib, img, n, quality, min_dist, mask=None, roi=None):
    img = np.ascontiguousarray(img)
    H, W = img.shape
    roi = roi or (0, 0, W, H)
    eig = min_eig_roi(lib, img, roi)
    x0, y0, w, h = roi
    out = np.zeros((w * h, 2), np.float32)  # max_corners <= 0 is unlimited: every pixel can be a corner
    m = None
    if mask is not None:
        m = np.ascontiguousarray(mask)
        mp = C.c_void_p(m.ctypes.data + y0 * W + x0)
    cnt = lib.icgo_good_features_from_eig(_p(eig), w, h, mp if mask is not None else None, W, n, quality, min_dist, _p(out))
    return out[:cnt].copy()


def corner_subpix(lib, img, pts, roi=None):
    img = np.ascontiguousarray(img)
    H, W = img.shape
    x0, y0, w, h = roi or (0, 0, W, H)
    p = np.array(pts, np.float32).reshape(-1, 2).copy()
    lib.icgo_corner_subpix_roi(_p(img), W, H, W, x0, y0, w, h, _p(p), p.shape[0], 5, 20, 0.01)
    return p


def rect_subpix(lib, img, centre, n=13):
    """cv2.getRectSubPix(img, (n, n), centre, patchType=CV_32F) of a u8 image."""
    img = np.ascontiguousarray(img)
    H, W = img.shape
    out = np.zeros((n, n), np.float32)
    lib.icgo_rect_subpix(_p(img), W, H, W, float(centre[0]), float(centre[1]), n, _p(out))
    return out


def detect_block(lib, img, mask, roi, n, quality, min_dist):
    img = np.ascontiguousarray(img)
    H, W = img.shape
    x0, y0, w, h = roi
    out = np.zeros((w * h, 2), np.float32)  # as in good_features
    m = np.ascontiguousarray(mask) if mask is not None else None
    cnt = lib.icgo_detect_block(_p(img), _p(m) if m is not None else None, W, H, W, x0, y0, w, h, n, quality, min_dist, _p(out))
    return out[:cnt].copy()


# ------------------------------------------------------------------------------------------------ CLAHE oracle
def clahe_apply(lib, img, clip, tiles_x, tiles_y, in_place=False):
    lib.icgo_clahe_apply.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, vp, C.c_int]
    lib.icgo_clahe_apply.restype = None
    img = img if in_place else np.ascontiguousarray(img)
    H, W = img.shape
    out = img if in_place else np.zeros_like(img)
    lib.icgo_clahe_apply(_p(img), W, H, W, float(clip), tiles_x, tiles_y, _p(out), W)
    return out
