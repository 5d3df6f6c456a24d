"""Generate the KLT edge golden vectors from cv2 (opencv-python-headless 4.13.0, as make_klt_golden.py).  Run HERE (needs cv2):

    python tests/golden/make_klt_edges_golden.py

Writes tests/golden/klt_edges_golden.npz: cv2.calcOpticalFlowPyrLK on points placed at every image edge of every pyramid level it builds,
at sizes where cv2 builds 1 to 4 levels and at every level-0 width residue mod 16, plus the CRC32 of every cv2.pyrDown level.  Frames are
not stored: they are re-rendered from datagen/synth_klt.py (make_texture + render_frame, arguments `<case>_args`) and guarded by a CRC32 per
frame.  The script is deterministic: re-running it reproduces the file byte for byte.

Per LK case `<c>` (W x H in `<c>_args` = W, H, texture seed, t; frames t - 1 and t):
  <c>_p0, <c>_init             edge rings (synth_klt.edge_rings) + corner points; init = true motion + N(0, 1 px), and a subset whose
                               initial flow lies beyond the far edge of the top level
  <c>_lk<m>f<f>_{fwd,st,err}   forward LK with err, maxLevel m = 0..3, flags f = 0 or 4 (USE_INITIAL_FLOW)
  <c>_fb_{fwd,bwd,st,st2,good} the reference's forward + backward + gates sequence (make_klt_golden.fb)
  <c>_count_*, <c>_eps_*       maxLevel 3, USE_INITIAL_FLOW, criteria (COUNT, 30, 0.5) and (EPS, 5, 0.01)
  <c>_rc_{p0,init,dir,fwd,st,err}  maxLevel 0, initial flow 6-20 px off the true motion in direction dir (0 +x, 1 -x, 2 +y, 3 -y): the
                               track walks out of its first search window
  <c>_dropped                  points dropped as ambiguous: cv2's forward position within 2e-3 px of a 5-px border gate threshold, or its
                               forward-backward distance within 2e-3 of 0.5
Every recorded call also has `_tie`: the points whose cv2 position the tests do not hold to 1e-3 px (see ties()).
`mc_*` (case `mc_case`): maxLevel 0, (COUNT+EPS, 150, 0), points whose cv2 result changes between 99 and 100 iterations (cv2 clamps
maxCount to 100).  `pyr_sizes` + `pyr_<W>x<H>_{args,crc}`: CRC32 of levels 0..3 of both frames (rows: frame, columns: level).
"""
import os
import sys
import zlib

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, HERE)
from datagen import synth_klt as synth  # noqa: E402
from make_klt_golden import CRIT, fb  # noqa: E402
from make_klt_golden import lk as lk_cv2  # noqa: E402

LK_SIZES = [(32, 32), (42, 100), (43, 100), (320, 168), (320, 169), (168, 240), (176, 180), (179, 180), (186, 180), (191, 180)]
PYR_SIZES = LK_SIZES[:6] + [(w, 180) for w in range(176, 192)]
T = {0: 1, 1: 30, 2: 12, 3: 47, 4: 60, 5: 25, 6: 5, 7: 38, 8: 53, 9: 18}  # frame index per LK case: motions in all four quadrants
CRIT_COUNT = (cv2.TERM_CRITERIA_COUNT, 30, 0.5)
CRIT_EPS = (cv2.TERM_CRITERIA_EPS, 5, 0.01)
CRIT_MC = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 150, 0.0)
AMBIG = 2e-3
TIE_PX = 5e-4


def lk(*a, **kw):
    """make_klt_golden.lk with err zeroed where the status is 0 (cv2 leaves err of some lost points unwritten)"""
    q, st, err = lk_cv2(*a, **kw)
    return q, st, np.where(st == 1, err, np.float32(0))


def ties(f0, f1, p0, init, q, **kw):
    """points whose cv2 position sits on a discrete decision of the iteration rather than on the image: it moves by more than TIE_PX when
    the epsilon moves by 1 %, when one more iteration is allowed, or when the start point moves by 1e-4 px along an axis.  Tiny rounding
    differences can flip such a decision (an exit one step earlier or later) or, in an ill-conditioned window, move the solution by more
    than 1e-3 px, so the position bar skips these points; their status is compared all the same."""
    crit = kw.pop("criteria", CRIT)
    count = min(crit[1], 100) if crit[0] & cv2.TERM_CRITERIA_COUNT else 30  # cv2's effective criteria
    eps = crit[2] if crit[0] & cv2.TERM_CRITERIA_EPS else 0.01
    both = cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS
    variants = [(p0 + d, crit) for d in np.array([[1e-4, 0], [-1e-4, 0], [0, 1e-4], [0, -1e-4]], np.float32)]
    if eps > 0:
        variants += [(p0, (both, count, 0.99 * eps)), (p0, (both, count, 1.01 * eps))]
    if count < 100:
        variants.append((p0, (both, count + 1, eps)))
    t = np.zeros(len(p0), bool)
    for a, c in variants:
        t |= np.abs(lk(f0, f1, a, init, criteria=c, **kw)[0] - q).max(axis=1) > TIE_PX
    return t.astype(np.uint8)


def case_name(W, H):
    return f"s{W}x{H}"


def frames(W, H, seed, t):
    tex = synth.make_texture(W, H, seed)
    return synth.render_frame(tex, t - 1, W, H), synth.render_frame(tex, t, W, H)


def true_motion(p0, t, W, H):
    """where the texture point seen at p0 in frame t - 1 appears in frame t"""
    bx, by = synth.unwarp_point(p0[:, 0].astype(np.float64), p0[:, 1].astype(np.float64), t - 1, W, H)
    x1, y1 = synth.warp_point(bx, by, t, W, H)
    return np.stack([x1, y1], axis=1)


def check_origins(p, W, H, n_levels):
    """every fixed-fraction ring point lands on its intended level-l origin after the float32 round trip (x 2^-l - 10, as the tracker)"""
    k = 0
    for level, (wl, hl) in enumerate(synth.pyramid_sizes(W, H, n_levels)):
        s = np.float32(2.0 ** -level)
        for axis, nl in ((0, wl), (1, hl)):
            for o in [*synth.EDGE_LO, *(nl + d for d in synth.EDGE_HI)]:
                for _ in synth.EDGE_FRACS:
                    assert int(np.floor(p[k, axis] * s - np.float32(10))) == o, (W, H, level, axis, o)
                    k += 1
        k += 16


def lk_case(idx, W, H, out):
    c = case_name(W, H)
    seed, t = 300 + idx, T[idx]
    f0, f1 = frames(W, H, seed, t)
    nl = synth.lk_levels(W, H)
    assert len(cv2.buildOpticalFlowPyramid(f0, (21, 21), 3, withDerivatives=False)[1]) == nl
    rng = np.random.Generator(np.random.PCG64(seed))
    p0 = synth.edge_rings(W, H, nl, rng)
    check_origins(p0, W, H, nl)
    init = true_motion(p0, t, W, H) + rng.normal(0.0, 1.0, p0.shape)
    # every 8th point: initial flow beyond the far edge of the top level (its first search window is never staged there)
    top_w, top_h = synth.pyramid_sizes(W, H, nl)[-1]
    s = float(1 << (nl - 1))
    far = np.arange(0, len(p0), 8)
    side = rng.integers(0, 4, far.size)
    d = rng.uniform(0.5, 8.0, far.size)
    init[far[side == 0], 0] = (top_w + 10 + d[side == 0]) * s
    init[far[side == 1], 1] = (top_h + 10 + d[side == 1]) * s
    init[far[side == 2], 0] = (-21 - d[side == 2] + 10) * s
    init[far[side == 3], 1] = (-21 - d[side == 3] + 10) * s
    init = init.astype(np.float32)
    # ambiguous points of the forward-backward gate
    fwd, bwd, st, st2, good = fb(f0, f1, p0, init)
    both = (st == 1) & (st2 == 1)
    near_border = np.zeros(len(p0), bool)
    for v, thr in ((fwd[:, 0], 5.0), (fwd[:, 1], 5.0), (fwd[:, 0], W - 5.0), (fwd[:, 1], H - 5.0)):
        near_border |= np.abs(v.astype(np.float64) - thr) < AMBIG
    dist = np.hypot((bwd[:, 0] - p0[:, 0]).astype(np.float64), (bwd[:, 1] - p0[:, 1]).astype(np.float64))
    drop = both & (near_border | (np.abs(dist - 0.5) < AMBIG))
    p0, init = p0[~drop], init[~drop]
    out[c + "_args"] = np.array([W, H, seed, t], np.int64)
    out[c + "_crc"] = np.array([zlib.crc32(f0.tobytes()), zlib.crc32(f1.tobytes())], np.uint64)
    out[c + "_p0"], out[c + "_init"], out[c + "_dropped"] = p0, init, np.int64(drop.sum())
    for m in range(4):
        for flags in (0, cv2.OPTFLOW_USE_INITIAL_FLOW):
            q, st, err = lk(f0, f1, p0, init, max_level=m, flags=flags)
            out[f"{c}_lk{m}f{flags}_fwd"], out[f"{c}_lk{m}f{flags}_st"], out[f"{c}_lk{m}f{flags}_err"] = q, st, err
            out[f"{c}_lk{m}f{flags}_tie"] = ties(f0, f1, p0, init, q, max_level=m, flags=flags)
    for k, v in zip(("fwd", "bwd", "st", "st2", "good"), fb(f0, f1, p0, init)):
        out[f"{c}_fb_{k}"] = v
    # forward call = lk3f4; backward call as fb makes it
    out[c + "_fb_tie"] = out[c + "_lk3f4_tie"] | ties(f1, f0, out[c + "_fb_fwd"], p0, out[c + "_fb_bwd"])
    ref = lk(f0, f1, p0, init)
    for key, crit in (("count", CRIT_COUNT), ("eps", CRIT_EPS)):
        q, st, err = lk(f0, f1, p0, init, criteria=crit)
        out[f"{c}_{key}_fwd"], out[f"{c}_{key}_st"], out[f"{c}_{key}_err"] = q, st, err
        out[f"{c}_{key}_tie"] = ties(f0, f1, p0, init, q, criteria=crit)
    # COUNT without EPS is COUNT + EPS with cv2's default epsilon 0.01
    assert np.array_equal(out[c + "_count_fwd"], ref[0]) and np.array_equal(out[c + "_count_st"], ref[1])
    # re-centre: interior points, initial flow 6-20 px off the true motion in each direction, maxLevel 0
    n = 60
    m = 25 if min(W, H) > 60 else 11
    rp = np.stack([rng.uniform(m, W - m, 4 * n), rng.uniform(m, H - m, 4 * n)], axis=1).astype(np.float32)
    rdir = np.repeat(np.arange(4), n)
    off = rng.uniform(6.0, 20.0, 4 * n)
    step = np.array([[1, 0], [-1, 0], [0, 1], [0, -1]], np.float64)[rdir] * off[:, None]
    rinit = (true_motion(rp, t, W, H) + step).astype(np.float32)
    q, st, err = lk(f0, f1, rp, rinit, max_level=0)
    out[c + "_rc_p0"], out[c + "_rc_init"], out[c + "_rc_dir"] = rp, rinit, rdir.astype(np.int8)
    out[c + "_rc_fwd"], out[c + "_rc_st"], out[c + "_rc_err"] = q, st, err
    out[c + "_rc_tie"] = ties(f0, f1, rp, rinit, q, max_level=0)
    print(c, "levels", nl, "points", len(p0), "dropped", int(drop.sum()), "lk3 tracked", int(out[c + "_lk3f4_st"].sum()),
          "ties", int((out[c + "_lk3f4_tie"] & out[c + "_lk3f4_st"]).sum()), "fb good", int(out[c + "_fb_good"].sum()),
          "rc tracked", int(st.sum()), "ties", int((out[c + "_rc_tie"] & st).sum()))


def max_count_case(out):
    """points that are still moving at iteration 100 (cv2's result differs between maxCount 99 and 100): 150 must stop at 100"""
    W, H = 320, 169
    idx = LK_SIZES.index((W, H))
    seed, t = 300 + idx, T[idx]
    f0, f1 = frames(W, H, seed, t)
    rng = np.random.Generator(np.random.PCG64(seed + 1000))
    p = np.stack([rng.uniform(-20, W + 20, 4000), rng.uniform(-20, H + 20, 4000)], axis=1).astype(np.float32)
    init = (true_motion(p, t, W, H) + rng.normal(0.0, 4.0, p.shape)).astype(np.float32)
    r = {k: lk(f0, f1, p, init, max_level=0, criteria=(CRIT_MC[0], k, 0.0)) for k in (99, 100)}
    q, st, err = lk(f0, f1, p, init, max_level=0, criteria=CRIT_MC)
    assert np.array_equal(q, r[100][0]) and np.array_equal(st, r[100][1])
    sel = (np.abs(r[99][0] - r[100][0]).max(axis=1) > 0) | (r[99][1] != r[100][1])
    sel |= np.arange(len(p)) < 100  # and some ordinary points around them
    out["mc_case"] = np.array([W, H], np.int64)
    out["mc_p0"], out["mc_init"], out["mc_fwd"], out["mc_st"], out["mc_err"] = p[sel], init[sel], q[sel], st[sel], err[sel]
    out["mc_tie"] = ties(f0, f1, p[sel], init[sel], q[sel], max_level=0, criteria=CRIT_MC)
    print("maxCount 150:", int(sel.sum()), "points,", int((sel & (st == 1)).sum()), "tracked")


def main():
    out = {}
    for idx, (W, H) in enumerate(LK_SIZES):
        lk_case(idx, W, H, out)
    max_count_case(out)
    out["pyr_sizes"] = np.array(PYR_SIZES, np.int64)
    for k, (W, H) in enumerate(PYR_SIZES):
        seed, t = 500 + k, 2
        crc = np.zeros((2, 4), np.uint64)
        for i, img in enumerate(frames(W, H, seed, t)):
            for level in range(4):
                crc[i, level] = zlib.crc32(np.ascontiguousarray(img).tobytes())
                img = cv2.pyrDown(img)
        out[f"pyr_{W}x{H}_args"] = np.array([W, H, seed, t], np.int64)
        out[f"pyr_{W}x{H}_crc"] = crc
    path = os.path.join(HERE, "klt_edges_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes; cv2", cv2.__version__)


if __name__ == "__main__":
    main()
