"""Generate the detection edge golden vectors from cv2 (opencv-python-headless 4.13.0, as make_detect_golden.py).  Run HERE (needs cv2
and the CPU oracle, which it builds):

    python tests/golden/make_detect_edges_golden.py

Writes tests/golden/detect_edges_golden.npz.  Frames are not stored: they are re-rendered from datagen/synth_klt.py or drawn in numpy
(`frame()` below) and guarded by a CRC32 each.  The script is deterministic: re-running it reproduces the file byte for byte.

Whole frames `wf_<W>x<H>` (the sizes in `wf_sizes`) cover the residues the kernels tile by: W % 32 in {0, 1, 31} (the AVX2 row filter
of Sobel covers W & ~31 columns), H % 16 in {0, 1, 15} and every H % 8 (the eig and NMS tiles), W % 16 != 0 (the handle's padded pitch),
frames barely above the 16-px minimum and 752x480:
  _crc, _eig_crc              CRC32 of the frame and of cv2.cornerMinEigenVal(frame, 3, 3)
  _mask                       a mask with two discs cut out (stored: it is small)
  _<tag>_md<k>_{pts,sub}      cv2.goodFeaturesToTrack(frame, WF_N, 0.01, MIN_DISTS[k], mask) in order, and cv2.cornerSubPix of that list
                              (win (5,5), COUNT+EPS 20 / 0.01); tag = nomask or mask
Ties `tie_<name>` (checkerboards of period 4, 7, 8 and a cross-hatch of stripes): many equal eigenvalues, so the order of the list comes
from the address tie-break alone.  `_n` = the number of corners cv2 returns without a limit, `_mc<m>_pts` the list for maxCorners
m in {1, n - 1, n, n + 1} (`_mcs`), at minDistance TIE_MD.
Masks `mask_<name>` on frame `mask_img`: empty, the single pixel of the strongest corner, a single pixel that is no local maximum, the
frame's 1-px border (which NMS skips), and a flat region (masked maximum 0): `_mask` and `_pts` (maxCorners MASK_N, minDistance 5).
Blocks `blk_<W>x<H>`: the reference's block grid (ic_gvins_b200.detect.block_rois, 300 features) on frames 0..N_FRAMES-1 of
synth_klt.KltStream(W, H, 300, 77) (`_crc`: one per frame).  The integer corners come from the oracle (`_pts`, block-local, and
`_idx` = (frame, block)); `_sub` is cv2.cornerSubPix run on a copy of the block.  That copy gives exactly the C++ ROI-view semantics,
because cornerSubPix never reads outside the image it is given (getRectSubPix samples the ROI alone), unlike the Sobel of
goodFeaturesToTrack.  `_placed_{blk,pts,sub}`: corners placed 0-7 px (integer and quarter-pixel) from every edge and corner of two
blocks of frame 0, refined by cv2 on the block copy.
`_tie` (per corner): cv2's result moves by more than TIE_PX when the start point moves 1e-4 px along an axis, or when epsilon changes
by 1 %.  At such corners a window is ill-conditioned or an exit decision is close, so rounding can move the result by more than 1e-3 px.
`flat_*`: a corner at the centre of a flat square (the det ~ 0 break returns it unchanged).
`rs_*`: cv2.getRectSubPix(img, (13, 13), c, patchType=CV_32F) on a 32x24 textured frame, CRC32 of each patch, for every quarter-pixel
centre c inside the frame within 7 px of an edge (`rs_centres`).
"""
import ctypes as C
import os
import subprocess
import sys
import zlib

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..", "..")
sys.path.insert(0, ROOT)
from datagen import synth_klt as synth  # noqa: E402
from ic_gvins_b200.detect import block_rois  # noqa: E402
from tests import oracle_api as oa  # noqa: E402

CRIT = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 20, 0.01)
WF_SIZES = [(17, 16), (17, 20), (31, 22), (33, 18), (64, 48), (65, 33), (95, 31), (97, 17), (127, 60), (129, 61), (160, 47), (200, 43),
            (752, 480)]
MIN_DISTS = [1.0, 1.5, 2.5, 3.49, 5.0, 40.0]  # 1.5 and 2.5 both give a cell of 2 (cvRound rounds half to even)
WF_N = 120
TIE_MD = 1.5
MASK_N = 40
GRIDS = [(1280, 560), (752, 480), (997, 413)]
N_FRAMES = 20
TIE_PX = 5e-4


def frame(seed, W, H):
    return synth.render_frame(synth.make_texture(W, H, seed), 0, W, H)


def subpix(img, pts, crit=CRIT):
    if len(pts) == 0:
        return np.zeros((0, 2), np.float32)
    return cv2.cornerSubPix(img, np.ascontiguousarray(pts, np.float32).reshape(-1, 1, 2).copy(), (5, 5), (-1, -1), crit).reshape(-1, 2)


def ties(img, pts, sub):
    """corners whose cv2 result is not a stable function of the image (see the module docstring)"""
    tie = np.zeros(len(pts), bool)
    H, W = img.shape
    for d in ((1e-4, 0), (0, 1e-4), (-1e-4, 0), (0, -1e-4)):
        q = pts + np.float32(d)
        inside = (q[:, 0] >= 0) & (q[:, 0] < W) & (q[:, 1] >= 0) & (q[:, 1] < H)  # cv2 asserts that a start point lies in the image
        tie |= inside & (np.abs(subpix(img, np.where(inside[:, None], q, pts)) - sub).max(axis=1) > TIE_PX)
    for eps in (0.0099, 0.0101):
        tie |= np.abs(subpix(img, pts, (CRIT[0], CRIT[1], eps)) - sub).max(axis=1) > TIE_PX
    return tie


def gftt(img, n, md, mask=None):
    p = cv2.goodFeaturesToTrack(img, n, 0.01, md, mask=mask)
    return np.zeros((0, 2), np.float32) if p is None else p.reshape(-1, 2)


def crc(a):
    return np.array([zlib.crc32(np.ascontiguousarray(a).tobytes())], np.uint64)


def tie_images():
    yy, xx = np.mgrid[0:48, 0:64]
    out = {}
    for p in (4, 7, 8):
        out[f"checker{p}"] = (((2 * xx // p) + (2 * yy // p)) % 2 * 200 + 20).astype(np.uint8)
    out["stripes"] = np.where((xx % 6 < 2) | (yy % 5 < 2), 230, 30).astype(np.uint8)
    return out


def placed(w, h):
    """0-7 px (integer and quarter steps) from each edge, at a point away from the corners, and from each corner along its diagonal"""
    u = np.array([d + f for d in range(8) for f in (0, 0.25, 0.5, 0.75)], np.float32)
    cx, cy = np.float32(w // 2 + 0.25), np.float32(h // 2 - 0.5)
    lo_x, hi_x, lo_y, hi_y = u, np.float32(w - 1) - u, u, np.float32(h - 1) - u
    full = lambda v: np.full_like(u, v)  # noqa: E731
    pts = [np.stack(p, 1) for p in ((lo_x, full(cy)), (hi_x, full(cy)), (full(cx), lo_y), (full(cx), hi_y),
                                    (lo_x, lo_y), (hi_x, lo_y), (lo_x, hi_y), (hi_x, hi_y))]
    return np.concatenate(pts).astype(np.float32)


def main():
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s"], check=True)
    olib = C.CDLL(os.path.join(ROOT, "oracle", "libicg_oracle.so"))
    oa.declare_detect(olib)
    out = {"wf_sizes": np.array(WF_SIZES, np.int32), "min_dists": np.array(MIN_DISTS), "wf_n": np.array([WF_N], np.int32)}
    for k, (W, H) in enumerate(WF_SIZES):
        img = frame(100 + k, W, H)
        mask = np.full((H, W), 255, np.uint8)
        cv2.circle(mask, (W // 2, H // 2), max(2, min(W, H) // 6), 0, cv2.FILLED)
        cv2.circle(mask, (W // 5, H // 4), max(2, min(W, H) // 8), 0, cv2.FILLED)
        c = f"wf_{W}x{H}"
        out[c + "_crc"], out[c + "_eig_crc"], out[c + "_mask"] = crc(img), crc(cv2.cornerMinEigenVal(img, 3, ksize=3)), mask
        for tag, m in (("nomask", None), ("mask", mask)):
            for j, md in enumerate(MIN_DISTS):
                pts = gftt(img, WF_N, md, m)
                out[f"{c}_{tag}_md{j}_pts"], out[f"{c}_{tag}_md{j}_sub"] = pts, subpix(img, pts)
    for name, img in tie_images().items():
        c = f"tie_{name}"
        n = len(gftt(img, 0, TIE_MD))
        out[c + "_crc"], out[c + "_n"], out[c + "_mcs"] = crc(img), np.array([n], np.int32), np.array([1, n - 1, n, n + 1], np.int32)
        for m in (1, n - 1, n, n + 1):
            out[f"{c}_mc{m}_pts"] = gftt(img, m, TIE_MD)
    # masks
    img = frame(140, 97, 65)
    img[20:44, 30:60] = 117  # flat region
    out["mask_img_crc"] = crc(img)
    best = gftt(img, 1, 5.0)[0].astype(int)
    masks = {"empty": np.zeros_like(img), "best_pixel": np.zeros_like(img), "other_pixel": np.zeros_like(img), "border": np.zeros_like(img),
             "flat": np.zeros_like(img)}
    masks["best_pixel"][best[1], best[0]] = 255
    eig = cv2.cornerMinEigenVal(img, 3, ksize=3)
    masks["other_pixel"][best[1], best[0] + 1] = 255  # a neighbour of the strongest corner is no 3x3 maximum
    assert eig[best[1], best[0] + 1] < eig[best[1], best[0]]
    masks["border"][[0, -1], :] = 255
    masks["border"][:, [0, -1]] = 255
    masks["flat"][23:41, 33:57] = 255
    for name, m in masks.items():
        out[f"mask_{name}_mask"], out[f"mask_{name}_pts"] = m, gftt(img, MASK_N, 5.0, m)
    # flat corner
    out["flat_pts"] = np.array([[45.0, 32.0], [44.25, 31.5]], np.float32)
    out["flat_sub"] = subpix(img, out["flat_pts"])
    # blocks
    for W, H in GRIDS:
        c = f"blk_{W}x{H}"
        rois, quota, md, _ = block_rois(W, H, 300)
        st = synth.KltStream(W, H, 300, 77)
        crcs, idx, pts, sub, tie = [], [], [], [], []
        for t in range(N_FRAMES):
            f = st.frame(t)
            crcs.append(zlib.crc32(f.tobytes()))
            for b, (x0, y0, w, h) in enumerate(rois):
                p = oa.good_features(olib, f, quota, 0.01, float(md), roi=(x0, y0, w, h))
                blk = np.ascontiguousarray(f[y0:y0 + h, x0:x0 + w])
                s = subpix(blk, p)
                idx.append(np.tile([t, b], (len(p), 1))), pts.append(p), sub.append(s), tie.append(ties(blk, p, s))
        out[c + "_crc"] = np.array(crcs, np.uint64)
        out[c + "_idx"], out[c + "_pts"] = np.concatenate(idx).astype(np.int16), np.concatenate(pts).astype(np.int16)
        out[c + "_sub"], out[c + "_tie"] = np.concatenate(sub), np.concatenate(tie)
        f = st.frame(0)
        pb, pp, ps, pt = [], [], [], []
        for b in (len(rois) // 2, len(rois) - 1):
            x0, y0, w, h = rois[b]
            blk = np.ascontiguousarray(f[y0:y0 + h, x0:x0 + w])
            p = placed(w, h)
            s = subpix(blk, p)
            pb.append(np.full(len(p), b, np.int16)), pp.append(p), ps.append(s), pt.append(ties(blk, p, s))
        out[c + "_placed_blk"], out[c + "_placed_pts"] = np.concatenate(pb), np.concatenate(pp)
        out[c + "_placed_sub"], out[c + "_placed_tie"] = np.concatenate(ps), np.concatenate(pt)
        print(c, len(out[c + "_pts"]), "corners,", int(out[c + "_tie"].sum()), "ties;", len(out[c + "_placed_pts"]), "placed,",
              int(out[c + "_placed_tie"].sum()), "ties")
    # getRectSubPix patches
    img = frame(150, 32, 24)
    q = np.arange(0, 32 * 4) / 4.0
    centres = [(x, y) for y in q[q < 24] for x in q if min(x, 31 - x, y, 23 - y) <= 7]
    out["rs_crc"] = crc(img)
    out["rs_centres"] = np.array(centres, np.float32)
    out["rs_patch_crc"] = np.array([zlib.crc32(cv2.getRectSubPix(img, (13, 13), (float(x), float(y)), patchType=cv2.CV_32F).tobytes())
                                    for x, y in out["rs_centres"]], np.uint32)
    path = os.path.join(HERE, "detect_edges_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes; cv2", cv2.__version__)


if __name__ == "__main__":
    main()
