"""GPU tests of the detection kernels (csrc/detect.cu) at every ROI edge, width / height residue and tie, against the cv2 edge goldens
(tests/golden/make_detect_edges_golden.py) and the CPU oracle.  Bars: corner lists identical in content and order; sub-pixel positions
within 1e-3 px, except at the golden's ties (corners whose cv2 result moves by more than 5e-4 px under a 1e-4 px nudge of the start
point or a 1 % change of epsilon; see the golden script)."""
import numpy as np
import pytest

from ic_gvins_b200 import IcgError
from ic_gvins_b200.detect import Detector, block_rois
from tests import oracle_api as oa
from tests.test_oracle_detect_edges import G, GRIDS, MASKS, TIES, WF, assert_subpix, mask_frame, stream, tie_frame, wf_frame

pytestmark = pytest.mark.gpu
DET_MAX_CELLS = 1024  # min-distance grid cells per block (detect.cu)
DET_MAX_CAND = 16384  # NMS candidates per block (detect.cu)


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_detect(oracle)
    return oracle


@pytest.fixture(scope="module")
def detectors():
    cache = {}

    def get(W, H, cap=256, max_blocks=32):
        if (W, H, cap, max_blocks) not in cache:
            cache[(W, H, cap, max_blocks)] = Detector(W, H, max_blocks=max_blocks, max_corners_per_block=cap)
        return cache[(W, H, cap, max_blocks)]
    yield get
    for d in cache.values():
        d.close()


def grid_cells(w, h, md):
    cell = int(np.rint(md))
    return -(-w // cell) * -(-h // cell)


def nms_candidates(eig, mask):
    """goodFeaturesToTrack's candidate count (threshold at 1 % of the masked maximum, 3x3 maximum, interior, mask) from an eig map"""
    m = np.ones(eig.shape, bool) if mask is None else mask != 0
    thr = np.float32(float(eig[m].max()) * 0.01) if m.any() else np.float32(0)
    e = np.where(eig > thr, eig, np.float32(0))
    c = e[1:-1, 1:-1]
    mx = np.max([e[1 + j:e.shape[0] - 1 + j, 1 + i:e.shape[1] - 1 + i] for j in (-1, 0, 1) for i in (-1, 0, 1)], axis=0)
    return int(((c > thr) & (c == mx) & m[1:-1, 1:-1]).sum())


def oracle_ties(olib, img, pts, roi=None):
    """the golden's tie rule applied to the oracle (for seeded cases without a cv2 golden): start nudged 1e-4 px along each axis"""
    H, W = img.shape
    x0, y0, w, h = roi or (0, 0, W, H)
    ref = oa.corner_subpix(olib, img, pts, roi)
    tie = np.zeros(len(pts), bool)
    for d in ((1e-4, 0), (0, 1e-4), (-1e-4, 0), (0, -1e-4)):
        q = pts + np.float32(d)
        inside = (q[:, 0] >= 0) & (q[:, 0] < w) & (q[:, 1] >= 0) & (q[:, 1] < h)
        tie |= inside & (np.abs(oa.corner_subpix(olib, img, np.where(inside[:, None], q, pts), roi) - ref).max(axis=1) > 5e-4)
    return ref, tie


@pytest.mark.parametrize("W,H", WF, ids=[f"{w}x{h}" for w, h in WF])
def test_whole_frame_lists_and_subpix_vs_cv2(detectors, olib, W, H):
    """whole frames as one block; where the frame exceeds a capacity of the kernels (more than DET_MAX_CAND candidates, or a min-distance
    grid over DET_MAX_CELLS cells), the call must raise instead (its recovery is tested below)"""
    img = wf_frame(W, H)
    d = detectors(W, H)
    c = f"wf_{W}x{H}"
    n = int(G["wf_n"][0])
    eig = oa.min_eig_roi(olib, img, (0, 0, W, H))
    n_checked = 0
    for tag, m in (("nomask", None), ("mask", G[c + "_mask"])):
        too_many = nms_candidates(eig, m) > DET_MAX_CAND
        for j, md in enumerate(G["min_dists"]):
            if too_many or grid_cells(W, H, md) > DET_MAX_CELLS:
                with pytest.raises(IcgError):
                    d.goodFeaturesToTrack(img, n, 0.01, float(md), mask=m)
                continue
            pts = d.goodFeaturesToTrack(img, n, 0.01, float(md), mask=m)
            assert np.array_equal(pts, G[f"{c}_{tag}_md{j}_pts"]), (tag, md)
            assert_subpix(d.cornerSubPix(img, pts), G[f"{c}_{tag}_md{j}_sub"], W, H, f"{tag} minDistance {md}")
            n_checked += 1
    assert n_checked >= 2 or nms_candidates(eig, None) > DET_MAX_CAND  # 752x480 has 17238 candidates: the capacity path only


@pytest.mark.parametrize("name", TIES)
def test_tie_break_order_vs_cv2(detectors, name):
    img = tie_frame(name)
    d = detectors(64, 48, cap=1024)
    for m in G[f"tie_{name}_mcs"]:
        want = G[f"tie_{name}_mc{m}_pts"] if m > 0 else np.zeros((0, 2), np.float32)  # the library: maxCorners <= 0 gives no corners
        assert np.array_equal(d.goodFeaturesToTrack(img, int(m), 0.01, 1.5), want), m


@pytest.mark.parametrize("name", MASKS)
def test_masks_vs_cv2(detectors, name):
    img = mask_frame()
    d = detectors(97, 65)
    assert np.array_equal(d.goodFeaturesToTrack(img, 40, 0.01, 5.0, mask=G[f"mask_{name}_mask"]), G[f"mask_{name}_pts"])
    if name == "flat":
        assert np.array_equal(d.cornerSubPix(img, G["flat_pts"]), G["flat_pts"])


@pytest.mark.parametrize("W,H", GRIDS, ids=[f"{w}x{h}" for w, h in GRIDS])
def test_block_grid_vs_cv2_and_oracle(detectors, W, H):
    """detect_blocks on the reference's grid over 20 stream frames: integer selection identical to the oracle, sub-pixel within 1e-3 px
    of cv2.cornerSubPix on the block copy"""
    c = f"blk_{W}x{H}"
    rois, quota, md, _ = block_rois(W, H, 300)
    d = detectors(W, H, cap=64)
    idx, pts, ref, tie = G[c + "_idx"], G[c + "_pts"], G[c + "_sub"], G[c + "_tie"]
    n_checked = 0
    for t, f in stream(W, H):
        raw = d.detect_blocks(f, rois, [quota] * len(rois), 0.01, float(md), None, subpix=False)
        sub = d.detect_blocks(f, rois, [quota] * len(rois), 0.01, float(md), None, subpix=True)
        for b, roi in enumerate(rois):
            sel = (idx[:, 0] == t) & (idx[:, 1] == b)
            assert np.array_equal(raw[b], pts[sel].astype(np.float32)), (t, b)
            keep = ~tie[sel]
            assert_subpix(sub[b][keep], ref[sel][keep], roi[2], roi[3], f"frame {t} block {b}")
            n_checked += int(keep.sum())
    assert n_checked > 0.9 * len(pts)


@pytest.mark.parametrize("W,H", GRIDS, ids=[f"{w}x{h}" for w, h in GRIDS])
def test_placed_corners_vs_cv2(detectors, W, H):
    """corners 0-7 px from every block edge and corner, refined by the cornerSubPix drop-in on the block copy"""
    c = f"blk_{W}x{H}"
    rois, _, _, _ = block_rois(W, H, 300)
    _, f = next(stream(W, H))
    blk, pts, ref, tie = G[c + "_placed_blk"], G[c + "_placed_pts"], G[c + "_placed_sub"], G[c + "_placed_tie"]
    for b in np.unique(blk):
        x0, y0, w, h = rois[b]
        sel = blk == b
        d = detectors(w, h, cap=int(sel.sum()), max_blocks=1)
        got = d.cornerSubPix(np.ascontiguousarray(f[y0:y0 + h, x0:x0 + w]), pts[sel])
        keep = ~tie[sel]
        assert_subpix(got[keep], ref[sel][keep], w, h, f"block {b}")


def sweep_rois(W, H, rng):
    """ROIs touching each frame edge and corner, with w % 32 in {0, 1, 31}, h % 16 in {0, 1, 15}, and 3x3, 3xN, Nx3 ROIs"""
    rois = []
    for w, h in ((64, 48), (65, 49), (63, 47), (96, 33), (33, 31), (3, 3), (3, 40), (40, 3), (97, 17)):
        for ax, ay in ((0, 0), (1, 0), (0, 1), (1, 1), (0.5, 0), (0.5, 1), (0, 0.5), (1, 0.5), (rng.random(), rng.random())):
            rois.append((int(round(ax * (W - w))), int(round(ay * (H - h))), w, h))
    return rois


def test_seeded_roi_sweep_vs_oracle(detectors, olib):
    """every ROI of the sweep in one call, mixed max_corners: <= 0 gives no corners, above the handle's cap is clamped to it"""
    from datagen import synth_klt as synth
    W, H, cap = 301, 207, 24
    rng = np.random.default_rng(11)
    img = synth.render_frame(synth.make_texture(W, H, 61), 0, W, H)
    mask = np.full((H, W), 255, np.uint8)
    mask[rng.random((H, W)) < 0.05] = 0
    rois = sweep_rois(W, H, rng)
    mcs = [[0, -3, 5, cap, cap + 7, 100][k % 6] for k in range(len(rois))]
    d = Detector(W, H, max_blocks=len(rois), max_corners_per_block=cap)
    try:
        for m, md in ((None, 3.0), (mask, 5.0)):
            raw = d.detect_blocks(img, rois, mcs, 0.01, md, m, subpix=False)
            sub = d.detect_blocks(img, rois, mcs, 0.01, md, m, subpix=True)
            n_total = 0
            for roi, mc, r, s in zip(rois, mcs, raw, sub):
                if mc <= 0:
                    assert len(r) == 0 and len(s) == 0
                    continue
                want = oa.good_features(olib, img, min(mc, cap), 0.01, md, m, roi=roi)
                assert np.array_equal(r, want), (roi, mc)
                ref, tie = oracle_ties(olib, img, want, roi)
                assert_subpix(s[~tie], ref[~tie], roi[2], roi[3], f"ROI {roi}")
                n_total += len(r)
            assert n_total > 200
    finally:
        d.close()


def test_corner_subpix_drop_in_on_frame_edges(olib):
    """caller-given corners on and next to the frame edge, n equal to the handle's cap"""
    from datagen import synth_klt as synth
    W, H, cap = 97, 65, 64
    img = synth.render_frame(synth.make_texture(W, H, 62), 0, W, H)
    rng = np.random.default_rng(12)
    u = rng.integers(0, 3, cap) + rng.integers(0, 4, cap) * np.float32(0.25)
    along = rng.random(cap)
    side = np.arange(cap) % 4
    x = np.where(side == 0, u, np.where(side == 1, W - 1 - u, along * (W - 1)))
    y = np.where(side == 2, u, np.where(side == 3, H - 1 - u, along * (H - 1)))
    pts = np.stack([x, y], 1).astype(np.float32)
    d = Detector(W, H, max_blocks=1, max_corners_per_block=cap)
    try:
        got = d.cornerSubPix(img, pts)
    finally:
        d.close()
    ref, tie = oracle_ties(olib, img, pts)
    assert_subpix(got[~tie], ref[~tie], W, H, "frame-edge corners")
    assert (~tie).sum() > cap // 2


def test_detect_blocks_dev_equals_per_frame_calls():
    """icg_detect_blocks_dev on several device-resident 752x480 frames in one call == icg_detect_blocks frame by frame"""
    import torch
    W, H, NF = 752, 480, 4
    rois, quota, md, _ = block_rois(W, H, 300)
    frames = [f for _, f in zip(range(NF), stream(W, H))]
    want = [quota - (b % 3) for b in range(len(rois))]
    d1 = Detector(W, H, max_blocks=len(rois), max_corners_per_block=64)
    dN = Detector(W, H, max_blocks=NF * len(rois), max_corners_per_block=64, max_roi_pixels=max(w * h for _, _, w, h in rois))
    try:
        ref = [d1.detect_blocks(f, rois, want, 0.01, float(md), None, subpix=True) for _, f in frames]
        dev = torch.from_numpy(np.stack([f for _, f in frames])).cuda()
        torch.cuda.synchronize()
        got = dN.detect_blocks_dev(NF, dev.data_ptr(), W, W * H, rois, want, 0.01, float(md))
    finally:
        d1.close()
        dN.close()
    for f in range(NF):
        for b in range(len(rois)):
            assert np.array_equal(got[f][b], ref[f][b]), (f, b)


def test_capacity_errors_then_recovery(olib):
    """more than DET_MAX_CAND NMS candidates in a block, and a min-distance grid over DET_MAX_CELLS: IcgError, then the same handle
    returns correct results on its next call"""
    from datagen import synth_klt as synth
    W, H = 640, 480
    noisy = np.random.default_rng(13).integers(0, 256, (H, W)).astype(np.uint8)
    img = synth.render_frame(synth.make_texture(W, H, 63), 0, W, H)
    roi = (0, 0, 160, 120)  # minDistance 5: 32 x 24 cells
    d = Detector(W, H, max_blocks=2, max_corners_per_block=64)
    try:
        want = oa.good_features(olib, img, 40, 0.01, 5.0, roi=roi)
        with pytest.raises(IcgError):
            d.detect_blocks(noisy, [(0, 0, W, H)], [64], 0.0, 0.0)
        assert np.array_equal(d.detect_blocks(img, [roi], [40], 0.01, 5.0, subpix=False)[0], want)
        with pytest.raises(IcgError):
            d.detect_blocks(img, [roi], [40], 0.01, 1.0)
        assert np.array_equal(d.detect_blocks(img, [roi], [40], 0.01, 5.0, subpix=False)[0], want)
    finally:
        d.close()
