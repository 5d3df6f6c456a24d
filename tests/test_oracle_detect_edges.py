"""Pin the detection oracle (oracle/detect_ref.c) to the cv2 edge goldens (tests/golden/make_detect_edges_golden.py).  CPU only.
Bars: eig maps and getRectSubPix patches bit-exact (CRC), corner lists identical in content and order, every sub-pixel position
within 1e-3 px of cv2 (ties included)."""
import os
import zlib

import numpy as np
import pytest

from datagen import synth_klt as synth
from ic_gvins_b200.detect import block_rois
from tests import oracle_api as oa

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "detect_edges_golden.npz"))
WF = [tuple(int(v) for v in s) for s in G["wf_sizes"]]
TIES = ["checker4", "checker7", "checker8", "stripes"]
MASKS = ["empty", "best_pixel", "other_pixel", "border", "flat"]
GRIDS = [(1280, 560), (752, 480), (997, 413)]
SUB_PX = 1e-3


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_detect(oracle)
    return oracle


def crc(a):
    return zlib.crc32(np.ascontiguousarray(a).tobytes())


def wf_frame(W, H):
    img = synth.render_frame(synth.make_texture(W, H, 100 + WF.index((W, H))), 0, W, H)
    assert crc(img) == int(G[f"wf_{W}x{H}_crc"][0])
    return img


def tie_frame(name):
    yy, xx = np.mgrid[0:48, 0:64]
    if name == "stripes":
        img = np.where((xx % 6 < 2) | (yy % 5 < 2), 230, 30).astype(np.uint8)
    else:
        p = int(name[len("checker"):])
        img = (((2 * xx // p) + (2 * yy // p)) % 2 * 200 + 20).astype(np.uint8)
    assert crc(img) == int(G[f"tie_{name}_crc"][0])
    return img


def mask_frame():
    img = synth.render_frame(synth.make_texture(97, 65, 140), 0, 97, 65)
    img[20:44, 30:60] = 117
    assert crc(img) == int(G["mask_img_crc"][0])
    return img


def edge_dist(xy, w, h):
    """distance of each point to the nearest ROI edge, for failure messages"""
    xy = np.asarray(xy, np.float64).reshape(-1, 2)
    return np.minimum.reduce([xy[:, 0], w - 1 - xy[:, 0], xy[:, 1], h - 1 - xy[:, 1]])


def assert_subpix(got, want, w, h, what):
    d = np.abs(np.asarray(got) - want).max(axis=1) if len(want) else np.zeros(0)
    bad = np.nonzero(d > SUB_PX)[0]
    assert len(bad) == 0, (f"{what}: {len(bad)} of {len(d)} corners more than {SUB_PX} px from cv2 (worst {d.max():.4g} px); first: "
                           + ", ".join(f"start {tuple(want[i])} got {tuple(got[i])} at {edge_dist(want[i], w, h)[0]:.2f} px from an edge"
                                       for i in bad[:4]))


@pytest.mark.parametrize("W,H", WF, ids=[f"{w}x{h}" for w, h in WF])
def test_whole_frame_eig_lists_and_subpix(olib, W, H):
    img = wf_frame(W, H)
    c = f"wf_{W}x{H}"
    assert crc(oa.min_eig_roi(olib, img, (0, 0, W, H))) == int(G[c + "_eig_crc"][0])
    for tag, m in (("nomask", None), ("mask", G[c + "_mask"])):
        for j, md in enumerate(G["min_dists"]):
            pts = oa.good_features(olib, img, int(G["wf_n"][0]), 0.01, float(md), m)
            want = G[f"{c}_{tag}_md{j}_pts"]
            assert np.array_equal(pts, want), (tag, md)
            sub = oa.corner_subpix(olib, img, pts)
            ref = G[f"{c}_{tag}_md{j}_sub"]
            assert_subpix(sub, ref, W, H, f"{tag} minDistance {md}")


@pytest.mark.parametrize("name", TIES)
def test_tie_break_order(olib, name):
    img = tie_frame(name)
    n = int(G[f"tie_{name}_n"][0])
    assert len(oa.good_features(olib, img, 0, 0.01, 1.5)) == n  # maxCorners 0 = no limit: the output buffer holds every candidate
    for m in G[f"tie_{name}_mcs"]:
        assert np.array_equal(oa.good_features(olib, img, int(m), 0.01, 1.5), G[f"tie_{name}_mc{m}_pts"]), m


@pytest.mark.parametrize("name", MASKS)
def test_masks(olib, name):
    img = mask_frame()
    pts = oa.good_features(olib, img, 40, 0.01, 5.0, G[f"mask_{name}_mask"])
    assert np.array_equal(pts, G[f"mask_{name}_pts"])
    assert len(pts) == (1 if name == "best_pixel" else 0)


def test_flat_corner_unchanged(olib):
    img = mask_frame()
    sub = oa.corner_subpix(olib, img, G["flat_pts"])
    assert np.array_equal(sub, G["flat_sub"]) and np.array_equal(sub, G["flat_pts"])


def test_rect_subpix_patches_bit_exact(olib):
    img = synth.render_frame(synth.make_texture(32, 24, 150), 0, 32, 24)
    assert crc(img) == int(G["rs_crc"][0])
    bad = [tuple(c) for c, want in zip(G["rs_centres"], G["rs_patch_crc"]) if crc(oa.rect_subpix(olib, img, c)) != int(want)]
    top_right = [c for c in bad if c[0] > 31 - 7 and c[1] < 7]
    assert not bad, f"{len(bad)} of {len(G['rs_centres'])} patches differ from cv2 ({len(top_right)} at the top-right corner); first {bad[:6]}"


def stream(W, H):
    st = synth.KltStream(W, H, 300, 77)
    crcs = G[f"blk_{W}x{H}_crc"]
    for t in range(len(crcs)):
        f = st.frame(t)
        assert crc(f) == int(crcs[t])
        yield t, f


@pytest.mark.parametrize("W,H", GRIDS, ids=[f"{w}x{h}" for w, h in GRIDS])
def test_block_grid_stream_subpix(olib, W, H):
    """every corner of every block of 20 stream frames within 1e-3 px of cv2.cornerSubPix on the block copy"""
    c = f"blk_{W}x{H}"
    rois, quota, md, _ = block_rois(W, H, 300)
    idx, pts, ref = G[c + "_idx"], G[c + "_pts"], G[c + "_sub"]
    for t, f in stream(W, H):
        for b, roi in enumerate(rois):
            sel = (idx[:, 0] == t) & (idx[:, 1] == b)
            p = oa.good_features(olib, f, quota, 0.01, float(md), roi=roi)
            assert np.array_equal(p, pts[sel].astype(np.float32)), (t, b)
            sub = oa.corner_subpix(olib, f, p, roi=roi)
            assert_subpix(sub, ref[sel], roi[2], roi[3], f"frame {t} block {b}")
            assert np.array_equal(oa.detect_block(olib, f, None, roi, quota, 0.01, float(md)), sub)


@pytest.mark.parametrize("W,H", GRIDS, ids=[f"{w}x{h}" for w, h in GRIDS])
def test_placed_corners_at_block_edges(olib, W, H):
    c = f"blk_{W}x{H}"
    rois, _, _, _ = block_rois(W, H, 300)
    _, f = next(stream(W, H))
    blk, pts, ref = G[c + "_placed_blk"], G[c + "_placed_pts"], G[c + "_placed_sub"]
    for b in np.unique(blk):
        roi = rois[b]
        sel = blk == b
        assert_subpix(oa.corner_subpix(olib, f, pts[sel], roi=roi), ref[sel], roi[2], roi[3], f"block {b}")
