"""CPU: the featuresDetection restatement (tests/features_oracle.py) that the device path is compared with.  The occupancy mask is pinned
against cv2.circle (tests/golden/mask_golden.npz); the counts, the aliasing of the block index and the gate against hand-made cases
(IG/tracking/tracking.cc:579-620)."""
import os

import numpy as np
import pytest

from tests import features_oracle as fo

W, H = 1280, 560
GRID = fo.grid(W, H, 300)


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "mask_golden.npz"))


def test_grid_of_the_reference_frame():
    assert GRID == (6, 3, 213, 186, 17, 40)
    assert fo.rois(W, H, 300)[0] == (0, 0, 208, 181) and fo.rois(W, H, 300)[17] == (1065, 372, 213, 186)


def test_disc_mask_equals_cv2_circle_golden(golden):
    names = sorted({k[:-5] for k in golden.files if k.endswith("_mask")})
    assert len(names) >= 17
    radii = set()
    for n in names:
        w, h = (int(v) for v in golden[n + "_size"])
        r = int(golden[n + "_r"])
        radii.add(r)
        got = fo.disc_mask(w, h, golden[n + "_pts"], r)
        assert np.array_equal(got, golden[n + "_mask"]), n
    assert radii == {1, 2, 17, 40}


def _idx(x, y):
    return int(fo.block_index([(x, y)], *GRID[:4])[0])


def test_block_index_on_boundaries_and_one_ulp_below():
    cols, rows, bw, bh = GRID[:4]
    below = lambda v: float(np.nextafter(np.float32(v), np.float32(0)))  # noqa: E731
    assert _idx(0.0, 0.0) == 0
    assert _idx(213.0, 0.0) == 1 and _idx(below(213.0), 0.0) == 0
    assert _idx(0.0, 186.0) == cols and _idx(0.0, below(186.0)) == 0
    assert _idx(426.0, 372.0) == 2 * cols + 2 and _idx(below(426.0), below(372.0)) == cols + 1
    assert _idx(1277.9, 557.9) == 17
    # rows * bh = 558 < H: the last two pixel rows of the frame are past the grid's last row (the reference writes out of bounds): dropped
    assert _idx(100.0, 558.0) == -1


def test_block_index_aliasing_and_dropping():
    cols = GRID[0]
    # undistorted points beyond cols * bw = 1278: col == cols lands in the next row's first block (the reference's flat index)
    assert _idx(1278.0, 10.0) == cols and _idx(1290.5, 200.0) == 2 * cols
    # ... and past the last row it leaves the grid: dropped
    assert _idx(1290.5, 400.0) == -1
    # truncation toward zero: slightly negative coordinates count into column / row 0
    assert _idx(-5.0, -5.0) == 0 and _idx(-212.9, 3.0) == 0
    # col == -1 in row 1 aliases into row 0's last block; col == -1 in row 0 is outside the grid
    assert _idx(-300.0, 200.0) == cols - 1 and _idx(-300.0, 10.0) == -1
    assert _idx(1e6, 10.0) == -1 and _idx(10.0, -1e7) == -1 and _idx(10.0, 1e30) == -1 and _idx(float("nan"), 5.0) == -1


def test_counts_include_both_lists():
    feat = [(10.0, 10.0), (1290.5, 200.0), (1e6, 1e6)]
    new = [(213.0, 0.0), (10.0, 10.0), (-300.0, 200.0)]
    c = fo.counts(feat, new, *GRID[:4])
    expect = np.zeros(18, np.int64)
    expect[0], expect[1], expect[5], expect[12] = 2, 1, 1, 1
    assert np.array_equal(c, expect)


class _NoDetect:
    """stands in for the C oracle where a test only looks at the gate, counts and mask"""


def test_gate_uses_n_ref_not_the_new_list(monkeypatch):
    monkeypatch.setattr(fo.oa, "detect_block", lambda *a, **k: np.zeros((0, 2), np.float32))
    img = np.zeros((H, W), np.uint8)
    new = np.array([(100.0 + 3 * i, 100.0) for i in range(10)], np.float32)
    feat = np.array([(600.0, 300.0)] * 4, np.float32)
    # |feat| + n_ref > max_features - 5 skips the frame; n_ref = pts2d_ref_.size() may differ from |pts2d_new_| (tracking.cc:557, 220)
    assert fo.features_detection(_NoDetect, img, feat, new, n_ref=292)["skipped"]
    r = fo.features_detection(_NoDetect, img, feat, new, n_ref=291)
    assert not r["skipped"] and r["counts"].sum() == 14
    assert not fo.features_detection(_NoDetect, img, [], new, n_ref=0)["skipped"]
    assert fo.features_detection(_NoDetect, img, np.zeros((296, 2), np.float32), [], n_ref=0)["skipped"]
    assert not fo.features_detection(_NoDetect, img, np.zeros((295, 2), np.float32), [], n_ref=0)["skipped"]
    # ismask selects the mask only; the counts are the same either way
    r0 = fo.features_detection(_NoDetect, img, feat, new, n_ref=0, ismask=False)
    assert np.array_equal(r0["counts"], r["counts"]) and (r0["mask"] == 255).all() and (r["mask"] == 0).sum() > 0
