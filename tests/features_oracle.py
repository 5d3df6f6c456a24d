"""CPU restatement of Tracking::featuresDetection (IG/tracking/tracking.cc:576-685) up to the append into the reference's lists: the block
grid of Tracking::Tracking (:66-85), the gate (:579-582), the per-block counts (:591-606), the occupancy mask (:609-620), per-block detection
(:627-656, the C oracle's ROI-exact icgo_detect_block) and the shift to frame coordinates (:669-675).  Tests only."""
import math

import numpy as np

from tests import oracle_api as oa

TRACK_BLOCK_SIZE = 200.0  # IG/tracking/tracking.h:112


def _lround(v: float) -> int:
    """C lround / round: half away from zero"""
    return int(math.floor(abs(v) + 0.5)) * (1 if v >= 0 else -1)


def grid(W, H, max_features):
    """(cols, rows, bw, bh, quota, min_dist) exactly as Tracking::Tracking computes them"""
    cols, rows = _lround(W / TRACK_BLOCK_SIZE), _lround(H / TRACK_BLOCK_SIZE)
    bw, bh = W // cols, H // rows
    quota = _lround(float(max_features) / float(cols * rows))
    min_dist = int(_lround(TRACK_BLOCK_SIZE / math.sqrt(quota * 1.5)))
    return cols, rows, bw, bh, quota, min_dist


def rois(W, H, max_features):
    """tracking.cc:631-645: every block but the last is shrunk by 5 px"""
    cols, rows, bw, bh, _, _ = grid(W, H, max_features)
    out = []
    for k in range(cols * rows):
        c, r = k % cols, k // cols
        s = 5 if k != cols * rows - 1 else 0
        out.append((c * bw, r * bh, bw - s, bh - s))
    return out


def block_index(pts, cols, rows, bw, bh):
    """int(y / (float) bh) * cols + int(x / (float) bw) in float32 with truncation toward zero (tracking.cc:598-605); -1 where the index
    falls outside [0, cols * rows) (the reference writes past its array there)"""
    p = np.asarray(pts, np.float32).reshape(-1, 2)
    with np.errstate(invalid="ignore"):
        qx = np.clip(p[:, 0] / np.float32(bw), -1e9, 1e9)
        qy = np.clip(p[:, 1] / np.float32(bh), -1e9, 1e9)
    ok = np.isfinite(qx) & np.isfinite(qy)
    k = np.trunc(np.where(ok, qy, 0)).astype(np.int64) * cols + np.trunc(np.where(ok, qx, 0)).astype(np.int64)
    return np.where(ok & (k >= 0) & (k < cols * rows), k, -1)


def counts(feat_xy, new_xy, cols, rows, bw, bh):
    k = np.concatenate([block_index(feat_xy, cols, rows, bw, bh), block_index(new_xy, cols, rows, bw, bh)])
    return np.bincount(k[k >= 0], minlength=cols * rows)[:cols * rows].astype(np.int64)


def disc_mask(W, H, pts, radius, mask=None):
    """cv::circle(mask, cv::Point(pt), radius, 0, FILLED) for every point: the pixels with (x - cx)^2 + (y - cy)^2 <= radius^2, clipped to the
    frame, with cv::Point(Point2f) = cvRound (round half to even) of each coordinate"""
    mask = np.full((H, W), 255, np.uint8) if mask is None else mask
    r = int(radius)
    for x, y in np.asarray(pts, np.float32).reshape(-1, 2):
        if not (np.isfinite(x) and np.isfinite(y)) or abs(float(x)) > 2 ** 30 or abs(float(y)) > 2 ** 30:
            continue
        cx, cy = int(np.rint(np.float64(x))), int(np.rint(np.float64(y)))
        x0, x1, y0, y1 = max(0, cx - r), min(W - 1, cx + r), max(0, cy - r), min(H - 1, cy + r)
        if x0 > x1 or y0 > y1:
            continue
        yy, xx = np.mgrid[y0:y1 + 1, x0:x1 + 1]
        sub = mask[y0:y1 + 1, x0:x1 + 1]
        sub[(xx - cx) ** 2 + (yy - cy) ** 2 <= r * r] = 0
    return mask


def features_detection(olib, img, feat_xy, new_xy, n_ref=None, ismask=True, max_features=300):
    """dict(skipped, counts, mask, corners): corners (n, 2) float32 in frame coordinates and block order; skipped frames have no counts,
    mask or corners (the reference returns at :581)."""
    H, W = img.shape
    feat_xy = np.asarray(feat_xy, np.float32).reshape(-1, 2)
    new_xy = np.asarray(new_xy, np.float32).reshape(-1, 2)
    n_ref = len(new_xy) if n_ref is None else int(n_ref)
    if len(feat_xy) + n_ref > max_features - 5:
        return dict(skipped=True, counts=None, mask=None, corners=None)
    cols, rows, bw, bh, quota, min_dist = grid(W, H, max_features)
    cnt = counts(feat_xy, new_xy, cols, rows, bw, bh)
    mask = np.full((H, W), 255, np.uint8)
    if ismask:
        disc_mask(W, H, feat_xy, min_dist, mask)
        disc_mask(W, H, new_xy, min_dist, mask)
    out = []
    for k, roi in enumerate(rois(W, H, max_features)):
        want = quota - int(cnt[k])
        if want <= 0:
            continue
        p = oa.detect_block(olib, img, mask, roi, want, 0.01, float(min_dist))
        if len(p):
            c, r = k % cols, k // cols
            out.append(np.stack([np.float32(c * bw) + p[:, 0], np.float32(r * bh) + p[:, 1]], axis=1).astype(np.float32))
    corners = np.concatenate(out, axis=0) if out else np.zeros((0, 2), np.float32)
    return dict(skipped=False, counts=cnt, mask=mask, corners=corners)
