"""Host-side mirror of Tracking::featuresDetection (IG/tracking/tracking.cc:576-688): block grid bookkeeping on the host
(as in the reference), Shi-Tomasi + sub-pixel refinement of all blocks in one call into libicgvins_b200.so."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import check, lib, vp

TRACK_BLOCK_SIZE = 200  # IG/tracking/tracking.h:112


def block_grid(width: int, height: int, max_features: int):
    """Tracking::Tracking block setup (tracking.cc:66-85): returns (block_cols, block_rows, bw, bh, per_block_quota, min_dist)."""
    cols = int(round(width / float(TRACK_BLOCK_SIZE)))   # lround
    rows = int(round(height / float(TRACK_BLOCK_SIZE)))
    bw, bh = width // cols, height // rows
    cnt = cols * rows
    quota = int(round(max_features / float(cnt)))
    min_dist = int(round(TRACK_BLOCK_SIZE / np.sqrt(quota * 1.5)))
    return cols, rows, bw, bh, quota, min_dist


def block_rois(width: int, height: int, max_features: int):
    """ROIs of the blocks as featuresDetection forms them (tracking.cc:631-645): every block but the last is shrunk by 5 px."""
    cols, rows, bw, bh, quota, min_dist = block_grid(width, height, max_features)
    rois = []
    for k in range(cols * rows):
        c, r = k % cols, k // cols
        x0, y0, x1, y1 = c * bw, r * bh, c * bw + bw, r * bh + bh
        if k != cols * rows - 1:
            x1 -= 5
            y1 -= 5
        rois.append((x0, y0, x1 - x0, y1 - y0))
    return rois, quota, min_dist, (cols, rows, bw, bh)


class Detector:
    def __init__(self, width: int, height: int, max_blocks: int = 32, max_corners_per_block: int = 64, max_roi_pixels: int = 0, device: int = 0,
                 stream=None):
        self.W, self.H, self.cap, self.max_blocks = width, height, max_corners_per_block, max_blocks
        self._h = vp()
        check(lib().icg_detect_create(C.byref(self._h), width, height, max_blocks, max_corners_per_block, max_roi_pixels or width * height, device,
                                      vp(stream) if stream else None), "icg_detect_create")

    def close(self):
        if getattr(self, "_h", None):
            lib().icg_detect_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def detect_blocks(self, img, rois, max_corners, quality=0.01, min_distance=40.0, mask=None, subpix=True):
        """goodFeaturesToTrack (+ cornerSubPix) on every ROI.  Returns a list of (n_b, 2) float32 arrays (block-local coordinates)."""
        img = np.ascontiguousarray(img, np.uint8)
        n = len(rois)
        r = np.ascontiguousarray(np.array(rois, np.int32).reshape(-1, 4))
        mc = np.ascontiguousarray(np.array(max_corners, np.int32).reshape(-1))
        out = np.zeros((n, self.cap, 2), np.float32)
        cnt = np.zeros(n, np.int32)
        m = np.ascontiguousarray(mask, np.uint8) if mask is not None else None
        check(lib().icg_detect_blocks(self._h, vp(img.ctypes.data), vp(m.ctypes.data) if m is not None else None, self.W, n, vp(r.ctypes.data),
                                      vp(mc.ctypes.data), float(quality), float(min_distance), 1 if subpix else 0, vp(out.ctypes.data),
                                      vp(cnt.ctypes.data)), "icg_detect_blocks")
        return [out[b, :cnt[b]].copy() for b in range(n)]

    def detect_blocks_dev(self, n_frames, dev_img, pitch, frame_stride, rois, max_corners, quality=0.01, min_distance=40.0, dev_mask=None, subpix=True):
        """The same on `n_frames` device-resident frames in ONE call (dev_img: device address of frame 0, row pitch, byte stride between frames).
        Returns out[f][b] = (n, 2) float32 arrays (block-local coordinates)."""
        nb = len(rois)
        r = np.ascontiguousarray(np.array(rois, np.int32).reshape(-1, 4))
        mc = np.ascontiguousarray(np.array(max_corners, np.int32).reshape(-1))
        if mc.size == nb:
            mc = np.tile(mc, n_frames)
        out = np.zeros((n_frames * nb, self.cap, 2), np.float32)
        cnt = np.zeros(n_frames * nb, np.int32)
        check(lib().icg_detect_blocks_dev(self._h, n_frames, vp(dev_img), pitch, frame_stride, vp(dev_mask) if dev_mask else None, nb, vp(r.ctypes.data),
                                          vp(mc.ctypes.data), float(quality), float(min_distance), 1 if subpix else 0, vp(out.ctypes.data),
                                          vp(cnt.ctypes.data)), "icg_detect_blocks_dev")
        return [[out[f * nb + b, :cnt[f * nb + b]].copy() for b in range(nb)] for f in range(n_frames)]

    # cv2.goodFeaturesToTrack(image, maxCorners, qualityLevel, minDistance, mask=...) on the whole frame
    def goodFeaturesToTrack(self, image, maxCorners, qualityLevel, minDistance, mask=None):
        return self.detect_blocks(image, [(0, 0, self.W, self.H)], [maxCorners], qualityLevel, minDistance, mask, subpix=False)[0]

    # cv2.cornerSubPix(image, corners, (5,5), (-1,-1), (COUNT+EPS, 20, 0.01))
    def cornerSubPix(self, image, corners):
        image = np.ascontiguousarray(image, np.uint8)
        c = np.array(corners, np.float32).reshape(-1, 2).copy()
        check(lib().icg_corner_subpix(self._h, vp(image.ctypes.data), self.W, vp(c.ctypes.data), c.shape[0]), "icg_corner_subpix")
        return c

    def features_detection(self, img, max_features=300, mask=None, counts=None):
        """Tracking::featuresDetection's detection step: per-block deficit = quota - existing count (tracking.cc:629), blocks with no
        deficit are skipped, results shifted to frame coordinates and appended in block order (tracking.cc:669-685)."""
        rois, quota, min_dist, _ = block_rois(self.W, self.H, max_features)
        counts = counts if counts is not None else [0] * len(rois)
        want = [max(0, quota - c) for c in counts]
        pts = self.detect_blocks(img, rois, want, 0.01, float(min_dist), mask, subpix=True)
        out = []
        for (x0, y0, _, _), p in zip(rois, pts):
            if len(p):
                out.append(p + np.array([x0, y0], np.float32))
        return np.concatenate(out, axis=0) if out else np.zeros((0, 2), np.float32)

    def features_detection_points(self, img, feat_xy, new_xy, n_ref=None, ismask=True, max_features=300):
        """Tracking::featuresDetection (tracking.cc:579-685) driven by the point lists, in one synchronous call (icg_detect_features):
        feat_xy = the frame's map-point features (undistorted keyPoint()), new_xy = pts2d_new_ (distorted), n_ref = pts2d_ref_.size()
        (default len(new_xy)); the library counts the points per block, draws the occupancy mask when `ismask` and detects the deficits.
        Returns the new corners in frame coordinates (block order), or None when the gate skipped the frame (the caller keeps its lists)."""
        img = np.ascontiguousarray(img, np.uint8)
        a = np.ascontiguousarray(np.asarray(feat_xy, np.float32).reshape(-1, 2))
        b = np.ascontiguousarray(np.asarray(new_xy, np.float32).reshape(-1, 2))
        _, _, _, _, quota, _ = block_grid(self.W, self.H, max_features)
        out = np.zeros((self.max_blocks * self.cap, 2), np.float32)
        n = np.zeros(1, np.int32)
        check(lib().icg_detect_features(self._h, vp(img.ctypes.data), img.strides[0], vp(a.ctypes.data), a.shape[0], vp(b.ctypes.data), b.shape[0],
                                        len(b) if n_ref is None else int(n_ref), 1 if ismask else 0, int(max_features), vp(out.ctypes.data),
                                        vp(n.ctypes.data)), "icg_detect_features")
        return None if n[0] < 0 else out[:n[0]].copy()

    def features_detection_dev(self, n_frames, dev_img, pitch, frame_stride, dev_feat_xy, dev_feat_status, feat_off, dev_new_xy, dev_new_status,
                               new_off, dev_out_xy, dev_out_n, n_ref=None, ismask=None, max_features=300):
        """The same for `n_frames` device-resident frames (icg_detect_features_dev; asynchronous on the handle's stream).  Point lists, status
        bytes (or 0) and outputs are device addresses; feat_off / new_off (n_frames + 1), n_ref and ismask (n_frames) are host sequences.
        Frame f's corners land at dev_out_xy + f * cols * rows * quota * 2 floats, dev_out_n[f] = their number (-1: gated, -2: capacity)."""
        fo = np.ascontiguousarray(np.asarray(feat_off, np.int32).reshape(-1))
        no = np.ascontiguousarray(np.asarray(new_off, np.int32).reshape(-1))
        if fo.size != n_frames + 1 or no.size != n_frames + 1:
            raise ValueError("feat_off and new_off need n_frames + 1 entries")
        nr = np.ascontiguousarray(np.asarray(n_ref, np.int32).reshape(-1)) if n_ref is not None else None
        im = np.ascontiguousarray(np.asarray(ismask, np.uint8).reshape(-1)) if ismask is not None else None
        for x in (nr, im):
            if x is not None and x.size != n_frames:
                raise ValueError("n_ref and ismask need n_frames entries")
        check(lib().icg_detect_features_dev(self._h, n_frames, vp(dev_img), pitch, frame_stride, vp(dev_feat_xy) if dev_feat_xy else None,
                                            vp(dev_feat_status) if dev_feat_status else None, vp(fo.ctypes.data), vp(dev_new_xy) if dev_new_xy else None,
                                            vp(dev_new_status) if dev_new_status else None, vp(no.ctypes.data),
                                            vp(nr.ctypes.data) if nr is not None else None, vp(im.ctypes.data) if im is not None else None,
                                            int(max_features), vp(dev_out_xy), vp(dev_out_n)), "icg_detect_features_dev")

    def mask_dev(self, frame=0):
        """(device address, row pitch) of frame `frame`'s occupancy mask as the last features_detection_* call built it."""
        p, pitch = vp(), C.c_int()
        check(lib().icg_detect_mask_dev(self._h, frame, C.byref(p), C.byref(pitch)), "icg_detect_mask_dev")
        return p.value, pitch.value
