"""Regenerate mask_golden.npz: occupancy masks drawn by cv2.circle(mask, cv::Point(pt), r, 0, cv2.FILLED) (LINE_8, shift 0), the call
Tracking::featuresDetection makes for every tracked point (IG/tracking/tracking.cc:609-620).  cv::Point(Point2f) rounds with cvRound
(round half to even), which Python's round reproduces on the float value.

Cases (one frame each): centres inside the frame, on its border and outside it, half-integer centres (rounding ties), radii 1, 2, 17, 40.
Stored per case: <case>_size (W, H), <case>_r, <case>_pts (float32 n x 2), <case>_mask (u8 H x W).

    python tests/golden/make_mask_golden.py      (needs cv2; pinned against cv2 4.13.0)
"""
import os

import cv2
import numpy as np

W, H = 160, 120


def draw(pts, r):
    m = np.full((H, W), 255, np.uint8)
    for x, y in pts:
        cv2.circle(m, (int(round(float(x))), int(round(float(y)))), int(r), 0, cv2.FILLED)
    return m


def cases():
    rng = np.random.default_rng(20261015)
    border = [(0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1), (W / 2, 0), (0, H / 2), (W - 1, H / 2), (W / 2, H - 1)]
    outside = [(-3, 40), (-20.4, -7.6), (W + 2, 60), (W + 15.5, H + 15.5), (80, -39.6), (80, H + 39.4), (-45, 60), (W + 45, -45)]
    ties = [(10.5, 20.5), (11.5, 21.5), (30.5, 30.0), (31.0, 31.5), (-0.5, 50.5), (W - 0.5, 60.5), (100.5, H - 0.5), (2.5, 3.5)]
    for r in (1, 2, 17, 40):
        inside = rng.uniform([0, 0], [W - 1, H - 1], size=(12, 2))
        yield f"inside_r{r}", r, inside
        yield f"border_r{r}", r, np.array(border, np.float64)
        yield f"outside_r{r}", r, np.array(outside, np.float64)
        yield f"ties_r{r}", r, np.array(ties, np.float64)
    yield "mixed_r40", 40, np.concatenate([rng.uniform([-60, -60], [W + 60, H + 60], size=(30, 2)), np.array(ties, np.float64)])


def main():
    out = {}
    for name, r, pts in cases():
        pts = np.asarray(pts, np.float32)
        out[name + "_size"] = np.array([W, H], np.int32)
        out[name + "_r"] = np.array(r, np.int32)
        out[name + "_pts"] = pts
        out[name + "_mask"] = draw(pts, r)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mask_golden.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out) // 4} masks (cv2 {cv2.__version__})")


if __name__ == "__main__":
    main()
