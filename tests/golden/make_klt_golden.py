"""Generate golden vectors for the KLT path from cv2 (the OpenCV build the reference links against is
un-vendored; this container pins opencv-python-headless 4.13.0).  Run HERE (needs cv2):

    python tests/golden/make_klt_golden.py

Writes tests/golden/klt_golden.npz.  Calls cv2 exactly as the reference does
(ic_gvins/ic_gvins/tracking/tracking.cc:385-403): forward LK with USE_INITIAL_FLOW, backward LK,
win 21x21, maxLevel 3, (COUNT+EPS, 30, 0.01).

Large images are not stored: they are re-rendered from datagen/synth_klt.py (numpy PCG64, deterministic) and
guarded by a CRC32 stored beside the outputs.  Small cases store their images.
"""
import os
import sys
import zlib

import cv2
import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))
from datagen import synth_klt as synth  # noqa: E402

CRIT = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.01)


def lk(a, b, p, init, max_level=3, criteria=CRIT, flags=cv2.OPTFLOW_USE_INITIAL_FLOW):
    out, st, err = cv2.calcOpticalFlowPyrLK(a, b, p.reshape(-1, 1, 2), init.reshape(-1, 1, 2).copy(), winSize=(21, 21),
                                            maxLevel=max_level, criteria=criteria, flags=flags)
    return out.reshape(-1, 2), st.ravel().astype(np.uint8), err.ravel()


def fb(a, b, p, init):
    fwd, st, _ = lk(a, b, p, init)
    bwd, st2, _ = lk(b, a, fwd, p)
    H, W = a.shape
    on_border = (fwd[:, 0] < 5.0) | (fwd[:, 1] < 5.0) | (fwd[:, 0] > W - 5.0) | (fwd[:, 1] > H - 5.0)
    dx = (bwd[:, 0] - p[:, 0]).astype(np.float64)
    dy = (bwd[:, 1] - p[:, 1]).astype(np.float64)
    dist = np.sqrt(dx * dx + dy * dy)
    good = (st != 0) & (st2 != 0) & (~on_border) & (dist < 0.5)
    return fwd, bwd, st, st2, good.astype(np.uint8)


def small_case(seed, W, H, n, noise, flat=False, edge=False):
    f0, f1, p0, init, _ = synth.klt_pair(W, H, n, seed, t=2, noise_px=noise)
    if flat:  # texture-less patch -> minEig rejection
        f0 = f0.copy(); f1 = f1.copy()
        f0[H // 4: 3 * H // 4, W // 4: 3 * W // 4] = 128
        f1[H // 4: 3 * H // 4, W // 4: 3 * W // 4] = 128
    if edge:  # points on / outside the border, initial flow far outside
        rng = np.random.Generator(np.random.PCG64(seed + 99))
        k = n // 3
        p0[:k, 0] = rng.uniform(-30, 12, k)
        p0[k:2 * k, 1] = rng.uniform(H - 12, H + 30, k)
        init[:k] = p0[:k] + rng.normal(0, 3, (k, 2))
        init[k:2 * k] = p0[k:2 * k] + rng.normal(0, 3, (k, 2))
        init[2 * k:2 * k + 5] = [W + 100.0, H + 100.0]
        p0 = p0.astype(np.float32); init = init.astype(np.float32)
    return f0, f1, p0, init


def main():
    out = {}
    # case A/B: full-size stream frames (images regenerated, CRC-guarded)
    for name, (t, noise) in {"full_t3": (3, 1.0), "full_t40": (40, 2.0)}.items():
        f0, f1, p0, init, _ = synth.klt_pair(1280, 560, 300, 1234, t=t, noise_px=noise)
        fwd, bwd, st, st2, good = fb(f0, f1, p0, init)
        out[name + "_crc"] = np.array([zlib.crc32(f0.tobytes()), zlib.crc32(f1.tobytes())], dtype=np.uint64)
        out[name + "_args"] = np.array([1280, 560, 300, 1234, t, noise], dtype=np.float64)
        for k, v in dict(p0=p0, init=init, fwd=fwd, bwd=bwd, st=st, st2=st2, good=good).items():
            out[f"{name}_{k}"] = v
    # small cases: images stored
    cases = {
        "small_plain": small_case(7, 320, 240, 120, 1.0),
        "small_noisy": small_case(8, 320, 240, 120, 6.0),
        "small_flat": small_case(9, 320, 240, 120, 1.0, flat=True),
        "small_edge": small_case(10, 320, 240, 120, 1.0, edge=True),
        "odd_size": small_case(11, 333, 187, 80, 2.0),
    }
    for name, (f0, f1, p0, init) in cases.items():
        fwd, bwd, st, st2, good = fb(f0, f1, p0, init)
        for k, v in dict(f0=f0, f1=f1, p0=p0, init=init, fwd=fwd, bwd=bwd, st=st, st2=st2, good=good).items():
            out[f"{name}_{k}"] = v
        print(name, "status", int(st.sum()), "/", len(st), "good", int(good.sum()))
    # pyrDown golden (bit-exact): 3 levels of a small image and of an odd-sized image
    for name in ("small_plain", "odd_size"):
        img = out[name + "_f0"]
        for l in range(1, 4):
            img = cv2.pyrDown(img)
            out[f"{name}_pyr{l}"] = img
    path = os.path.join(os.path.dirname(__file__), "klt_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes; cv2", cv2.__version__)


if __name__ == "__main__":
    main()
