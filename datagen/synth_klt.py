"""Synthetic inputs for the IC-GVINS hot paths (SURVEY.md section 8d).  numpy only (cv2 optional for CLAHE).

Input generators only (no algorithm under test lives here): seeds are fixed so that the oracle, the golden vectors and the CUDA path all see
byte-identical inputs.  Nothing here is on the product path.
"""
from __future__ import annotations

import math

import numpy as np


# --------------------------------------------------------------------------------------------- KLT stream
def _gauss_kernel(sigma: float) -> np.ndarray:
    r = int(math.ceil(3 * sigma))
    x = np.arange(-r, r + 1, dtype=np.float64)
    k = np.exp(-0.5 * (x / sigma) ** 2)
    return k / k.sum()


def make_texture(W: int, H: int, seed: int = 1234, margin: int = 64, sigma: float = 1.5) -> np.ndarray:
    """Uniform u8 noise (W+2m)x(H+2m) -> separable Gaussian blur -> min-max normalise to 0..255 (float64)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    tw, th = W + 2 * margin, H + 2 * margin
    tex = rng.integers(0, 256, size=(th, tw), dtype=np.uint8).astype(np.float64)
    # add low-frequency structure so that coarse pyramid levels carry signal, as real images do
    low = rng.integers(0, 256, size=(th // 16 + 2, tw // 16 + 2)).astype(np.float64)
    low = np.kron(low, np.ones((16, 16)))[:th, :tw]
    k = _gauss_kernel(sigma)
    kl = _gauss_kernel(8.0)
    for kk, arr in ((k, tex), (kl, low)):
        arr[:] = np.apply_along_axis(lambda r: np.convolve(r, kk, mode="same"), 1, arr)
        arr[:] = np.apply_along_axis(lambda c: np.convolve(c, kk, mode="same"), 0, arr)
    tex = 0.55 * (tex - tex.min()) / (tex.max() - tex.min()) + 0.45 * (low - low.min()) / (low.max() - low.min())
    tex = (tex - tex.min()) / (tex.max() - tex.min()) * 255.0
    return tex


def ego_motion(t: int):
    """Cumulative smooth ego motion at frame t: (tx, ty, rot[rad], scale) (SURVEY 8d recipe, integrated)."""
    tx = sum(3.0 + 2.0 * math.sin(0.1 * i) for i in range(1, t + 1))
    ty = sum(2.0 * math.cos(0.07 * i) for i in range(1, t + 1))
    # keep the crop inside the texture margin: wrap the translation into +-24 px with a triangle wave
    def tri(v, a=24.0):
        p = 4 * a
        v = (v + a) % p
        return (v if v < 2 * a else p - v) - a
    rot = math.radians(0.1) * math.sin(0.05 * t) * 4.0
    sc = 1.0 + 0.002 * math.sin(0.03 * t) * 4.0
    return tri(tx), tri(ty), rot, sc


def warp_point(x, y, t: int, W: int, H: int):
    """Where does texture-space point (x, y) (frame-0 pixel coords) appear in frame t."""
    tx, ty, rot, sc = ego_motion(t)
    cx, cy = W / 2.0, H / 2.0
    c, s = math.cos(rot) * sc, math.sin(rot) * sc
    xr = c * (x - cx) - s * (y - cy) + cx + tx
    yr = s * (x - cx) + c * (y - cy) + cy + ty
    return xr, yr


def unwarp_point(x, y, t: int, W: int, H: int):
    """Inverse of warp_point: the frame-0 pixel coords of the point that appears at (x, y) in frame t."""
    tx, ty, rot, sc = ego_motion(t)
    cx, cy = W / 2.0, H / 2.0
    c, s = math.cos(rot) * sc, math.sin(rot) * sc
    det = c * c + s * s
    u, v = x - cx - tx, y - cy - ty
    return (c * u + s * v) / det + cx, (-s * u + c * v) / det + cy


def render_frame(tex: np.ndarray, t: int, W: int, H: int, margin: int = 64) -> np.ndarray:
    """Bilinear resample of the texture under the inverse ego-motion; returns u8 HxW."""
    tx, ty, rot, sc = ego_motion(t)
    cx, cy = W / 2.0, H / 2.0
    c, s = math.cos(rot) * sc, math.sin(rot) * sc
    det = c * c + s * s
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    u = xs - cx - tx
    v = ys - cy - ty
    # inverse of [[c,-s],[s,c]]
    x0 = (c * u + s * v) / det + cx + margin
    y0 = (-s * u + c * v) / det + cy + margin
    xi = np.floor(x0).astype(np.int64)
    yi = np.floor(y0).astype(np.int64)
    fx = x0 - xi
    fy = y0 - yi
    xi = np.clip(xi, 0, tex.shape[1] - 2)
    yi = np.clip(yi, 0, tex.shape[0] - 2)
    val = (tex[yi, xi] * (1 - fx) * (1 - fy) + tex[yi, xi + 1] * fx * (1 - fy) +
           tex[yi + 1, xi] * (1 - fx) * fy + tex[yi + 1, xi + 1] * fx * fy)
    return np.clip(np.rint(val), 0, 255).astype(np.uint8)


def grid_points(W: int, H: int, n: int, seed: int, border: float = 30.0) -> np.ndarray:
    """n pseudo-random feature positions (float32, N x 2) away from the border (stand-in for the block detector)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    x = rng.uniform(border, W - border, size=n)
    y = rng.uniform(border, H - border, size=n)
    return np.stack([x, y], axis=1).astype(np.float32)


def klt_pair(W=1280, H=560, n=300, seed=1234, t=1, noise_px=1.0, clahe=False):
    """One (prev, cur, prev_pts, init_pts, true_pts) tuple of the synthetic stream."""
    tex = make_texture(W, H, seed)
    f0 = render_frame(tex, t - 1, W, H)
    f1 = render_frame(tex, t, W, H)
    if clahe:
        import cv2
        cl = cv2.createCLAHE(3.0, (21, 21))
        f0, f1 = cl.apply(f0), cl.apply(f1)
    base = grid_points(W, H, n, seed + 7)
    p0 = np.array([warp_point(x, y, t - 1, W, H) for x, y in base], dtype=np.float64)
    p1 = np.array([warp_point(x, y, t, W, H) for x, y in base], dtype=np.float64)
    rng = np.random.Generator(np.random.PCG64(seed + 13 + t))
    init = p1 + rng.normal(0.0, noise_px, size=p1.shape)
    return f0, f1, p0.astype(np.float32), init.astype(np.float32), p1.astype(np.float32)


def pyramid_sizes(W: int, H: int, levels: int = 4):
    """(W_l, H_l) of levels 0 .. levels - 1 of a pyramid built with cv::pyrDown ((n + 1) / 2 per level)."""
    out = [(W, H)]
    for _ in range(levels - 1):
        W, H = (W + 1) // 2, (H + 1) // 2
        out.append((W, H))
    return out


def lk_levels(W: int, H: int, max_level: int = 3, win: int = 21) -> int:
    """Levels cv::buildOpticalFlowPyramid builds: it stops at the first level whose width or height is <= win."""
    n = 1
    for w, h in pyramid_sizes(W, H, max_level + 1)[1:]:
        if w <= win or h <= win:
            break
        n += 1
    return n


# window origins floor(x 2^-l - 10) of the LK edge rings at level l: low side, and offsets from W_l (H_l) on the high side.  -21 / W_l - 1
# are the last origins LK tracks at all, -1 / W_l - 23 the last ones whose 24 x 24 template taps (bilinear + Scharr) stay inside the level
EDGE_LO = (-22, -21, -20, -1, 0, 1, 2)
EDGE_HI = (-24, -23, -22, -2, -1, 0)
EDGE_FRACS = (0.0, 0.25, 0.5, 0.999)


def edge_rings(W: int, H: int, n_levels: int, rng: np.random.Generator, fracs=EDGE_FRACS, corner_origins=(-21, -1, -23, -1)):
    """Level-0 points (float32, N x 2) on all four sides of every level l < n_levels: for each edge origin o (EDGE_LO, W_l + EDGE_HI) and
    fractional part f, the level-l coordinate is o + 10 + f (2^-l is exact, so the level-l origin is exactly o); the other coordinate is
    uniform over the image.  Plus corner points (two low and two high origins per axis).  fracs=None draws a fresh fractional part per point."""
    def frac_list():
        return list(fracs) if fracs is not None else list(rng.uniform(0.0, 1.0, len(EDGE_FRACS)))

    def frac():
        return float(rng.choice(fracs)) if fracs is not None else float(rng.uniform(0.0, 1.0))

    pts = []
    for level, (wl, hl) in enumerate(pyramid_sizes(W, H, n_levels)):
        s = float(1 << level)
        for axis, (nl, full) in enumerate(((wl, H), (hl, W))):
            for o in [*EDGE_LO, *(nl + d for d in EDGE_HI)]:
                for f in frac_list():
                    c, other = (o + 10 + f) * s, rng.uniform(0.0, full)
                    pts.append((c, other) if axis == 0 else (other, c))
        lo, hi = corner_origins[:2], corner_origins[2:]
        for ox in [*lo, *(wl + d for d in hi)]:
            for oy in [*lo, *(hl + d for d in hi)]:
                pts.append(((ox + 10 + frac()) * s, (oy + 10 + frac()) * s))
    return np.array(pts, np.float32)


class KltStream:
    """Frame generator for one synthetic stream (renders lazily, caches the texture)."""

    def __init__(self, W=1280, H=560, n=300, seed=1234):
        self.W, self.H, self.n, self.seed = W, H, n, seed
        self.tex = make_texture(W, H, seed)
        self.base = grid_points(W, H, n, seed + 7)

    def frame(self, t: int) -> np.ndarray:
        return render_frame(self.tex, t, self.W, self.H)

    def points(self, t: int) -> np.ndarray:
        return np.array([warp_point(x, y, t, self.W, self.H) for x, y in self.base], dtype=np.float64)

    def pair(self, t: int, noise_px=1.0):
        p0, p1 = self.points(t - 1), self.points(t)
        rng = np.random.Generator(np.random.PCG64(self.seed + 13 + t))
        init = p1 + rng.normal(0.0, noise_px, size=p1.shape)
        return (self.frame(t - 1), self.frame(t), p0.astype(np.float32), init.astype(np.float32),
                p1.astype(np.float32))
