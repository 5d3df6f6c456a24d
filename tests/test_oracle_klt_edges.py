"""Pin the KLT oracle (oracle/klt_ref.c) at the image edges against cv2 (tests/golden/klt_edges_golden.npz, make_klt_edges_golden.py).

Points sit at every edge of every pyramid level cv2 builds, at sizes where it builds 1 to 4 levels; the pyrDown levels of 22 sizes (every
level-0 width residue mod 16) are pinned by CRC32.  Bars: status bit-exact, positions <= 1e-3 px, err <= 2e-3, pyrDown bit-exact.  These
pins are what lets the GPU edge tests (test_klt_edges_gpu.py) use the oracle for their randomized sweeps.  CPU only.
"""
import functools
import os
import zlib

import numpy as np
import pytest

from datagen import synth_klt as synth
from tests import oracle_api as oa

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LK_CASES = ["s32x32", "s42x100", "s43x100", "s320x168", "s320x169", "s168x240", "s176x180", "s179x180", "s186x180", "s191x180"]
PYR_SIZES = [(32, 32), (42, 100), (43, 100), (320, 168), (320, 169), (168, 240)] + [(w, 180) for w in range(176, 192)]
TOL_PX, TOL_ERR = 1e-3, 2e-3
KLT_MARGIN, KLT_BOXW, KLT_BOXH_J = 5, 48, 32  # the tracker's search window (klt_handle.cuh)
START_NUDGES = np.array([[1e-4, 0], [-1e-4, 0], [0, 1e-4], [0, -1e-4]], np.float32)  # start-point moves of the tie rule


@functools.lru_cache(maxsize=None)
def edges_golden():
    g = np.load(os.path.join(ROOT, "tests", "golden", "klt_edges_golden.npz"))
    return {k: g[k] for k in g.files}


@functools.lru_cache(maxsize=None)
def frames(W, H, seed, t):
    tex = synth.make_texture(W, H, seed)
    return synth.render_frame(tex, t - 1, W, H), synth.render_frame(tex, t, W, H)


def case_frames(name):
    """the case's two frames, re-rendered and checked against the CRC32s cv2 saw"""
    g = edges_golden()
    W, H, seed, t = (int(v) for v in g[name + "_args"])
    f0, f1 = frames(W, H, seed, t)
    crc = g[name + "_crc"]
    assert zlib.crc32(f0.tobytes()) == int(crc[0]) and zlib.crc32(f1.tobytes()) == int(crc[1]), "synthetic frames drifted"
    return f0, f1


def pyr_frames(W, H):
    W_, H_, seed, t = (int(v) for v in edges_golden()[f"pyr_{W}x{H}_args"])
    return frames(W_, H_, seed, t)


def true_motion(p, t_from, t_to, W, H):
    """where the texture point seen at p in frame t_from appears in frame t_to"""
    bx, by = synth.unwarp_point(p[:, 0].astype(np.float64), p[:, 1].astype(np.float64), t_from, W, H)
    return np.stack(synth.warp_point(bx, by, t_to, W, H), axis=1)


def assert_lk(q, st, err, g, key, what=None):
    """status bit-exact with the golden call `key`; positions and err on the tracked points that are not ties (`<key>_tie`: cv2's
    position moves by more than 5e-4 px when its epsilon moves by 1 %, when it may iterate once more, or when the start point moves by
    1e-4 px along an axis -- an exit decision on a knife edge or an ill-conditioned window, see make_klt_edges_golden.ties)"""
    what = what or key
    st_ref = g[key + "_st"]
    assert np.array_equal(st, st_ref), f"{what}: status differs at {np.flatnonzero(st != st_ref)[:10]}"
    ok = (st == 1) & (g[key + "_tie"] == 0)
    q_ref, err_ref = g[key + "_fwd"], g[key + "_err"]
    if ok.any():
        d = np.abs(q - q_ref)[ok].max()
        assert d <= TOL_PX, f"{what}: {d} px"
        if err is not None:
            e = np.abs(err - err_ref)[ok].max()
            assert e <= TOL_ERR, f"{what}: err {e}"


def oracle_ties(oracle, a, b, p, init, q, max_level=3, max_iter=30, eps=0.01, flags=4):
    """the golden generator's tie rule with the oracle in cv2's place, for the seeded sweeps that have no golden: points whose oracle
    position q moves by more than 5e-4 px when eps moves by 1 %, when one more iteration is allowed, or when p moves by 1e-4 px along an axis"""
    variants = [(p + d, max_iter, eps) for d in START_NUDGES]
    if eps > 0:
        variants += [(p, max_iter, 0.99 * eps), (p, max_iter, 1.01 * eps)]
    if max_iter < 100:
        variants.append((p, max_iter + 1, eps))
    t = np.zeros(len(p), bool)
    for pv, it, ev in variants:
        qv, _, _ = oa.lk(oracle, a, b, pv, init, max_level=max_level, max_iter=it, eps=ev, flags=flags)
        t |= np.abs(qv - q).max(axis=1) > 5e-4
    return t


def first_box_escapes(init, fwd):
    """maxLevel-0 tracks whose final window origin floor(fwd - 10) lies outside the search window staged at the start (the tracker's
    box_origin: 5 px of slack, x aligned down to 16; a 48 x 32 box holds origins [jx0, jx0 + 26] x [jy0, jy0 + 10]).  Such a track was
    re-centred at least once, in the iteration or in the err epilogue."""
    ix, iy = np.floor(init[:, 0] - np.float32(10)).astype(np.int64), np.floor(init[:, 1] - np.float32(10)).astype(np.int64)
    jx0, jy0 = (ix - KLT_MARGIN) & ~15, iy - KLT_MARGIN
    fx, fy = np.floor(fwd[:, 0] - np.float32(10)).astype(np.int64), np.floor(fwd[:, 1] - np.float32(10)).astype(np.int64)
    ox, oy = fx - jx0, fy - jy0
    return (ox < 0) | (ox > KLT_BOXW - 22) | (oy < 0) | (oy > KLT_BOXH_J - 22)


def recentred(g, name):
    """tracked, position-compared re-centre points that leave their first search window"""
    return first_box_escapes(g[name + "_rc_init"], g[name + "_rc_fwd"]) & (g[name + "_rc_st"] == 1) & (g[name + "_rc_tie"] == 0)


@pytest.mark.parametrize("W,H", PYR_SIZES)
def test_pyr_down_crc_matches_cv2(oracle, W, H):
    crc = edges_golden()[f"pyr_{W}x{H}_crc"]
    for i, img in enumerate(pyr_frames(W, H)):
        for level in range(4):
            assert zlib.crc32(np.ascontiguousarray(img).tobytes()) == int(crc[i, level]), f"frame {i} level {level}"
            img = oa.pyr_down(oracle, img)


def test_golden_level_counts():
    """the sizes reach every pyramid depth cv2 can build (1 to 4 levels), each side of the width and the height limit"""
    g = edges_golden()
    levels = {n: synth.lk_levels(*(int(v) for v in g[n + "_args"][:2])) for n in LK_CASES}
    assert [levels[n] for n in ("s32x32", "s42x100", "s43x100", "s320x168", "s320x169", "s168x240")] == [1, 1, 2, 3, 4, 3]


@pytest.mark.parametrize("name", LK_CASES)
def test_lk_edges_match_cv2(oracle, name):
    g = edges_golden()
    f0, f1 = case_frames(name)
    p0, init = g[name + "_p0"], g[name + "_init"]
    for m in range(4):
        for flags in (0, 4):
            k = f"{name}_lk{m}f{flags}"
            q, st, err = oa.lk(oracle, f0, f1, p0, init, max_level=m, flags=flags)
            assert_lk(q, st, err, g, k)


@pytest.mark.parametrize("name", LK_CASES)
def test_track_fb_edges_match_cv2(oracle, name):
    g = edges_golden()
    f0, f1 = case_frames(name)
    q, back, good = oa.track_fb(oracle, f0, f1, g[name + "_p0"], g[name + "_init"])
    assert np.array_equal(good, g[name + "_fb_good"])
    ok = (good == 1) & (g[name + "_fb_tie"] == 0)
    assert np.abs(q - g[name + "_fb_fwd"])[ok].max() <= TOL_PX
    assert np.abs(back - g[name + "_fb_bwd"])[ok].max() <= TOL_PX


@pytest.mark.parametrize("name", LK_CASES)
def test_recentre_cases_match_cv2(oracle, name):
    g = edges_golden()
    f0, f1 = case_frames(name)
    q, st, err = oa.lk(oracle, f0, f1, g[name + "_rc_p0"], g[name + "_rc_init"], max_level=0)
    assert_lk(q, st, err, g, name + "_rc")


def test_recentre_cases_leave_their_first_window():
    """over all cases, at least 20 tracked points per direction end outside the search window the tracker stages first"""
    g = edges_golden()
    for d in range(4):
        n = sum(int((recentred(g, c) & (g[c + "_rc_dir"] == d)).sum()) for c in LK_CASES)
        assert n >= 20, (d, n)


def test_max_count_is_clamped_to_100(oracle):
    """(COUNT + EPS, 150, 0): cv2 iterates at most 100 times; the golden points are still moving at iteration 100"""
    g = edges_golden()
    W, H = (int(v) for v in g["mc_case"])
    name = f"s{W}x{H}"
    f0, f1 = case_frames(name)
    q, st, err = oa.lk(oracle, f0, f1, g["mc_p0"], g["mc_init"], max_level=0, max_iter=150, eps=0.0)
    assert_lk(q, st, err, g, "mc")
    q99, st99, _ = oa.lk(oracle, f0, f1, g["mc_p0"], g["mc_init"], max_level=0, max_iter=99, eps=0.0)
    assert ((np.abs(q99 - q).max(axis=1) > TOL_PX) & (st == 1)).sum() >= 10


def test_dropped_points_and_ties_are_few():
    """the position bar covers most tracked points: at most 15 % of them are ties (edge windows, partly outside the level, are more often
    ill-conditioned than interior ones)"""
    g = edges_golden()
    assert sum(int(g[n + "_dropped"]) for n in LK_CASES) <= 10
    for n in LK_CASES:
        for k in [f"{n}_lk{m}f{f}" for m in range(4) for f in (0, 4)] + [n + "_count", n + "_eps"]:
            tracked = g[k + "_st"] == 1
            assert (g[k + "_tie"][tracked] == 1).mean() <= 0.15, k
