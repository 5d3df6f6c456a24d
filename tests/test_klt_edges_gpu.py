"""GPU: the pyramid and the LK tracker at every image edge, pyramid depth and width residue (klt.cu), against cv2's golden vectors
(tests/golden/klt_edges_golden.npz) and, for seeded random sweeps, the CPU oracle that test_oracle_klt_edges.py pins to them.

Bars: pyramid levels and their reflect-101 padding bit-exact; status bit-exact; positions <= 1e-3 px and err <= 2e-3 (on the points that
are not knife-edge ties of cv2's exit decisions: see test_oracle_klt_edges.assert_lk)."""
import ctypes as C

import numpy as np
import pytest

from datagen import synth_klt as synth
from tests import oracle_api as oa
from tests.test_oracle_klt_edges import (LK_CASES, PYR_SIZES, TOL_ERR, TOL_PX, assert_lk, case_frames, edges_golden, first_box_escapes,
                                         frames, oracle_ties, pyr_frames, true_motion)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
KLT_PAD = 48


@pytest.fixture(scope="module")
def trackers():
    from ic_gvins_b200.klt import KltTracker
    cache = {}

    def get(W, H):
        if (W, H) not in cache:
            cache[(W, H)] = KltTracker(W, H, n_slots=4, max_points=4096)
        return cache[(W, H)]
    yield get
    for t in cache.values():
        t.close()


def size_of(name):
    return tuple(int(v) for v in edges_golden()[name + "_args"][:2])


def reflect101(p, n):
    """cv::borderInterpolate(BORDER_REFLECT_101) with the oracle's while loop: a pad wider than the level reflects more than once"""
    p = np.array(p, np.int64)
    if n == 1:
        return np.zeros_like(p)
    while ((p < 0) | (p >= n)).any():
        p = np.where(p < 0, -p, np.where(p >= n, 2 * (n - 1) - p, p))
    return p


def padded_plane(t, slot, level):
    """the raw padded plane (H_l + 96) x pitch of one slot and level, read from the device"""
    from ic_gvins_b200._lib import check, lib
    ptr, pitch, w, h = C.c_void_p(), C.c_int(), C.c_int(), C.c_int()
    check(lib().icg_klt_slot_level(t._h, slot, level, C.byref(ptr), C.byref(pitch), C.byref(w), C.byref(h)), "icg_klt_slot_level")
    t.sync()
    base = ptr.value - KLT_PAD * pitch.value - KLT_PAD

    class Plane:
        __cuda_array_interface__ = {"shape": (h.value + 2 * KLT_PAD, pitch.value), "typestr": "|u1", "data": (base, False), "version": 3}
    return torch.as_tensor(Plane(), device="cuda").cpu().numpy().copy(), w.value, h.value


def check_slot(t, slot, img, crc_row):
    import zlib
    for level in range(4):
        plane, w, h = padded_plane(t, slot, level)
        inner = plane[KLT_PAD:KLT_PAD + h, KLT_PAD:KLT_PAD + w]
        assert zlib.crc32(np.ascontiguousarray(inner).tobytes()) == int(crc_row[level]), f"slot {slot} level {level}"
        ys = reflect101(np.arange(plane.shape[0]) - KLT_PAD, h)
        xs = reflect101(np.arange(plane.shape[1]) - KLT_PAD, w)
        want = inner[ys][:, xs]
        bad = np.argwhere(plane != want)
        assert bad.size == 0, f"slot {slot} level {level} ({w}x{h}): padding differs at padded (y, x) {bad[:5].tolist()}"


@pytest.mark.parametrize("W,H", PYR_SIZES)
def test_pyramid_and_padding(trackers, W, H):
    """levels 0..3 bit-exact with cv2.pyrDown and the whole padded plane equal to the reflect-101 restatement, after icg_klt_upload and
    after icg_klt_upload_batch + icg_klt_build_pyramids into slots 2 and 3"""
    crc = edges_golden()[f"pyr_{W}x{H}_crc"]
    f0, f1 = (np.ascontiguousarray(f) for f in pyr_frames(W, H))
    t = trackers(W, H)
    t.upload(0, f0)
    check_slot(t, 0, f0, crc[0])
    t.upload_batch_ptrs(2, [f1.ctypes.data, f0.ctypes.data], W)
    t.build_pyramids(2, 2)
    check_slot(t, 2, f1, crc[1])
    check_slot(t, 3, f0, crc[0])


@pytest.mark.parametrize("name", LK_CASES)
def test_lk_edges_vs_golden(trackers, name):
    """forward LK with err, maxLevel 3..0, with and without initial flow, on the edge rings"""
    g = edges_golden()
    f0, f1 = case_frames(name)
    t = trackers(*size_of(name))
    for m in range(4):
        for flags in (0, 4):
            k = f"{name}_lk{m}f{flags}"
            q, st, err = t.calcOpticalFlowPyrLK(f0, f1, g[name + "_p0"], g[name + "_init"], maxLevel=m, flags=flags)
            assert_lk(q, st, err, g, k)


@pytest.mark.parametrize("name", LK_CASES)
def test_lk_edges_random_vs_oracle(trackers, oracle, name):
    """seeded random rings (fresh fractional parts and noise) against the oracle: forward LK with err and the fused forward + backward.
    Status bit-exact; positions off the oracle's knife-edge ties (oracle_ties), fb status off the gate thresholds"""
    W, H = size_of(name)
    f0, f1 = case_frames(name)
    t_frame = int(edges_golden()[name + "_args"][3])
    rng = np.random.Generator(np.random.PCG64(7000 + W * 1000 + H))
    p0 = synth.edge_rings(W, H, synth.lk_levels(W, H), rng, fracs=None)
    init = (true_motion(p0, t_frame - 1, t_frame, W, H) + rng.normal(0.0, 1.5, p0.shape)).astype(np.float32)
    t = trackers(W, H)
    for m in (3, 1, 0):
        q, st, err = t.calcOpticalFlowPyrLK(f0, f1, p0, init, maxLevel=m, flags=4)
        qo, sto, erro = oa.lk(oracle, f0, f1, p0, init, max_level=m)
        assert np.array_equal(st, sto), (m, np.flatnonzero(st != sto)[:10])
        ok = (st == 1) & ~oracle_ties(oracle, f0, f1, p0, init, qo, max_level=m)
        assert np.abs(q - qo)[ok].max() <= TOL_PX and np.abs(err - erro)[ok].max() <= TOL_ERR, m
    q, back, good = t.track_fb(f0, f1, p0, init)
    check_fb_vs_oracle(oracle, f0, f1, p0, init, q, back, good, "track_fb")


def check_fb_vs_oracle(oracle, a, b, p, init, fwd, back, good, what):
    """forward + backward + gates against the oracle: the gate status bit-exact off the gate thresholds (the oracle's forward position or
    forward-backward distance within 2e-3 of one); the forward positions off the oracle's ties; the backward positions against the oracle's
    backward call from THIS forward result (the call the kernel made: chaining from the oracle's own forward result would amplify the
    forward's rounding difference on ill-conditioned points)"""
    H, W = a.shape
    qo, backo, goodo = oa.track_fb(oracle, a, b, p, init)
    gate_tie = np.abs(np.hypot(*(backo - p).astype(np.float64).T) - 0.5) < 2e-3
    for v, thr in ((qo[:, 0], 5.0), (qo[:, 1], 5.0), (qo[:, 0], W - 5.0), (qo[:, 1], H - 5.0)):
        gate_tie |= np.abs(v.astype(np.float64) - thr) < 2e-3
    assert np.array_equal(good[~gate_tie], goodo[~gate_tie]), what
    ok = (good == 1) & (goodo == 1)
    okf = ok & ~oracle_ties(oracle, a, b, p, init, qo)
    assert np.abs(fwd - qo)[okf].max() <= TOL_PX, what
    bo, _, _ = oa.lk(oracle, b, a, fwd, p)
    okb = ok & ~oracle_ties(oracle, b, a, fwd, p, bo)
    assert np.abs(back - bo)[okb].max() <= TOL_PX, what


def test_recentre_vs_golden(trackers):
    """maxLevel 0 with the initial flow 6-20 px off the true motion: every case matches cv2, and at least 20 matched points per direction
    end outside the search window the kernel staged first, so each of them was re-centred (in the iteration or in the err epilogue)"""
    g = edges_golden()
    n = np.zeros(4, np.int64)
    for name in LK_CASES:
        f0, f1 = case_frames(name)
        init = g[name + "_rc_init"]
        q, st, err = trackers(*size_of(name)).calcOpticalFlowPyrLK(f0, f1, g[name + "_rc_p0"], init, maxLevel=0, flags=4)
        assert_lk(q, st, err, g, name + "_rc")
        esc = first_box_escapes(init, q) & (st == 1) & (g[name + "_rc_tie"] == 0)
        n += [int((esc & (g[name + "_rc_dir"] == d)).sum()) for d in range(4)]
    assert (n >= 20).all(), n


@pytest.mark.parametrize("name", LK_CASES)
def test_track_batch_dev_vs_oracle(trackers, oracle, name):
    """icg_klt_track_batch_dev, modes 0 and 1, four slots with different frames and task pairs mixed across slots and reversed in one launch;
    each pair against the oracle (which builds cv2's pyramid depth: fewer than 4 levels at the small sizes; positions off its ties)"""
    W, H = size_of(name)
    args = edges_golden()[name + "_args"]
    seed, t0 = int(args[2]), int(args[3]) - 1
    tex = synth.make_texture(W, H, seed)
    ts = [t0, t0 + 1, t0 + 2, t0 + 3]
    imgs = [np.ascontiguousarray(synth.render_frame(tex, t, W, H)) for t in ts]
    assert np.array_equal(imgs[0], frames(W, H, seed, t0 + 1)[0])
    trk = trackers(W, H)
    trk.upload_batch_ptrs(0, [im.ctypes.data for im in imgs], W)
    trk.build_pyramids(0, 4)
    rng = np.random.Generator(np.random.PCG64(9000 + W * 1000 + H))
    pairs = [(1, 3), (3, 1), (0, 2), (2, 0), (0, 1), (2, 3)]
    p_all, i_all, s_all, seg = [], [], [], [0]
    for a, b in pairs:
        p = synth.edge_rings(W, H, synth.lk_levels(W, H), rng, fracs=None)[::2]
        init = (true_motion(p, ts[a], ts[b], W, H) + rng.normal(0.0, 1.0, p.shape)).astype(np.float32)
        p_all.append(p), i_all.append(init), s_all.append(np.tile([a, b], (len(p), 1)))
        seg.append(seg[-1] + len(p))
    p_all, i_all, s_all = np.concatenate(p_all), np.concatenate(i_all), np.concatenate(s_all).astype(np.int32)
    n = len(p_all)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    d_slots, d_prev, d_init = dev(s_all), dev(p_all), dev(i_all)
    for mode in (0, 1):
        d_fwd = torch.zeros((n, 2), dtype=torch.float32, device="cuda")
        d_bwd = torch.zeros((n, 2), dtype=torch.float32, device="cuda")
        d_st = torch.zeros(n, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        trk.track_batch_dev(n, d_slots.data_ptr(), d_prev.data_ptr(), d_init.data_ptr(), d_fwd.data_ptr(), d_bwd.data_ptr() if mode else 0,
                            d_st.data_ptr(), mode=mode)
        trk.sync()
        fwd, bwd, st = d_fwd.cpu().numpy(), d_bwd.cpu().numpy(), d_st.cpu().numpy()
        for k, (a, b) in enumerate(pairs):
            sl = slice(seg[k], seg[k + 1])
            p, init = p_all[sl], i_all[sl]
            if mode == 0:
                qo, sto, _ = oa.lk(oracle, imgs[a], imgs[b], p, init)
                assert np.array_equal(st[sl], sto), (mode, a, b, np.flatnonzero(st[sl] != sto)[:10])
                ok = (sto == 1) & ~oracle_ties(oracle, imgs[a], imgs[b], p, init, qo)
                assert np.abs(fwd[sl] - qo)[ok].max() <= TOL_PX, (mode, a, b)
            else:
                check_fb_vs_oracle(oracle, imgs[a], imgs[b], p, init, fwd[sl], bwd[sl], st[sl], (mode, a, b))


@pytest.mark.parametrize("name", LK_CASES)
def test_criteria_vs_golden(trackers, name):
    """COUNT-only criteria take cv2's default epsilon 0.01, EPS-only criteria its default count 30"""
    from ic_gvins_b200.klt import TERM_COUNT, TERM_EPS
    g = edges_golden()
    f0, f1 = case_frames(name)
    t = trackers(*size_of(name))
    for key, crit in (("count", (TERM_COUNT, 30, 0.5)), ("eps", (TERM_EPS, 5, 0.01))):
        q, st, err = t.calcOpticalFlowPyrLK(f0, f1, g[name + "_p0"], g[name + "_init"], criteria=crit, flags=4)
        assert_lk(q, st, err, g, f"{name}_{key}")


def test_max_count_clamped_to_100(trackers):
    """(COUNT + EPS, 150, 0) iterates at most 100 times, as cv2: equal to the golden, bit-identical to maxCount 100, and the points are still
    moving at iteration 100 (maxCount 99 gives other positions)"""
    from ic_gvins_b200.klt import TERM_COUNT, TERM_EPS
    g = edges_golden()
    W, H = (int(v) for v in g["mc_case"])
    f0, f1 = case_frames(f"s{W}x{H}")
    t = trackers(W, H)
    run = lambda k: t.calcOpticalFlowPyrLK(f0, f1, g["mc_p0"], g["mc_init"], maxLevel=0, criteria=(TERM_COUNT + TERM_EPS, k, 0.0),  # noqa: E731
                                           flags=4)
    q, st, err = run(150)
    assert_lk(q, st, err, g, "mc")
    q100, st100, _ = run(100)
    assert np.array_equal(q, q100) and np.array_equal(st, st100)
    q99, _, _ = run(99)
    assert ((np.abs(q99 - q).max(axis=1) > TOL_PX) & (st == 1)).sum() >= 10
