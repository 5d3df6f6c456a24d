"""GPU parity tests for path A (pyramid + LK) through the C ABI, against the CPU oracle and the cv2 golden vectors.

Bars (north_star): status / feature selection bit-exact, tracked positions within 1e-3 px, pyrDown bit-exact.
"""
import zlib

import numpy as np
import pytest

from datagen import synth_klt as synth
from tests import oracle_api as oa
from tests.test_oracle_klt import SMALL, assert_px
from tests.test_oracle_klt_edges import LK_CASES, case_frames, edges_golden

pytestmark = pytest.mark.gpu


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


@pytest.mark.parametrize("name", ["small_plain", "odd_size"])
def test_pyramid_bit_exact(trackers, klt_golden, name):
    img = klt_golden[name + "_f0"]
    H, W = img.shape
    t = trackers(W, H)
    t.upload(0, img)
    assert np.array_equal(t.download_level(0, 0), img)
    for l in range(1, 4):
        assert np.array_equal(t.download_level(0, l), klt_golden[f"{name}_pyr{l}"]), f"level {l}"


@pytest.mark.parametrize("name", SMALL)
def test_lk_forward_vs_golden_and_oracle(trackers, oracle, klt_golden, name):
    g = klt_golden
    f0, f1, p0, init = g[name + "_f0"], g[name + "_f1"], g[name + "_p0"], g[name + "_init"]
    H, W = f0.shape
    q, st, err = trackers(W, H).calcOpticalFlowPyrLK(f0, f1, p0, init, flags=4)
    assert np.array_equal(st, g[name + "_st"])
    assert_px(q, g[name + "_fwd"], st == 1, name)
    qo, sto, erro = oa.lk(oracle, f0, f1, p0, init)
    assert np.array_equal(st, sto)
    assert_px(q, qo, st == 1, name)
    assert np.abs(err - erro)[st == 1].max() <= 2e-3


@pytest.mark.parametrize("name", SMALL + LK_CASES)
def test_track_fb_vs_golden(trackers, klt_golden, name):
    """the small cases of klt_golden.npz, and the edge rings of klt_edges_golden.npz (sizes where cv2 builds 1 to 4 levels; positions
    compared off the knife-edge ties its generator marks)"""
    if name in LK_CASES:
        e = edges_golden()
        (f0, f1), p0, init = case_frames(name), e[name + "_p0"], e[name + "_init"]
        good_ref, fwd_ref, bwd_ref, cmp = e[name + "_fb_good"], e[name + "_fb_fwd"], e[name + "_fb_bwd"], e[name + "_fb_tie"] == 0
    else:
        g = klt_golden
        f0, f1, p0, init = g[name + "_f0"], g[name + "_f1"], g[name + "_p0"], g[name + "_init"]
        good_ref, fwd_ref, bwd_ref, cmp = g[name + "_good"], g[name + "_fwd"], g[name + "_bwd"], True
    H, W = f0.shape
    q, back, good = trackers(W, H).track_fb(f0, f1, p0, init)
    assert np.array_equal(good, good_ref)
    assert_px(q, fwd_ref, (good == 1) & cmp, name)
    assert_px(back, bwd_ref, (good == 1) & cmp, name, chained_backward=True)  # the one explained exception: see assert_px


@pytest.mark.parametrize("name", SMALL)
def test_backward_call_from_cv2_forward_vs_golden(trackers, klt_golden, name):
    """The backward calcOpticalFlowPyrLK call with exactly cv2's arguments (prevPts = cv2's forward result): status identical, <= 1e-3 px in
    EVERY case (no exception: the `small_flat` rim points included)."""
    g = klt_golden
    f0, f1 = g[name + "_f0"], g[name + "_f1"]
    H, W = f0.shape
    b, st, _ = trackers(W, H).calcOpticalFlowPyrLK(f1, f0, g[name + "_fwd"], g[name + "_p0"], flags=4)
    sel = g[name + "_st"] == 1
    assert np.array_equal(st[sel], g[name + "_st2"][sel])
    ok = sel & (st == 1)
    assert np.abs(b - g[name + "_bwd"])[ok].max() <= 1e-3


@pytest.mark.parametrize("key", ["full_t3", "full_t40"])
def test_full_size_stream_frame(trackers, klt_golden, key):
    g = klt_golden
    W, H, n, seed, t, noise = g[key + "_args"]
    f0, f1, p0, init, _ = synth.klt_pair(int(W), int(H), int(n), int(seed), t=int(t), noise_px=float(noise))
    crc = g[key + "_crc"]
    assert zlib.crc32(f0.tobytes()) == int(crc[0]) and zlib.crc32(f1.tobytes()) == int(crc[1])
    q, back, good = trackers(1280, 560).track_fb(f0, f1, p0, init)
    assert np.array_equal(good, g[key + "_good"])
    assert_px(q, g[key + "_fwd"], good == 1, key)
    assert_px(back, g[key + "_bwd"], good == 1, key)


def test_no_initial_flow_and_fewer_levels(trackers, oracle, klt_golden):
    g = klt_golden
    f0, f1, p0 = g["small_plain_f0"], g["small_plain_f1"], g["small_plain_p0"]
    t = trackers(320, 240)
    for max_level in (0, 1, 3):
        q, st, _ = t.calcOpticalFlowPyrLK(f0, f1, p0, None, maxLevel=max_level, flags=0)
        qo, sto, _ = oa.lk(oracle, f0, f1, p0, p0, max_level=max_level, flags=0)
        assert np.array_equal(st, sto)
        assert_px(q, qo, st == 1, "small_plain")


def test_empty_and_unsupported(trackers):
    from ic_gvins_b200 import IcgError
    t = trackers(320, 240)
    img = np.zeros((240, 320), np.uint8)
    q, st, err = t.calcOpticalFlowPyrLK(img, img, np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32), flags=4)
    assert q.shape == (0, 2) and st.shape == (0,)
    with pytest.raises(IcgError):
        t.calcOpticalFlowPyrLK(img, img, np.ones((3, 2), np.float32), None, winSize=(15, 15))


def test_idempotent_and_cache(trackers, klt_golden):
    """Same inputs twice -> bit-identical outputs (pyramid cache hit on the second call)."""
    g = klt_golden
    f0, f1, p0, init = g["small_noisy_f0"], g["small_noisy_f1"], g["small_noisy_p0"], g["small_noisy_init"]
    t = trackers(320, 240)
    a = t.track_fb(f0, f1, p0, init)
    b = t.track_fb(f0, f1, p0, init)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_batched_upload_equals_single_uploads(trackers, klt_golden):
    """icg_klt_upload_batch (linear DMA + scatter kernel) fills the level-0 planes exactly like icg_klt_upload_level0; pyramids bit-exact."""
    g = klt_golden
    imgs = [np.ascontiguousarray(g[n]) for n in ("small_plain_f0", "small_plain_f1", "small_noisy_f0")]
    H, W = imgs[0].shape
    t = trackers(W, H)
    t.upload_batch_ptrs(1, [im.ctypes.data for im in imgs], W)
    t.build_pyramids(1, 3)
    for k, im in enumerate(imgs):
        assert np.array_equal(t.download_level(1 + k, 0), im)
    for l in range(1, 4):
        assert np.array_equal(t.download_level(1, l), g[f"small_plain_pyr{l}"]), f"level {l}"
