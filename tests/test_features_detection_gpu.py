"""GPU: Tracking::featuresDetection driven by the point lists (icg_detect_features / icg_detect_features_dev, IG/tracking/tracking.cc:576-685).
The occupancy mask is compared byte for byte with cv2.circle, the corners with the CPU restatement (tests/features_oracle.py) and bitwise
with icg_detect_blocks fed a cv2.circle mask and host-computed deficits; the device-list entry is compared frame by frame with the host one."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from datagen import synth_klt as synth
from tests import features_oracle as fo
from tests import oracle_api as oa

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, MAXF = 1280, 560, 300


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_detect(oracle)
    return oracle


@pytest.fixture(scope="module")
def img():
    return synth.render_frame(synth.make_texture(W, H, 41), 0, W, H)


def download(ptr, pitch, h, w):
    """a pitched u8 device plane -> host array (through torch's __cuda_array_interface__ import)"""
    class Plane:
        __cuda_array_interface__ = {"shape": (h, pitch), "typestr": "|u1", "data": (ptr, False), "version": 3}
    return torch.as_tensor(Plane(), device="cuda").cpu().numpy()[:, :w].copy()


def cv2_mask(pts, r, w=W, h=H):
    m = np.full((h, w), 255, np.uint8)
    for x, y in np.asarray(pts, np.float32).reshape(-1, 2):
        cv2.circle(m, (int(round(float(x))), int(round(float(y)))), int(r), 0, cv2.FILLED)
    return m


def random_lists(seed, n_feat, n_new):
    """list A: undistorted keypoints, some of them outside the frame; list B: tracked (distorted) points inside it"""
    rng = np.random.default_rng(seed)
    a = rng.uniform([-60, -60], [W + 60, H + 60], size=(n_feat, 2)).astype(np.float32)
    b = rng.uniform([0, 0], [W - 1, H - 1], size=(n_new, 2)).astype(np.float32)
    b[:4] = np.round(b[:4]) + 0.5  # rounding ties of the disc centres
    return a, b


def test_mask_equals_cv2_circle_golden():
    """icg_detect_mask_dev after a detection call on every golden frame (160 x 120: one block; max_features chosen so that min_dist is the
    case's radius).  Radii 1 and 2 make the min-distance grid of goodFeaturesToTrack too fine for the device selection (out_n = -2): the mask
    is built before detection and is checked all the same."""
    from ic_gvins_b200.detect import Detector
    g = np.load(os.path.join(ROOT, "tests", "golden", "mask_golden.npz"))
    quota_for = {40: 17, 17: 92, 2: 6667, 1: 26667}
    names = sorted({k[:-5] for k in g.files if k.endswith("_mask")})
    dets = {}
    s = torch.cuda.Stream()
    try:
        for n in names:
            w, h = (int(v) for v in g[n + "_size"])
            r = int(g[n + "_r"])
            q = quota_for[r]
            assert fo.grid(w, h, q)[5] == r
            d = dets.get(q) or dets.setdefault(q, Detector(w, h, max_blocks=1, max_corners_per_block=q, stream=s.cuda_stream))
            frame = torch.zeros((h, w), dtype=torch.uint8, device="cuda")
            pts = torch.from_numpy(np.ascontiguousarray(g[n + "_pts"])).cuda()
            out_xy = torch.zeros((q, 2), dtype=torch.float32, device="cuda")
            out_n = torch.zeros(1, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            d.features_detection_dev(1, frame.data_ptr(), w, w * h, 0, 0, [0, 0], pts.data_ptr(), 0, [0, len(pts)], out_xy.data_ptr(),
                                     out_n.data_ptr(), n_ref=[0], ismask=[1], max_features=q)
            s.synchronize()
            assert int(out_n.item()) >= 0 or (r <= 2 and int(out_n.item()) == -2), (n, int(out_n.item()))
            ptr, pitch = d.mask_dev(0)
            assert np.array_equal(download(ptr, pitch, h, w), g[n + "_mask"]), n
    finally:
        for d in dets.values():
            d.close()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_mask_equals_cv2_circle_on_random_points(img, seed):
    from ic_gvins_b200.detect import Detector
    a, b = random_lists(seed, 150, 150)
    d = Detector(W, H, max_blocks=18, max_corners_per_block=32)
    got = d.features_detection_points(img, a, b, n_ref=0, ismask=True)
    assert got is not None
    m = download(*d.mask_dev(0), H, W)
    d.close()
    assert np.array_equal(m, cv2_mask(np.concatenate([a, b]), 40))


CASES = [  # (seed, n_feat, n_new, n_ref, ismask): gated iff n_feat + n_ref > 295
    (11, 40, 120, None, True), (12, 0, 200, None, True), (13, 90, 60, 30, True), (14, 40, 120, None, False), (15, 0, 0, None, True),
    (16, 100, 150, 196, True), (17, 0, 296, None, True), (18, 150, 10, 146, False), (19, 60, 230, None, False),
]


@pytest.mark.parametrize("seed,n_feat,n_new,n_ref,ismask", CASES)
def test_host_call_equals_oracle_and_block_detection(olib, img, seed, n_feat, n_new, n_ref, ismask):
    from ic_gvins_b200.detect import Detector
    a, b = random_lists(seed, n_feat, n_new)
    d = Detector(W, H, max_blocks=18, max_corners_per_block=32)
    got = d.features_detection_points(img, a, b, n_ref=n_ref, ismask=ismask, max_features=MAXF)
    ref = fo.features_detection(olib, img, a, b, n_ref=n_ref, ismask=ismask, max_features=MAXF)
    gated = n_feat + (n_new if n_ref is None else n_ref) > MAXF - 5
    assert ref["skipped"] == gated and (got is None) == gated
    if gated:
        d.close()
        return
    assert got.shape == ref["corners"].shape and got.shape[0] > 0
    assert np.abs(got - ref["corners"]).max() <= 1e-3
    assert np.array_equal(download(*d.mask_dev(0), H, W), ref["mask"])
    # the existing block API with a cv2.circle mask and host-computed deficits gives the same corners, bit for bit
    cols, rows, bw, bh, quota, min_dist = fo.grid(W, H, MAXF)
    mask = cv2_mask(np.concatenate([a, b]), min_dist) if ismask else None
    want = [max(0, quota - int(c)) for c in fo.counts(a, b, cols, rows, bw, bh)]
    blocks = d.detect_blocks(img, fo.rois(W, H, MAXF), want, 0.01, float(min_dist), mask, subpix=True)
    d.close()
    host = [np.stack([np.float32(k % cols * bw) + p[:, 0], np.float32(k // cols * bh) + p[:, 1]], axis=1) for k, p in enumerate(blocks) if len(p)]
    assert np.array_equal(got, np.concatenate(host).astype(np.float32))


def test_integer_selection_equals_oracle(olib, img):
    """without sub-pixel refinement on either side: the device's integer-pixel corners of every block, with the deficits and mask the
    point lists imply, are the oracle's goodFeaturesToTrack selection exactly"""
    from ic_gvins_b200.detect import Detector
    a, b = random_lists(21, 60, 120)
    b = np.concatenate([b, np.random.default_rng(22).uniform(10, 190, size=(20, 2)).astype(np.float32)])  # block 0 has no deficit left
    cols, rows, bw, bh, quota, min_dist = fo.grid(W, H, MAXF)
    d = Detector(W, H, max_blocks=18, max_corners_per_block=32)
    assert d.features_detection_points(img, a, b) is not None
    mask = download(*d.mask_dev(0), H, W)
    want = [quota - int(c) for c in fo.counts(a, b, cols, rows, bw, bh)]
    raw = d.detect_blocks(img, fo.rois(W, H, MAXF), [max(0, w_) for w_ in want], 0.01, float(min_dist), mask, subpix=False)
    d.close()
    assert any(w_ <= 0 for w_ in want) and sum(len(p) for p in raw) > 50
    for roi, w_, p in zip(fo.rois(W, H, MAXF), want, raw):
        ref = oa.good_features(olib, img, w_, 0.01, float(min_dist), mask=mask, roi=roi) if w_ > 0 else np.zeros((0, 2), np.float32)
        assert np.array_equal(p, ref)


def test_device_lists_from_klt_equal_host_calls(img):
    """icg_detect_features_dev on consecutive KLT slots, list B straight from icg_klt_track_batch_dev (its status passed, n_ref = NULL),
    list A device-resident without status: frame by frame the host call on the compacted lists, bitwise; out_n == -1 exactly for gated frames."""
    from ic_gvins_b200.detect import Detector
    from ic_gvins_b200.klt import KltTracker
    from ic_gvins_b200._lib import lib, vp
    NF = 5
    st = synth.KltStream(W, H, MAXF, 99)
    frames = [st.frame(t) for t in range(NF + 1)]
    s = torch.cuda.Stream()
    trk = KltTracker(W, H, n_slots=NF + 1, max_points=NF * MAXF, stream=s.cuda_stream)
    for k, f in enumerate(frames):
        trk.upload(k, f, build=True)
    trk.sync()
    n_new = [200, 150, 250, 120, 300]
    n_feat = [30, 0, 60, 200, 5]           # frame 3: 200 + its valid tracks > 295 -> gated unless a fifth of them are lost
    rng = np.random.default_rng(5)
    prev, init, slots = [], [], []
    for f in range(NF):
        p = st.points(f)[:n_new[f]].astype(np.float32)
        prev.append(p)
        init.append((st.points(f + 1)[:n_new[f]] + rng.normal(0, 1.0, p.shape)).astype(np.float32))
        slots.append(np.stack([np.full(n_new[f], f), np.full(n_new[f], f + 1)], axis=1).astype(np.int32))
    prev, init, slots = (np.concatenate(x) for x in (prev, init, slots))
    nt = len(prev)
    d_prev, d_init, d_slots = (torch.from_numpy(x).cuda() for x in (prev, init, slots))
    d_fwd = torch.zeros((nt, 2), dtype=torch.float32, device="cuda")
    d_bwd = torch.zeros((nt, 2), dtype=torch.float32, device="cuda")
    d_st = torch.zeros(nt, dtype=torch.uint8, device="cuda")
    a_lists = [random_lists(100 + f, n_feat[f], 0)[0] for f in range(NF)]
    d_a = torch.from_numpy(np.concatenate(a_lists)).cuda()
    torch.cuda.synchronize()
    trk.track_batch_dev(nt, d_slots.data_ptr(), d_prev.data_ptr(), d_init.data_ptr(), d_fwd.data_ptr(), d_bwd.data_ptr(), d_st.data_ptr(), 1)
    p1, p2, pitch = vp(), vp(), C.c_int()
    lib().icg_klt_slot_level0(trk._h, 1, C.byref(p1), C.byref(pitch))
    lib().icg_klt_slot_level0(trk._h, 2, C.byref(p2), C.byref(pitch))
    cols, rows, _, _, quota, _ = fo.grid(W, H, MAXF)
    per = cols * rows * quota
    out_xy = torch.zeros((NF, per, 2), dtype=torch.float32, device="cuda")
    out_n = torch.zeros(NF, dtype=torch.int32, device="cuda")
    dN = Detector(W, H, max_blocks=NF * 18, max_corners_per_block=32, max_roi_pixels=213 * 186, stream=s.cuda_stream)
    ismask = [1, 1, 0, 1, 1]
    dN.features_detection_dev(NF, p1.value, pitch.value, p2.value - p1.value, d_a.data_ptr(), 0, np.cumsum([0] + n_feat), d_fwd.data_ptr(),
                              d_st.data_ptr(), np.cumsum([0] + n_new), out_xy.data_ptr(), out_n.data_ptr(), ismask=ismask)
    s.synchronize()
    masks = [download(dN.mask_dev(f)[0], dN.mask_dev(f)[1], H, W) for f in range(NF)]
    got_n, got_xy = out_n.cpu().numpy(), out_xy.cpu().numpy()
    fwd, good = d_fwd.cpu().numpy(), d_st.cpu().numpy()
    dN.close()
    trk.close()
    d1 = Detector(W, H, max_blocks=18, max_corners_per_block=32)
    off = np.cumsum([0] + n_new)
    n_gated = 0
    for f in range(NF):
        b = fwd[off[f]:off[f + 1]][good[off[f]:off[f + 1]] != 0]
        ref = d1.features_detection_points(frames[f + 1], a_lists[f], b, ismask=bool(ismask[f]))
        gated = n_feat[f] + len(b) > MAXF - 5
        assert (ref is None) == gated and (got_n[f] == -1) == gated, (f, got_n[f], len(b))
        n_gated += gated
        if not gated:
            assert got_n[f] == len(ref) and np.array_equal(got_xy[f, :got_n[f]], ref), f
            assert np.array_equal(masks[f], download(*d1.mask_dev(0), H, W)), f
    d1.close()
    assert 0 < n_gated < NF


def test_argument_errors(img):
    from ic_gvins_b200 import IcgError
    from ic_gvins_b200.detect import Detector
    a, b = random_lists(7, 10, 10)
    d = Detector(W, H, max_blocks=18, max_corners_per_block=8)
    with pytest.raises(IcgError, match="code -1"):  # quota 17 > max_corners_per_block 8
        d.features_detection_points(img, a, b, max_features=MAXF)
    assert d.features_detection_points(img, a, b, max_features=120) is not None  # quota 7
    d.close()
    frames = torch.zeros((2, H, W), dtype=torch.uint8, device="cuda")
    pts = torch.from_numpy(b).cuda()
    out_xy = torch.zeros((2, 18 * 17, 2), dtype=torch.float32, device="cuda")
    out_n = torch.zeros(2, dtype=torch.int32, device="cuda")
    d = Detector(W, H, max_blocks=18, max_corners_per_block=32)
    args = (frames.data_ptr(), W, W * H, 0, 0)
    with pytest.raises(IcgError, match="code -1"):  # 2 frames x 18 blocks > max_blocks 18
        d.features_detection_dev(2, *args, [0, 0, 0], pts.data_ptr(), 0, [0, 5, 10], out_xy.data_ptr(), out_n.data_ptr())
    with pytest.raises(IcgError, match="code -1"):  # offsets not monotone
        d.features_detection_dev(1, *args, [0, 0], pts.data_ptr(), 0, [5, 3], out_xy.data_ptr(), out_n.data_ptr())
    with pytest.raises(IcgError, match="code -1"):
        d.features_detection_dev(1, *args, [-1, 0], pts.data_ptr(), 0, [0, 3], out_xy.data_ptr(), out_n.data_ptr())
    d.close()
    torch.cuda.synchronize()


SHIM = r'''
#include <cstdio>
#include <vector>
#include "ic_gvins_b200/host/icg_shims.hpp"

int main(int argc, char **argv) {
    try {
        FILE *in = fopen(argv[1], "rb"), *out = fopen(argv[2], "wb");
        int dim[6];  // W, H, n_feat, n_new, n_ref, ismask
        if (!in || !out || fread(dim, 4, 6, in) != 6) return 2;
        const int W = dim[0], H = dim[1];
        std::vector<uint8_t> img((size_t) W * H);
        std::vector<icg_b200::Point2f> feat(dim[2]), pts(dim[3]);
        if (fread(img.data(), 1, img.size(), in) != img.size() || fread(feat.data(), 8, feat.size(), in) != feat.size() ||
            fread(pts.data(), 8, pts.size(), in) != pts.size())
            return 2;
        icg_b200::Mat frame{img.data(), H, W, W};
        icg_b200::BlockDetector det(W, H, 18, 32, 213 * 186);
        bool skipped = false;
        std::vector<icg_b200::Point2f> c = det.featuresDetection(frame, feat, pts, dim[4], dim[5] != 0, 300, &skipped);
        const int n = skipped ? -1 : (int) c.size();
        fwrite(&n, 4, 1, out);
        if (!c.empty()) fwrite(c.data(), 8, c.size(), out);
        fclose(in), fclose(out);
        return 0;
    } catch (const std::exception &e) {
        fprintf(stderr, "shim test: %s\n", e.what());
        return 1;
    }
}
'''


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_cpp_shim_features_detection_equals_python(img):
    from ic_gvins_b200.detect import Detector
    lib = os.path.join(ROOT, "ic_gvins_b200", "libicgvins_b200.so")
    d = Detector(W, H, max_blocks=18, max_corners_per_block=32)
    with tempfile.TemporaryDirectory() as td:
        cpp, exe = os.path.join(td, "shim.cpp"), os.path.join(td, "shim")
        open(cpp, "w").write(SHIM)
        r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", ROOT, cpp, "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        for k, (n_feat, n_new, n_ref, ismask) in enumerate([(40, 120, 120, 1), (20, 100, 60, 0), (100, 200, 200, 1)]):
            a, b = random_lists(300 + k, n_feat, n_new)
            fin, fout = os.path.join(td, "in.bin"), os.path.join(td, "out.bin")
            with open(fin, "wb") as fh:
                fh.write(np.array([W, H, n_feat, n_new, n_ref, ismask], np.int32).tobytes() + img.tobytes() + a.tobytes() + b.tobytes())
            r = subprocess.run([exe, fin, fout], capture_output=True, text=True, timeout=300)
            assert r.returncode == 0, (r.returncode, r.stderr)
            raw = open(fout, "rb").read()
            n = int(np.frombuffer(raw[:4], np.int32)[0])
            ref = d.features_detection_points(img, a, b, n_ref=n_ref, ismask=bool(ismask))
            if ref is None:
                assert n == -1
            else:
                assert n == len(ref) and np.array_equal(np.frombuffer(raw[4:], np.float32).reshape(-1, 2), ref)
    d.close()
