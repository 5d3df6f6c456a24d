"""GPU: trackMappoint + trackReferenceFrame on the KLT handle (icg_klt_track_frame / icg_klt_track_frames_dev, IG/tracking/tracking.cc:351-574)
and the batched device RANSAC (icg_geom_find_fundamental_mat_ransac_batch).

- the batched RANSAC gives the masks of the host function icg_find_fundamental_mat_ransac on the golden scenes and on 200+ random sets in one call;
- the host call is bitwise the composition of existing ABI calls (icg_camera_*, icg_klt_track_fb, icg_find_fundamental_mat_ransac) plus numpy
  compaction and fixed-order products;
- the device call for 64+ streams of mixed sizes equals the host call stream by stream, bitwise;
- against the C oracle's LK: statuses equal, positions within 1e-3 px;
- chained with no sync, the device call's keep flags and positions drive icg_detect_features_dev to the corners of host-compacted lists."""
import ctypes as C
import os

import numpy as np
import pytest

from datagen import synth_klt as synth
from oracle import camera_ref as cref
from tests import oracle_api as oa
from tests import tracking_oracle as to

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
W, H = 1280, 560
INTR = [460.0, 455.0, 640.0, 280.0, 0.0]
DIST = [-0.05, 0.01, 1e-4, -2e-5, 0.0]
MAXP = 64 * 400


def Rz(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])


class AbiCam:
    """the oracle/camera_ref.py interface on the library's host entry points (icg_camera_*)"""

    @staticmethod
    def _c(cam):
        from ic_gvins_b200.camera import Camera
        return Camera([cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["skew"]], [cam["k1"], cam["k2"], cam["p1"], cam["p2"], cam["k3"]])

    def undistort_points(self, cam, px):
        return self._c(cam).undistortPoints(px) if len(px) else np.zeros((0, 2), np.float32)

    def distort_points(self, cam, px):
        return self._c(cam).distortPoints(px) if len(px) else np.zeros((0, 2), np.float32)

    def distort_camera_point(self, cam, pc):
        return self._c(cam).distortCameraPoint(pc) if len(pc) else np.zeros((0, 2), np.float32)

    def pixel2cam(self, cam, px):
        return self._c(cam).pixel2cam(px) if len(px) else np.zeros((0, 3))

    def world2pixel(self, cam, pw, R, t):
        return self._c(cam).world2pixel(pw, R, t) if len(pw) else np.zeros((0, 2), np.float32)


def host_ransac(p1, p2, thr):
    from ic_gvins_b200.camera import findFundamentalMat
    return findFundamentalMat(p1, p2, thr, 0.99)[1] != 0


@pytest.fixture(scope="module")
def stream():
    return synth.KltStream(W, H, 400, 1234)


@pytest.fixture(scope="module")
def trk(stream):
    from ic_gvins_b200.klt import KltTracker
    t = KltTracker(W, H, n_slots=4, max_points=MAXP)
    for s, f in enumerate((0, 1, 2)):
        t.upload(s, stream.frame(f))
    t.sync()
    yield t
    t.close()


@pytest.fixture(scope="module")
def host_klt():
    from ic_gvins_b200.klt import KltTracker
    t = KltTracker(W, H, n_slots=4, max_points=4096)
    yield t
    t.close()


def make_case(stream, t, nm, nr, seed, ref_id=7, yaw=0.0):
    """map list: pw back-projected at depth 4 from the true current position (identity pose), ref_kp for every other point; reference list
    with frame ids around ref_id and random reference velocities"""
    rng = np.random.default_rng(seed)
    cam = to.cam_dict(INTR, DIST)
    p0, p1 = stream.points(t - 1).astype(np.float32), stream.points(t).astype(np.float32)
    idx = rng.permutation(len(p0))
    mi, ri = idx[:nm], idx[nm:nm + nr]
    pc = cref.pixel2cam(cam, cref.undistort_points(cam, p1[mi]))
    pw = pc * 4.0
    rk = cref.undistort_points(cam, p0[mi] + rng.normal(0, 2, (nm, 2)).astype(np.float32))
    rk[::2] = np.nan
    ml = dict(prev_xy=p0[mi], prev_undis_xy=cref.undistort_points(cam, p0[mi]), pw=pw, ref_kp_xy=rk) if nm else None
    rl = dict(new_xy=p0[ri], ref_xy=(p0[ri] + rng.normal(0, 3, (nr, 2))).astype(np.float32), ref_frame_id=rng.integers(ref_id - 2, ref_id + 3, nr),
              velocity_ref=rng.normal(0, 0.5, (nr, 2))) if nr else None
    P = dict(intrinsic=INTR, distortion=DIST, R_pre=Rz(yaw), R_cur=Rz(yaw), R_ref=Rz(0.003), t_cur=np.zeros(3), dt=0.05 + 0.01 * (seed % 3),
             ref_id=ref_id, fm_threshold=1.0 + 0.5 * (seed % 2))
    return P, ml, rl


def params_struct(P, prev_slot, cur_slot):
    from ic_gvins_b200.klt import track_frame_params
    return track_frame_params(prev_slot, cur_slot, P["intrinsic"], P["distortion"], P["R_pre"], P["R_cur"], P["R_ref"], P["t_cur"], P["dt"],
                              P["ref_id"], P["fm_threshold"])


def assert_same(a, b, what):
    for k in ("fwd_xy", "fwd_undis_xy", "keep", "cur_xy", "cur_undis_xy", "velocity", "src", "ref_out_xy", "ref_frame_id_out", "velocity_ref_out"):
        if k in b:
            assert np.array_equal(np.asarray(a[k]).reshape(np.asarray(b[k]).shape), b[k]), f"{what}: {k}"


# ------------------------------------------------------------------------------------------------ batched RANSAC
def test_batched_ransac_masks_equal_host_function():
    import importlib.util
    from ic_gvins_b200.camera import findFundamentalMat
    from ic_gvins_b200.geom import Geometry
    spec = importlib.util.spec_from_file_location("mk", os.path.join(GOLD, "make_fundamental_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    try:
        spec.loader.exec_module(mk)
    except ImportError:
        pytest.skip("cv2 not importable (the scene generator lives in the golden script)")
    g = np.load(os.path.join(GOLD, "fundamental_golden.npz"))
    sets, thr = [], []
    for name in sorted(k[:-3] for k in g.files if k.endswith("_p1")):
        # the golden arrays are not all C-ordered: the device reads interleaved (x, y) pairs
        sets.append((np.ascontiguousarray(g[name + "_p1"], np.float32), np.ascontiguousarray(g[name + "_p2"], np.float32))), thr.append(float(g[name + "_thr"][0]))
    rng = np.random.default_rng(77)
    for k in range(200):
        n = [14, 15][k] if k < 2 else int(rng.integers(15, 301))
        p1, p2 = mk.scene(rng, n, int(rng.uniform(0, 0.4) * n), 0.3, float(rng.uniform(0.0, 0.15)), (0.5, float(rng.uniform(-0.1, 0.1)), 0.1))
        if k % 25 == 3:  # collinear-degenerate: every point of image 1 on one line (no drawable subset)
            p1[:, 1] = np.float32(200.0)
        if k % 25 == 4:  # half of the points collinear in image 2 (re-draws)
            p2[: n // 2, 1] = np.float32(100.0)
        sets.append((p1, p2)), thr.append(float(rng.uniform(0.5, 3.0)))
    off = np.zeros(len(sets) + 1, np.int32)
    off[1:] = np.cumsum([len(a) for a, _ in sets])
    P1 = torch.from_numpy(np.ascontiguousarray(np.concatenate([a for a, _ in sets]))).cuda()
    P2 = torch.from_numpy(np.ascontiguousarray(np.concatenate([b for _, b in sets]))).cuda()
    mask = torch.full((int(off[-1]),), 7, dtype=torch.uint8, device="cuda")
    ninl = torch.zeros(len(sets), dtype=torch.int32, device="cuda")
    stats = torch.zeros((len(sets), 3), dtype=torch.int64, device="cuda")
    geom = Geometry()
    torch.cuda.synchronize()  # the handle works on its own stream
    try:
        geom.findFundamentalMat_batch_dev(off, P1.data_ptr(), P2.data_ptr(), mask.data_ptr(), ninl.data_ptr(), thresholds=thr, dev_stats=stats.data_ptr())
        torch.cuda.synchronize()
        m, ni, stt = mask.cpu().numpy(), ninl.cpu().numpy(), stats.cpu().numpy()
        n_zero = 0
        for s, ((a, b), th) in enumerate(zip(sets, thr)):
            got = m[off[s]:off[s + 1]]
            want = findFundamentalMat(a, b, th, 0.99)[1] if len(a) >= 15 else np.zeros(len(a), np.uint8)
            assert np.array_equal(got, want), f"set {s} (n = {len(a)})"
            assert ni[s] == int(want.sum())
            n_zero += int(want.sum() == 0)
        assert n_zero >= 8  # n = 14 and the degenerate sets
        assert (stt[:, 0] >= 0).all() and stt[:, 0].max() <= 1000
    finally:
        geom.close()


# ------------------------------------------------------------------------------------------------ host call
def test_host_call_is_the_composition_of_abi_calls(trk, host_klt, stream):
    a, b = stream.frame(0), stream.frame(1)
    lk = lambda x, y, p, init: host_klt.track_fb(x, y, p, init)[::2]  # noqa: E731
    for seed, (nm, nr, yaw) in enumerate([(100, 200, 0.0), (40, 0, 0.0), (0, 150, 0.004), (120, 14, 0.0), (3, 300, -0.002)]):
        P, ml, rl = make_case(stream, 1, nm, nr, seed, yaw=yaw)
        got = trk.track_frame(params_struct(P, 0, 1), ml, rl)
        want = to.track_frame(lk, a, b, P, ml, rl, ransac=host_ransac, ops=AbiCam())
        assert np.array_equal(got[2], want[2]), (seed, got[2], want[2])
        assert np.array_equal(got[4], want[4]), seed
        assert np.array_equal(got[3], want[3]), (seed, got[3], want[3])  # same sum order, IEEE sqrt / division: bitwise
        if nm:
            assert_same(got[0], want[0], f"case {seed} map")
        if nr:
            assert_same(got[1], want[1], f"case {seed} ref")
        assert got[2][0] == nm or nm == 0 or got[2][0] > 0.8 * nm


def test_host_call_against_oracle_lk(trk, oracle, stream):
    a, b = stream.frame(0), stream.frame(1)
    lk = lambda x, y, p, init: oa.track_fb(oracle, x, y, p, init)[::2]  # noqa: E731
    P, ml, rl = make_case(stream, 1, 100, 250, 11)
    got = trk.track_frame(params_struct(P, 0, 1), ml, rl)
    want = to.track_frame(lk, a, b, P, ml, rl)
    for k in (0, 1):
        assert np.array_equal(got[k]["keep"], want[k]["keep"]), k
        assert np.abs(got[k]["cur_xy"] - want[k]["cur_xy"]).max() <= 1e-3
    assert np.array_equal(got[2], want[2]) and np.array_equal(got[4], want[4])
    assert np.abs(got[3] - want[3]).max() <= 1e-3


# ------------------------------------------------------------------------------------------------ device call
def dev_lists(cases):
    """concatenate the streams' lists into device tensors (+ output tensors) and host offsets"""
    from ic_gvins_b200.klt import MAP_IN, MAP_OUT, REF_IN, REF_OUT, _SPEC
    out = {}
    for which, names_in, names_out, key in (("map", MAP_IN, MAP_OUT, 1), ("ref", REF_IN, REF_OUT, 2)):
        lens = [len(c[key][names_in[0]]) if c[key] else 0 for c in cases]
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        N = max(int(off[-1]), 1)
        tens = {}
        for k in names_in:
            dt, col = _SPEC[k]
            parts = [np.asarray(c[key][k], dt).reshape(-1, col) for c in cases if c[key]]
            arr = np.concatenate(parts) if parts else np.zeros((1, col), dt)
            tens[k] = torch.from_numpy(np.ascontiguousarray(arr)).cuda()
        for k in names_out:
            dt, col = _SPEC[k]
            tens[k] = torch.zeros((N, col), dtype=getattr(torch, np.dtype(dt).name), device="cuda")
        out[which] = (off, tens, {k: v.data_ptr() for k, v in tens.items()} if off[-1] else None)
    torch.cuda.synchronize()  # the KLT handle works on its own stream
    return out


def test_device_call_equals_host_call_per_stream(trk, stream):
    rng = np.random.default_rng(2026)
    sizes = [(0, 0), (0, 120), (60, 0), (14, 14), (15, 15), (16, 15), (5, 17)]
    cases = []
    for s in range(72):
        nm, nr = sizes[s] if s < len(sizes) else (int(rng.integers(0, 150)), int(rng.integers(0, 250)))
        P, ml, rl = make_case(stream, 1 + s % 2, nm, nr, 100 + s, yaw=float(rng.uniform(-0.003, 0.003)))
        if s == 8:  # every point lost: pushed off the frame
            ml = dict(ml or {})
            for k in ("prev_xy",):
                if ml:
                    ml[k] = np.full_like(ml[k], -50.0)
            if rl:
                rl = dict(rl, new_xy=np.full_like(rl["new_xy"], -50.0))
        cases.append((P, ml, rl, s % 2, 1 + s % 2))
    D = dev_lists([(c[0], c[1], c[2]) for c in cases])
    B = len(cases)
    n_out = torch.zeros(2 * B, dtype=torch.int32, device="cuda")
    par = torch.zeros(2 * B, dtype=torch.float64, device="cuda")
    par_n = torch.zeros(2 * B, dtype=torch.int32, device="cuda")
    trk.track_frames_dev([params_struct(c[0], c[3], c[4]) for c in cases], D["map"][0], D["map"][2], D["ref"][0], D["ref"][2],
                         n_out.data_ptr(), par.data_ptr(), par_n.data_ptr())
    trk.sync()
    n_out, par, par_n = n_out.cpu().numpy(), par.cpu().numpy(), par_n.cpu().numpy()
    for s, (P, ml, rl, ps, cs) in enumerate(cases):
        h = trk.track_frame(params_struct(P, ps, cs), ml, rl)
        assert np.array_equal(n_out[2 * s:2 * s + 2], h[2]), s
        assert np.array_equal(par[2 * s:2 * s + 2], h[3]), s
        assert np.array_equal(par_n[2 * s:2 * s + 2], h[4]), s
        for which, hk in (("map", 0), ("ref", 1)):
            off, tens, _ = D[which]
            a0, a1 = int(off[s]), int(off[s + 1])
            if a1 == a0:
                continue
            k_out = int(h[2][hk])
            for k, v in h[hk].items():
                d = tens[k].cpu().numpy()
                d = d[a0:a1] if k in ("fwd_xy", "fwd_undis_xy", "keep") else d[a0:a0 + k_out]
                assert np.array_equal(d.reshape(np.asarray(v).shape), v), (s, which, k)
    assert any(par_n[1::2] == -1) and any(par_n[0::2] == -1)


def test_chained_detection_equals_host_compacted_lists(trk, stream):
    from ic_gvins_b200.detect import Detector
    from ic_gvins_b200.klt import KltTracker  # noqa: F401
    B = 4
    cases = [make_case(stream, 1, 40 + 10 * s, 100 + 20 * s, 300 + s) for s in range(B)]
    D = dev_lists(cases)
    n_out = torch.zeros(2 * B, dtype=torch.int32, device="cuda")
    par = torch.zeros(2 * B, dtype=torch.float64, device="cuda")
    par_n = torch.zeros(2 * B, dtype=torch.int32, device="cuda")
    # every stream detects on slot 1 (frame 1): the frames are B copies of the slot's level-0 plane
    ptr, pitch = C.c_void_p(), C.c_int()
    from ic_gvins_b200._lib import lib
    lib().icg_klt_slot_level0(trk._h, 1, C.byref(ptr), C.byref(pitch))
    frames = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(stream.frame(1), (B, H, W)))).cuda()
    det = Detector(W, H, max_blocks=B * 32, max_corners_per_block=64, stream=None)
    try:
        from ic_gvins_b200.detect import block_rois
        rois, quota, _, grid = block_rois(W, H, 300)
        cap = len(rois) * quota
        out_a = torch.zeros((B, cap, 2), dtype=torch.float32, device="cuda")
        n_a = torch.zeros(B, dtype=torch.int32, device="cuda")
        out_b = torch.zeros_like(out_a)
        n_b = torch.zeros_like(n_a)
        trk.track_frames_dev([params_struct(P, 0, 1) for P, _, _ in cases], D["map"][0], D["map"][2], D["ref"][0], D["ref"][2],
                             n_out.data_ptr(), par.data_ptr(), par_n.data_ptr())
        trk.sync()  # the detector runs on its own stream
        mo, mt, _ = D["map"]
        ro, rt, _ = D["ref"]
        det.features_detection_dev(B, frames.data_ptr(), W, W * H, mt["fwd_undis_xy"].data_ptr(), mt["keep"].data_ptr(), mo,
                                   rt["fwd_xy"].data_ptr(), rt["keep"].data_ptr(), ro, out_a.data_ptr(), n_a.data_ptr())
        # the same detection from host-compacted lists
        no = n_out.cpu().numpy()
        fa = [mt["cur_undis_xy"].cpu().numpy()[mo[s]:mo[s] + no[2 * s]] for s in range(B)]
        fb = [rt["cur_xy"].cpu().numpy()[ro[s]:ro[s] + no[2 * s + 1]] for s in range(B)]
        ao = np.concatenate([[0], np.cumsum([len(x) for x in fa])]).astype(np.int32)
        bo = np.concatenate([[0], np.cumsum([len(x) for x in fb])]).astype(np.int32)
        A_ = torch.from_numpy(np.concatenate(fa)).cuda()
        B_ = torch.from_numpy(np.concatenate(fb)).cuda()
        torch.cuda.synchronize()
        det.features_detection_dev(B, frames.data_ptr(), W, W * H, A_.data_ptr(), 0, ao, B_.data_ptr(), 0, bo, out_b.data_ptr(), n_b.data_ptr())
        torch.cuda.synchronize()
        na, nb = n_a.cpu().numpy(), n_b.cpu().numpy()
        assert np.array_equal(na, nb)
        assert (na > 0).all()
        for s in range(B):
            assert np.array_equal(out_a[s, :na[s]].cpu().numpy(), out_b[s, :nb[s]].cpu().numpy()), s
    finally:
        det.close()


def test_argument_errors(trk):
    from ic_gvins_b200 import IcgError
    P, ml, rl = make_case(synth.KltStream(W, H, 50, 5), 1, 10, 10, 1)
    with pytest.raises(IcgError, match="bad slot"):
        trk.track_frame(params_struct(P, 0, 9), ml, rl)
    with pytest.raises(IcgError, match="monotone|start at 0"):
        trk.track_frames_dev([params_struct(P, 0, 1)], [0, 0], None, [1, 0], {"new_xy": 1}, 1, 1, 1)
    with pytest.raises(IcgError, match="NULL list pointer"):
        trk.track_frames_dev([params_struct(P, 0, 1)], [0, 3], None, [0, 0], None, 1, 1, 1)
    with pytest.raises(IcgError, match="exceed max_points"):
        trk.track_frames_dev([params_struct(P, 0, 1)], [0, MAXP + 1], {k: 1 for k in ("prev_xy", "prev_undis_xy", "pw", "ref_kp_xy", "fwd_xy",
                                                                                       "fwd_undis_xy", "keep", "cur_xy", "cur_undis_xy", "velocity", "src")},
                             [0, 0], None, 1, 1, 1)


SHIM_SRC = r"""
#include <cmath>
#include <cstdio>
#include <cstring>
#include "ic_gvins_b200/host/icg_shims.hpp"
template <class T> std::vector<T> rd(FILE *f) { int64_t n; fread(&n, 8, 1, f); std::vector<T> v(n); fread(v.data(), sizeof(T), n, f); return v; }
template <class T> void wr(FILE *f, const std::vector<T> &v) { int64_t n = v.size(); fwrite(&n, 8, 1, f); fwrite(v.data(), sizeof(T), n, f); }
int main(int, char **argv) {
    FILE *f = fopen(argv[1], "rb");
    auto wh = rd<int32_t>(f);
    auto f0 = rd<uint8_t>(f), f1 = rd<uint8_t>(f);
    auto pb = rd<uint8_t>(f);
    icg_track_frame p;
    memcpy(&p, pb.data(), sizeof(p));
    auto mp = rd<icg_b200::Point2f>(f), mu = rd<icg_b200::Point2f>(f), rk = rd<icg_b200::Point2f>(f);
    auto pw = rd<double>(f);
    auto nw = rd<icg_b200::Point2f>(f), rf = rd<icg_b200::Point2f>(f);
    auto id = rd<int64_t>(f);
    auto vr = rd<double>(f);
    fclose(f);
    icg_b200::KltContext k(wh[0], wh[1], 4096);
    icg_b200::Mat a{f0.data(), wh[1], wh[0], wh[0]}, b{f1.data(), wh[1], wh[0], wh[0]};
    std::vector<icg_b200::Point2f> m, mu2;
    std::vector<double> vel, vcur;
    std::vector<int32_t> src, src2;
    double pm = -7, pr = -7;
    int cm = -7, cr = -7;
    bool okm = k.trackMappoint(a, b, p, mp, mu, pw, rk, m, mu2, vel, src, pm, cm);
    bool okr = k.trackReferenceFrame(a, b, p, nw, rf, id, vr, vcur, src2, pr, cr);
    FILE *o = fopen(argv[2], "wb");
    wr(o, m), wr(o, mu2), wr(o, vel), wr(o, src), wr(o, nw), wr(o, rf), wr(o, id), wr(o, vr), wr(o, vcur), wr(o, src2);
    wr(o, std::vector<double>{pm, pr, (double) cm, (double) cr, (double) okm, (double) okr});
    fclose(o);
    return 0;
}
"""


def test_cpp_shims_track_mappoint_and_reference_frame(trk, stream):
    import shutil
    import subprocess
    import tempfile
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    lib = os.path.join(ROOT, "ic_gvins_b200", "libicgvins_b200.so")
    P, ml, rl = make_case(stream, 1, 90, 180, 41)
    ps = params_struct(P, 0, 1)
    hm = trk.track_frame(ps, ml, None)
    hr = trk.track_frame(ps, None, rl)

    def wr(fh, a):
        a = np.ascontiguousarray(a)
        fh.write(np.int64(a.size if a.dtype != np.float32 or a.ndim == 1 else a.shape[0]).tobytes())
        fh.write(a.tobytes())
    with tempfile.TemporaryDirectory() as td:
        cpp, exe, fin, fout = (os.path.join(td, x) for x in ("s.cpp", "s", "in.bin", "out.bin"))
        open(cpp, "w").write(SHIM_SRC)
        r = subprocess.run(["g++", "-std=c++17", "-O1", "-I", ROOT, cpp, "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        with open(fin, "wb") as fh:
            wr(fh, np.array([W, H], np.int32)), wr(fh, stream.frame(0)), wr(fh, stream.frame(1))
            wr(fh, np.frombuffer(bytes(ps), np.uint8))
            for k in ("prev_xy", "prev_undis_xy", "ref_kp_xy"):
                wr(fh, np.asarray(ml[k], np.float32))
            wr(fh, np.asarray(ml["pw"], np.float64).reshape(-1))
            wr(fh, np.asarray(rl["new_xy"], np.float32)), wr(fh, np.asarray(rl["ref_xy"], np.float32))
            wr(fh, np.asarray(rl["ref_frame_id"], np.int64)), wr(fh, np.asarray(rl["velocity_ref"], np.float64).reshape(-1))
        r = subprocess.run([exe, fin, fout], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, (r.returncode, r.stderr)
        out = []
        with open(fout, "rb") as fh:
            for dt in (np.float32, np.float32, np.float64, np.int32, np.float32, np.float32, np.int64, np.float64, np.float64, np.int32, np.float64):
                n = int(np.frombuffer(fh.read(8), np.int64)[0])
                w = 2 if dt == np.float32 else 1
                out.append(np.frombuffer(fh.read(n * w * np.dtype(dt).itemsize), dt))
    m, r_ = hm[0], hr[1]
    assert np.array_equal(out[0].reshape(-1, 2), m["cur_xy"]) and np.array_equal(out[1].reshape(-1, 2), m["cur_undis_xy"])
    assert np.array_equal(out[2].reshape(-1, 2), m["velocity"]) and np.array_equal(out[3], m["src"])
    assert np.array_equal(out[4].reshape(-1, 2), r_["cur_xy"]) and np.array_equal(out[5].reshape(-1, 2), r_["ref_out_xy"])
    assert np.array_equal(out[6], r_["ref_frame_id_out"]) and np.array_equal(out[7].reshape(-1, 2), r_["velocity_ref_out"])
    assert np.array_equal(out[8].reshape(-1, 2), r_["velocity"]) and np.array_equal(out[9], r_["src"])
    pm, pr, cm, cr, okm, okr = out[10]
    assert (pm, cm) == (hm[3][0], hm[4][0]) and (pr, cr) == (hr[3][1], hr[4][1]) and okm == 1 and okr == 1
