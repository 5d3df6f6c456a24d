"""GPU: Tracking::triangulation on the KLT handle (icg_klt_triangulate / icg_klt_triangulate_dev, IG/tracking/tracking.cc:690-798).

- the host call is bitwise the composition of existing ABI calls (icg_camera_*, icg_triangulate_points) plus fixed-order products, including
  reprojection gates that only the float difference of camera.cc:156 admits;
- the device call over 72 streams of mixed sizes equals the host call stream by stream, bitwise; streams with triangulate = 0 and a stream
  naming a frame missing from its table come back byte for byte unchanged;
- against the numpy oracle (SVD triangulation) the decisions are equal away from knife edges and pw agrees to 1e-9 relative;
- chained after icg_klt_track_frames_dev with no host sync (counts read from dev_n_out on the device) the result equals running both calls on
  host-compacted lists;
- argument errors, and the C++ shim KltContext::triangulation."""
import os

import numpy as np
import pytest

from oracle import camera_ref as cref
from tests import triangulation_oracle as tri
from tests.tracking_oracle import cam_dict

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INTR = [460.0, 455.0, 640.0, 280.0, 0.0]
DIST = [-0.05, 0.01, 1e-4, -2e-5, 0.0]
REF_ID, CUR_ID = 50, 53


def Ry(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def Rz(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])


def make_stream(rng, n, window_normal=False, std=1.5, n_kf=10, triangulate=True, intr=INTR, dist=DIST):
    """one stream's parameters, table and list: a known mix of resets, out-of-window points, low parallax, outliers (pixel noise and points
    too near) and successes"""
    cam = cam_dict(intr, dist)
    ids = [REF_ID - 3 * j for j in range(n_kf)]
    kfs = {fid: (Ry(0.01 * j) @ Rz(0.005 * j), np.array([-0.25 * j, 0.03 * j, 0.08 * j]), j < n_kf - 3) for j, fid in enumerate(ids)}
    R_cur, t_cur = Ry(-0.015), np.array([0.35 + rng.uniform(0, 0.2), 0.04, 0.1])
    P = dict(intrinsic=intr, distortion=dist, R_cur=R_cur, t_cur=t_cur, cur_id=CUR_ID, ref_id=REF_ID, window_normal=window_normal,
             reprojection_error_std=std, triangulate=triangulate)
    fid = np.array([ids[int(rng.integers(0, n_kf))] if rng.uniform() < 0.85 else REF_ID + int(rng.integers(1, 3)) for _ in range(n)], np.int64)
    pw = np.stack([rng.uniform(-5, 5, n), rng.uniform(-2, 2, n), rng.uniform(3, 40, n)], 1)
    pw[rng.uniform(size=n) < 0.05, 2] = 0.6
    ref, cur = np.zeros((n, 2), np.float32), np.zeros((n, 2), np.float32)
    for k in range(n):
        R0, t0, _ = kfs[int(fid[k])] if fid[k] <= REF_ID else (R_cur, t_cur, True)
        ref[k] = cref.cam2pixel(cam, np.array([tri.world2cam(pw[k], R0, t0)]))[0]
        cur[k] = cref.cam2pixel(cam, np.array([tri.world2cam(pw[k], R_cur, t_cur)]))[0]
    sig = np.where(rng.uniform(size=(n, 1)) < 0.1, 4.0, 0.3)
    ref = cref.distort_points(cam, ref + rng.normal(0, 1, (n, 2)) * sig).astype(np.float32)
    cur = cref.distort_points(cam, cur + rng.normal(0, 1, (n, 2)) * sig).astype(np.float32)
    L = dict(ref_out_xy=ref, ref_frame_id_out=fid, cur_xy=cur, velocity_ref_out=rng.normal(0, 0.5, (n, 2)), velocity=rng.normal(0, 0.5, (n, 2)))
    return P, kfs, L


def struct(P):
    from ic_gvins_b200.klt import tri_frame_params
    return tri_frame_params(P["intrinsic"], P["distortion"], P["R_cur"], P["t_cur"], P["cur_id"], P["ref_id"], P["window_normal"],
                            P["reprojection_error_std"], P.get("triangulate", True))


def kf_rows(kfs):
    return [(fid, R, t, m) for fid, (R, t, m) in kfs.items()]


@pytest.fixture(scope="module")
def klt():
    from ic_gvins_b200.klt import KltTracker
    t = KltTracker(640, 480, n_slots=2, max_points=4096)
    yield t
    t.close()


def assert_result(got, want, what):
    lo, no, cnt = got
    wl, wn, wc = want[:3]
    assert np.array_equal(cnt, wc), (what, cnt, wc)
    for k, v in wl.items():
        assert np.array_equal(np.asarray(lo[k]).reshape(np.asarray(v).shape), v), (what, k)
    for k, v in wn.items():
        assert np.array_equal(np.asarray(no[k]).reshape(np.asarray(v).shape), v), (what, k)


# ------------------------------------------------------------------------------------------------ host call
def test_host_call_is_the_composition_of_abi_calls(klt):
    rng = np.random.default_rng(5)
    branches = np.zeros(5, np.int64)
    for case in range(8):
        P, kfs, L = make_stream(rng, 300, window_normal=case % 2 == 1, std=1.0 + 0.25 * case)
        got = klt.triangulate(struct(P), kf_rows(kfs), L)
        want = tri.triangulation(P, kfs, L, ops=tri.AbiOps(), tri=tri.abi_triangulate)
        assert_result(got, want, case)
        branches += np.maximum(got[2], 0)
    assert (branches > 0).all(), branches  # every branch ran
    print("host call branches (kept, succeeded, outlier, reset, outtime):", branches.tolist())


def test_reprojection_gate_decided_by_the_float_difference(klt):
    from tests.test_oracle_triangulation import KF, float_double_cases, params
    P = params((1, 0, 0))
    hits = 0
    for L, std in float_double_cases(P, KF, 300, 3):
        Q = dict(P, reprojection_error_std=std)
        got = klt.triangulate(struct(Q), kf_rows(KF), L)
        assert list(got[2]) == [0, 1, 0, 0, 0]  # admitted at the float error; a double difference exceeds std
        assert_result(got, tri.triangulation(Q, KF, L, ops=tri.AbiOps(), tri=tri.abi_triangulate), "float gate")
        got = klt.triangulate(struct(dict(P, reprojection_error_std=np.nextafter(std, 0))), kf_rows(KF), L)
        assert list(got[2]) == [0, 0, 1, 0, 0]
        hits += 1
    assert hits >= 3


def test_host_call_against_numpy_oracle(klt):
    rng = np.random.default_rng(9)
    edges, n_pw = 0, 0
    for case in range(6):
        P, kfs, L = make_stream(rng, 300, window_normal=case % 2 == 0)
        lo, no, cnt = klt.triangulate(struct(P), kf_rows(kfs), L)
        wl, wn, wc, st, diag = tri.triangulation(P, kfs, L)
        got_st = np.zeros(len(st), np.int32)
        got_st[lo["src"]] = 1
        got_st[no["src"]] = 2
        differ = np.nonzero(got_st != st)[0]
        for k in differ:
            assert tri.knife_edge(diag[k]), (case, k, diag[k])
        edges += len(differ)
        both = np.intersect1d(no["src"], wn["src"])
        a = no["pw"][np.searchsorted(no["src"], both)]
        b = wn["pw"][np.searchsorted(wn["src"], both)]
        assert np.abs(a - b).max() <= 1e-9 * np.abs(b).max(), case
        n_pw += len(both)
    assert n_pw >= 100
    print(f"numpy oracle: {n_pw} map points compared, {edges} decisions within 1e-9 of a threshold")


# ------------------------------------------------------------------------------------------------ device call
def to_dev(arrs, names, spec, n_rows):
    out = {}
    for k in names:
        dt, c = spec[k]
        a = arrs.get(k)
        a = np.zeros((max(n_rows, 1), c), dt) if a is None or n_rows == 0 else np.ascontiguousarray(np.asarray(a, dt).reshape(n_rows, c))
        out[k] = torch.from_numpy(a.copy()).cuda()
    return out


def concat_lists(cases):
    from ic_gvins_b200.klt import TRI_LIST, _SPEC
    lens = [len(c[2]["cur_xy"]) if c[2] else 0 for c in cases]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    arrs = {}
    for k in TRI_LIST:
        if k == "src":
            continue
        dt, col = _SPEC[k]
        parts = [np.asarray(c[2][k], dt).reshape(-1, col) for c in cases if c[2] and len(c[2]["cur_xy"])]
        arrs[k] = np.concatenate(parts) if parts else None
    return off, arrs


def run_dev(klt, cases, dev_n_in=None, stride=1, lists=None):
    """cases: (P, kfs, L); returns (list tensors, new tensors, counts (B, 5), ref_off) after a synchronising read"""
    from ic_gvins_b200.klt import _SPEC, _TRI_NEW_SPEC, TRI_LIST
    off, arrs = concat_lists(cases)
    N = int(off[-1])
    lt = lists if lists is not None else to_dev(arrs, TRI_LIST, _SPEC, N)
    nt = {k: torch.zeros((N, c), dtype=getattr(torch, np.dtype(dt).name), device="cuda") for k, (dt, c) in _TRI_NEW_SPEC.items()} if N else {}
    counts = torch.full((len(cases), 5), 99, dtype=torch.int32, device="cuda")
    kf_off = np.concatenate([[0], np.cumsum([len(c[1]) for c in cases])]).astype(np.int32)
    rows = [r for c in cases for r in kf_rows(c[1])]
    torch.cuda.synchronize()  # the KLT handle works on its own stream
    klt.triangulate_dev([struct(c[0]) for c in cases], kf_off, rows, off, dev_n_in or 0, stride, {k: v.data_ptr() for k, v in lt.items()} if N else None,
                        {k: v.data_ptr() for k, v in nt.items()} if N else None, counts.data_ptr())
    klt.sync()
    return lt, nt, counts.cpu().numpy(), off


def test_device_call_equals_host_call_per_stream(klt):
    from ic_gvins_b200.klt import TRI_NEW
    rng = np.random.default_rng(2026)
    sizes = [0, 1, 255, 256, 257, 300, 300, 2, 40]
    cases = []
    for s in range(72):
        n = sizes[s] if s < len(sizes) else (120 if s == 11 else int(rng.integers(0, 320)))
        P, kfs, L = make_stream(rng, n, window_normal=s % 3 == 0, std=1.0 + 0.5 * (s % 3), n_kf=10 if s % 5 else 4, triangulate=s % 7 != 3)
        if s == 11:  # a point naming a frame that is not in the table
            kfs = {k: v for k, v in kfs.items() if k != REF_ID}
            L["ref_frame_id_out"][n // 2] = REF_ID
        cases.append((P, kfs, L))
    before = {k: v.copy() for k, v in concat_lists(cases)[1].items()}
    lt, nt, counts, off = run_dev(klt, cases)
    lists = {k: v.cpu().numpy() for k, v in lt.items()}
    news = {k: v.cpu().numpy() for k, v in nt.items()}
    seen = set()
    for s, (P, kfs, L) in enumerate(cases):
        a0, a1 = int(off[s]), int(off[s + 1])
        h = klt.triangulate(struct(P), kf_rows(kfs), L)
        assert np.array_equal(counts[s], h[2]), (s, counts[s], h[2])
        if counts[s][0] < 0:  # untouched: empty list, triangulate == 0, or a missing frame
            seen.add(int(counts[s][0]) if a1 > a0 else 0)
            for k, v in before.items():
                assert lists[k][a0:a1].tobytes() == v.reshape(lists[k].shape)[a0:a1].tobytes(), (s, k)
            continue
        kk, mm = int(counts[s][0]), int(counts[s][1])
        for k, v in h[0].items():
            assert np.array_equal(lists[k][a0:a0 + kk].reshape(np.asarray(v).shape), v), (s, k)
        for k in TRI_NEW:
            assert np.array_equal(news[k][a0:a0 + mm].reshape(np.asarray(h[1][k]).shape), h[1][k]), (s, k)
    assert {0, -1, -2} <= seen, seen
    assert counts[11][0] == -2


def test_chained_after_the_tracking_step_without_host_sync(klt):
    from datagen import synth_klt as synth
    from ic_gvins_b200.klt import _TRI_NEW_SPEC, TRI_NEW, KltTracker
    from tests.test_track_frame_gpu import H, MAXP, W, dev_lists, make_case, params_struct
    stream = synth.KltStream(W, H, 400, 1234)
    trk = KltTracker(W, H, n_slots=4, max_points=MAXP)
    try:
        for s, f in enumerate((0, 1, 2)):
            trk.upload(s, stream.frame(f))
        trk.sync()
        B = 6
        tcases = [make_case(stream, 1 + s % 2, 30, 150 + 20 * s, 500 + s, ref_id=7) for s in range(B)]
        rng = np.random.default_rng(4)
        tri_cases = []
        for s in range(B):
            kfs = {fid: (Ry(0.004 * j), np.array([-0.2 * j - 0.1, 0.0, 0.02 * j]), j != 1) for j, fid in enumerate((7, 6, 5))}
            P = dict(intrinsic=INTR, distortion=DIST, R_cur=Ry(0.002), t_cur=np.array([0.5 + 0.1 * s, 0.0, 0.05]), cur_id=9, ref_id=7,
                     window_normal=s % 2 == 0, reprojection_error_std=2.0, triangulate=s != 4)
            tri_cases.append((P, kfs))

        def track(D):
            n_out = torch.zeros(2 * B, dtype=torch.int32, device="cuda")
            par = torch.zeros(2 * B, dtype=torch.float64, device="cuda")
            par_n = torch.zeros(2 * B, dtype=torch.int32, device="cuda")
            trk.track_frames_dev([params_struct(c[0], s % 2, 1 + s % 2) for s, c in enumerate(tcases)], D["map"][0], D["map"][2], D["ref"][0],
                                 D["ref"][2], n_out.data_ptr(), par.data_ptr(), par_n.data_ptr())
            return n_out
        # chained: the tracking step's compacted reference lists, counts read on the device from dev_n_out + 1 (stride 2)
        D = dev_lists(tcases)
        roff, rt, _ = D["ref"]
        n_out = track(D)
        N = int(roff[-1])
        src = torch.zeros(N, dtype=torch.int32, device="cuda")
        lt = dict(ref_out_xy=rt["ref_out_xy"], ref_frame_id_out=rt["ref_frame_id_out"], cur_xy=rt["cur_xy"], velocity_ref_out=rt["velocity_ref_out"],
                  velocity=rt["velocity"], src=src)
        nt = {k: torch.zeros((N, c), dtype=getattr(torch, np.dtype(dt).name), device="cuda") for k, (dt, c) in _TRI_NEW_SPEC.items()}
        counts = torch.zeros((B, 5), dtype=torch.int32, device="cuda")
        kf_off = np.concatenate([[0], np.cumsum([len(c[1]) for c in tri_cases])]).astype(np.int32)
        rows = [r for c in tri_cases for r in kf_rows(c[1])]
        trk.triangulate_dev([struct(c[0]) for c in tri_cases], kf_off, rows, roff, n_out.data_ptr() + 4, 2, {k: v.data_ptr() for k, v in lt.items()},
                            {k: v.data_ptr() for k, v in nt.items()}, counts.data_ptr())
        trk.sync()
        counts = counts.cpu().numpy()
        no = n_out.cpu().numpy()
        # reference: the same tracking step, host-compacted lists, the host triangulation call per stream
        D2 = dev_lists(tcases)
        n2 = track(D2)
        trk.sync()
        assert np.array_equal(n2.cpu().numpy(), no)
        rt2 = {k: v.cpu().numpy() for k, v in D2["ref"][1].items()}
        made = 0
        for s in range(B):
            a0, k = int(roff[s]), int(no[2 * s + 1])
            L = {key: rt2[key][a0:a0 + k] for key in ("ref_out_xy", "ref_frame_id_out", "cur_xy", "velocity_ref_out", "velocity")}
            L["ref_frame_id_out"] = L["ref_frame_id_out"].reshape(-1)
            h = trk.triangulate(struct(tri_cases[s][0]), kf_rows(tri_cases[s][1]), L)
            assert np.array_equal(counts[s], h[2]), (s, counts[s], h[2])
            if h[2][0] < 0:
                continue
            kk, mm = int(h[2][0]), int(h[2][1])
            for key, v in h[0].items():
                assert np.array_equal(lt[key].cpu().numpy()[a0:a0 + kk].reshape(np.asarray(v).shape), v), (s, key)
            for key in TRI_NEW:
                assert np.array_equal(nt[key].cpu().numpy()[a0:a0 + mm].reshape(np.asarray(h[1][key]).shape), h[1][key]), (s, key)
            made += mm
        assert (counts[:, 0] >= 0).sum() == B - 1 and counts[4][0] == -1
        print("chained counts (kept, succeeded, outlier, reset, outtime):", counts.tolist(), "new points:", made)
    finally:
        trk.close()


def test_argument_errors(klt):
    from ic_gvins_b200 import IcgError
    rng = np.random.default_rng(1)
    P, kfs, L = make_stream(rng, 10)
    rows = kf_rows(kfs)
    with pytest.raises(IcgError, match="monotone|start at 0"):
        klt.triangulate_dev([struct(P)], [0, len(rows)], rows, [1, 0], 0, 1, None, None, 1)
    with pytest.raises(IcgError, match="monotone|start at 0"):
        klt.triangulate_dev([struct(P)], [1, len(rows)], rows, [0, 0], 0, 1, None, None, 1)
    big = [(k, np.eye(3), np.zeros(3), True) for k in range(65)]
    with pytest.raises(IcgError, match="exceed 64"):
        klt.triangulate(struct(P), big, L)
    dup = rows + [rows[0]]
    with pytest.raises(IcgError, match="duplicate keyframe id"):
        klt.triangulate(struct(P), dup, L)
    with pytest.raises(IcgError, match="NULL list pointer"):
        klt.triangulate_dev([struct(P)], [0, len(rows)], rows, [0, 5], 0, 1, None, None, 1)
    with pytest.raises(IcgError, match="exceed max_points"):
        klt.triangulate(struct(P), rows, {k: np.zeros((5000,) + np.shape(v)[1:], np.asarray(v).dtype) for k, v in L.items()})


SHIM_SRC = r"""
#include <cstdio>
#include <cstring>
#include "ic_gvins_b200/host/icg_shims.hpp"
template <class T> std::vector<T> rd(FILE *f) { int64_t n; fread(&n, 8, 1, f); std::vector<T> v(n); fread(v.data(), sizeof(T), n, f); return v; }
template <class T> void wr(FILE *f, const std::vector<T> &v) { int64_t n = v.size(); fwrite(&n, 8, 1, f); fwrite(v.data(), sizeof(T), n, f); }
int main(int, char **argv) {
    FILE *f = fopen(argv[1], "rb");
    auto pb = rd<uint8_t>(f), kb = rd<uint8_t>(f);
    auto ref = rd<icg_b200::Point2f>(f), cur = rd<icg_b200::Point2f>(f);
    auto id = rd<int64_t>(f);
    auto vr = rd<double>(f), vc = rd<double>(f);
    fclose(f);
    icg_tri_frame p;
    memcpy(&p, pb.data(), sizeof(p));
    std::vector<icg_tri_keyframe> kf(kb.size() / sizeof(icg_tri_keyframe));
    memcpy(kf.data(), kb.data(), kb.size());
    icg_b200::KltContext k(640, 480, 4096);
    std::vector<icg_b200::Point2f> pnew;
    std::vector<int32_t> src;
    std::vector<icg_b200::KltContext::NewMapPoint> pts;
    int32_t c[5];
    bool ok = k.triangulation(p, kf, ref, id, cur, vr, vc, pnew, src, pts, c);
    std::vector<double> pw, depth;
    std::vector<int32_t> nsrc;
    for (auto &q : pts) pw.insert(pw.end(), q.pw, q.pw + 3), depth.push_back(q.depth), nsrc.push_back(q.src);
    FILE *o = fopen(argv[2], "wb");
    wr(o, ref), wr(o, id), wr(o, cur), wr(o, vr), wr(o, src), wr(o, pnew), wr(o, pw), wr(o, depth), wr(o, nsrc);
    wr(o, std::vector<int32_t>{c[0], c[1], c[2], c[3], c[4], (int32_t) ok});
    fclose(o);
    return 0;
}
"""


def test_cpp_shim_triangulation(klt):
    import shutil
    import subprocess
    import tempfile
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    from ic_gvins_b200.klt import tri_keyframes
    lib = os.path.join(ROOT, "ic_gvins_b200", "libicgvins_b200.so")
    P, kfs, L = make_stream(np.random.default_rng(41), 280, window_normal=True)
    ps = struct(P)
    rows = kf_rows(kfs)
    h = klt.triangulate(ps, rows, L)

    def wr(fh, a, n=None):
        a = np.ascontiguousarray(a)
        fh.write(np.int64(a.size if n is None else n).tobytes())
        fh.write(a.tobytes())
    with tempfile.TemporaryDirectory() as td:
        cpp, exe, fin, fout = (os.path.join(td, x) for x in ("s.cpp", "s", "in.bin", "out.bin"))
        open(cpp, "w").write(SHIM_SRC)
        r = subprocess.run(["g++", "-std=c++17", "-O1", "-I", ROOT, cpp, "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        with open(fin, "wb") as fh:
            wr(fh, np.frombuffer(bytes(ps), np.uint8))
            wr(fh, np.frombuffer(bytes(tri_keyframes(rows)), np.uint8))
            n = len(L["cur_xy"])
            wr(fh, L["ref_out_xy"], n), wr(fh, L["cur_xy"], n), wr(fh, L["ref_frame_id_out"])
            wr(fh, L["velocity_ref_out"].reshape(-1)), wr(fh, L["velocity"].reshape(-1))
        r = subprocess.run([exe, fin, fout], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, (r.returncode, r.stderr)
        out = []
        with open(fout, "rb") as fh:
            for dt, w in ((np.float32, 2), (np.int64, 1), (np.float32, 2), (np.float64, 1), (np.int32, 1), (np.float32, 2), (np.float64, 1),
                          (np.float64, 1), (np.int32, 1), (np.int32, 1)):
                n = int(np.frombuffer(fh.read(8), np.int64)[0])
                out.append(np.frombuffer(fh.read(n * w * np.dtype(dt).itemsize), dt))
    lo, no, cnt = h
    assert np.array_equal(out[9][:5], cnt) and out[9][5] == 1
    assert np.array_equal(out[0].reshape(-1, 2), lo["ref_out_xy"]) and np.array_equal(out[1], lo["ref_frame_id_out"])
    assert np.array_equal(out[2].reshape(-1, 2), lo["cur_xy"]) and np.array_equal(out[3].reshape(-1, 2), lo["velocity_ref_out"])
    assert np.array_equal(out[4], lo["src"]) and np.array_equal(out[5].reshape(-1, 2), lo["cur_xy"])
    assert np.array_equal(out[6].reshape(-1, 3), no["pw"]) and np.array_equal(out[7], no["depth"]) and np.array_equal(out[8], no["src"])
    assert cnt[1] > 0
