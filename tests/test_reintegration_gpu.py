"""GPU: GVINS::doReintegration on the resident IMU factors (icg_ba_reintegrate_resident) -- the gate against a numpy restatement, the values
against the plain batch (bitwise) and the oracle, the handle's state after the call against a fresh upload of the reintegrated factors,
the call chained after the real two-pass solve at cfg 3 and cfg 4, the error paths, and the C++ shim."""
import copy
import ctypes as C
import math
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from datagen import synth_ba
from tests import oracle_api as oa

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOISE5 = synth_ba.NOISE5
SG, SA = 6 * NOISE5[2], 6 * NOISE5[3]  # the gate's thresholds, as the device forms them
STATION = np.array([30.5 * math.pi / 180.0, 114.3 * math.pi / 180.0, 21.7])


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def geom():
    from ic_gvins_b200.geom import Geometry
    g = Geometry()
    yield g
    g.close()


# ---------------------------------------------------------------------------------------------- numpy restatements
def earth_iewn(origin, local):
    """Earth::iewn(origin, local) (earth.h): blh2ecef(origin) + cne(origin) local -> ecef2blh's latitude loop -> (wie cos, 0, -wie sin)"""
    WIE, RA, E1 = 7.2921151467e-5, 6378137.0, 0.0066943799901413156
    lat0, lon0, h0 = origin
    sl, cl, so, co = math.sin(lat0), math.cos(lat0), math.sin(lon0), math.cos(lon0)
    rn = RA / math.sqrt(1.0 - E1 * sl * sl)
    e0 = np.array([(rn + h0) * cl * co, (rn + h0) * cl * so, (rn + h0 - rn * E1) * sl])
    cne = np.array([[-sl * co, -so, -cl * co], [-sl * so, co, -cl * so], [cl, 0.0, -sl]])
    x, y, z = e0 + cne @ np.asarray(local, np.float64)
    p = math.sqrt(x * x + y * y)
    lat, h = math.atan(z / (p * (1.0 - E1))), 0.0
    while True:
        h2 = h
        s = math.sin(lat)
        r = RA / math.sqrt(1.0 - E1 * s * s)
        h = p / math.cos(lat) - r
        lat = math.atan(z / (p * (1.0 - E1 * r / (r + h))))
        if not abs(h - h2) > 1e-4:
            break
    return np.array([WIE * math.cos(lat), 0.0, -WIE * math.sin(lat)])


def gate(blob, mix, noise5=NOISE5):
    """doReintegration's test: sqrt of the fixed-order sum of squares, strict comparison"""
    g, a = blob[11:14] - mix[3:6], blob[14:17] - mix[6:9]
    ng = math.sqrt((g[0] * g[0] + g[1] * g[1]) + g[2] * g[2])
    na = math.sqrt((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2])
    return ng > 6 * noise5[2] or na > 6 * noise5[3]


def state16(pose, mix):
    x, y, z, w = pose[3:7]
    n = math.sqrt(((x * x + y * y) + z * z) + w * w)
    return np.concatenate([pose[:3], [x / n, y / n, z / n, w / n], mix])


# ---------------------------------------------------------------------------------------------- windows
def window(olib, seed, K=10, L=60, earth=True, lin=None):
    """a synthetic window whose factors are re-linearised here on fresh IMU rows (kept for the call): factor k at node k's mix biases plus
    lin(k) = (dbg, dba) (None: the window's own linearisation point)"""
    prob = synth_ba.make_window(lambda *a: oa.preintegrate(olib, *a), K=K, L=L, seed=seed, earth=earth)[0]
    rng = np.random.default_rng(seed + 77)
    pose, mix = prob["pose"].reshape(K, 7), prob["mix"].reshape(K, 9)
    blobs, rows = prob["imu_blob"].reshape(K - 1, 480), []
    for k in range(K - 1):
        t0 = 0.5 * k
        imu = synth_ba.imu_samples(t0, t0 + 0.5, 200.0, rng, mix[k, 3:6], mix[k, 6:9], earth=earth)
        st = np.concatenate([pose[k], mix[k]])
        if lin is not None:
            dbg, dba = lin(k)
            st[10:13] += dbg
            st[13:16] += dba
        blobs[k] = oa.preintegrate(olib, st, synth_ba.IEWN if earth else None, synth_ba.GRAVITY, NOISE5, imu)[0]
        rows.append(imu)
    return prob, rows


def gate_cases(k):
    """per factor: neither, gyro only, accel only, both, then three random offsets around the thresholds"""
    z = np.zeros(3)
    return [(z, z), (np.array([7 * NOISE5[2], 0, 0]), z), (z, np.array([0, 7 * NOISE5[3], 0])), (np.full(3, 5 * NOISE5[2]), np.full(3, 5 * NOISE5[3])),
            (z, z), (z, z), (np.array([0, 3 * NOISE5[2], 0]), z), (z, np.array([2 * NOISE5[3], 2 * NOISE5[3], 2 * NOISE5[3]])),
            (np.array([6.5 * NOISE5[2], 0, 0]), np.array([0, 0, 5.9 * NOISE5[3]]))][k % 9]


def knife_edges(prob):
    """factor 4: mix.bg = blob.bg - (6 sigma, 0, 0) exactly (sqrt(x^2) == |x|: closed); factor 5: the next double up (open)"""
    mix, blobs = prob["mix"].reshape(prob["K"], 9), prob["imu_blob"].reshape(-1, 480)
    for k, x in ((4, -SG), (5, np.nextafter(-SG, -np.inf))):
        blobs[k, 11] = 0.0  # the factor's linearisation bg.x (the blob is otherwise unchanged: only the gate reads it before the replay)
        mix[k, 3] = x
        mix[k, 6:9] = blobs[k, 14:17]
        mix[k, 4:6] = blobs[k, 12:14]
        assert (blobs[k, 11] - mix[k, 3] == SG) == (k == 4)


def solver_for(probs, max_K=None):
    from ic_gvins_b200.ba import WindowSolver
    return WindowSolver(max_windows=len(probs), max_K=max_K or max(p["K"] for p in probs), max_L=max(1, max(p["L"] for p in probs)),
                        max_F=max(1, max(p["F"] for p in probs)), max_gnss=16, max_marg_r=160)


def gate_set(olib):
    w0, r0 = window(olib, 301, lin=gate_cases)
    knife_edges(w0)
    w1, r1 = window(olib, 302, earth=False, lin=lambda k: gate_cases(k + 3))
    w2, r2 = window(olib, 303, lin=lambda k: (np.full(3, 9 * NOISE5[2]), np.zeros(3)))  # every gate open, but reintegrate = 0
    w3, _ = window(olib, 304, K=6)
    w3["n_imu"] = 0
    return [w0, w1, w2, w3], [r0, r1, r2, None], [1, 1, 0, 1]


def expected_status(prob):
    K = prob["K"]
    mix, blobs = prob["mix"].reshape(K, 9), prob["imu_blob"].reshape(-1, 480)
    return np.array([1 if gate(blobs[k], mix[k]) else 0 for k in range(prob["n_imu"])], np.int8)


def host_iewn(prob, k, station):
    if prob["imu_blob"].reshape(-1, 480)[k, 477] != 0:
        return None
    return earth_iewn(station, prob["pose"].reshape(prob["K"], 7)[k, :3])


# ---------------------------------------------------------------------------------------------- 1 + 2 + 3: gate, values, resident state
@pytest.mark.parametrize("station", [np.zeros(3), STATION], ids=["station0", "station"])
def test_gate_values_and_resident_state(olib, geom, station):
    from ic_gvins_b200.ba import WindowSolver
    probs, rows, flags = gate_set(olib)
    before = copy.deepcopy(probs)
    want = [expected_status(p) if f and p["n_imu"] else np.zeros(p["n_imu"], np.int8) for p, f in zip(probs, flags)]
    assert want[0][4] == 0 and want[0][5] == 1 and want[0][0] == 0 and want[0][1:4].all()
    s = solver_for(probs)
    t = u = None
    try:
        s.upload(probs)
        out = s.reintegrate(probs, NOISE5, station, rows, reintegrate=flags)
        for w in range(4):
            assert np.array_equal(out[w]["status"], want[w]), w
            assert out[w]["count"] == int((want[w] != 0).sum())
        assert out[2]["count"] == 0 and np.array_equal(probs[2]["imu_blob"], before[2]["imu_blob"]) and not out[2]["end_states"].any()
        assert out[3]["count"] == 0 and out[3]["status"].size == 0
        # 2. values: the plain batch on the same state (uploaded pose with q normalised, mix) and the iewn the call wrote -> bitwise
        for w in (0, 1):
            p, o = before[w], out[w]
            pose, mix = p["pose"].reshape(p["K"], 7), p["mix"].reshape(p["K"], 9)
            for k in np.nonzero(o["status"] == 1)[0]:
                got = o["blobs"][k]
                assert np.array_equal(probs[w]["imu_blob"].reshape(-1, 480)[k], got)
                st = state16(pose[k], mix[k])
                iw = host_iewn(p, k, station)
                if iw is None:
                    assert not got[20:23].any() and got[477] == 1.0
                else:
                    assert np.abs(got[20:23] - iw).max() <= 1e-15 * np.abs(iw).max(), (w, k)
                b, e = geom.imu_preintegrate_batch(st[None], got[20:23] if iw is not None else None, synth_ba.GRAVITY, NOISE5, [rows[w][k]])
                assert np.array_equal(b[0], got), (w, k)
                assert np.array_equal(e[0], o["end_states"][k]), (w, k)
                bo, _, eo = oa.preintegrate(olib, st, iw, synth_ba.GRAVITY, NOISE5, rows[w][k])
                assert np.abs(got[:27] - bo[:27]).max() <= 1e-12 * max(1.0, np.abs(bo[:27]).max())
                assert np.abs(got[27:252] - bo[27:252]).max() <= 1e-12 * np.abs(bo[27:252]).max()
                assert np.abs(got[252:477] - bo[252:477]).max() <= 1e-10 * np.abs(bo[252:477]).max()
                assert np.abs(o["end_states"][k] - eo).max() <= 1e-13 * np.abs(eo).max()
            for k in np.nonzero(o["status"] == 0)[0]:  # closed: the factor is untouched
                assert np.array_equal(probs[w]["imu_blob"].reshape(-1, 480)[k], p["imu_blob"].reshape(-1, 480)[k])
        # 3. the handle now holds the reintegrated factors.  The same problems with the returned blobs, uploaded afresh: the restart solve
        #    gives the same summaries and parameters, and after the two-pass solve the resident marginalization equals the uploading call on
        #    the written-back arrays (device U == host U).  Every marginalization follows a solve on its handle, as the resident one requires.
        fresh, fresh2 = copy.deepcopy(probs), copy.deepcopy(probs)
        t = WindowSolver(max_windows=len(probs), max_K=10, max_L=max(p["L"] for p in probs), max_F=max(p["F"] for p in probs), max_gnss=16,
                         max_marg_r=160)
        u = WindowSolver(max_windows=len(probs), max_K=10, max_L=max(p["L"] for p in probs), max_F=max(p["F"] for p in probs), max_gnss=16,
                         max_marg_r=160)
        s.run_gvins(20, restart=True)
        t.upload(fresh)
        t.run_gvins(20, restart=True)
        sa, sb = s.download(), t.download()
        assert sa == sb
        for a, b in zip(probs, fresh):
            for key in ("pose", "mix", "ext", "invdepth"):
                assert np.array_equal(a[key], b[key]), key
        u.gvins_optimization_batch(fresh2, 20)
        for a, b in zip(probs, fresh2):
            for key in ("pose", "mix", "ext", "invdepth"):
                assert np.array_equal(a[key], b[key]), key
        m_res = s.marginalize(probs, 1, resident=True)
        m_up = u.marginalize(fresh2, 1)
        for a, b in zip(m_res, m_up):
            for key in ("J0", "e0", "Hp", "bp", "x0"):
                assert np.array_equal(a[key], b[key]), key
    finally:
        for h in (s, t, u):
            if h is not None:
                h.close()


# ---------------------------------------------------------------------------------------------- 4: after the real protocol
def chained(olib, K, L, nwin, max_K, seeds):
    from ic_gvins_b200.ba import imu_preintegrate
    off = lambda k: (np.array([(-1) ** k * 8 * NOISE5[2], 0, 0]), np.zeros(3)) if k % 3 != 1 else (np.zeros(3), np.zeros(3))
    made = [window(olib, sd, K=K, L=L, earth=(w % 2 == 0), lin=off) for w, sd in enumerate(seeds[:nwin])]
    probs, rows = [m[0] for m in made], [m[1] for m in made]
    s = solver_for(probs, max_K=max_K)
    try:
        s.gvins_optimization_batch(probs, 20)
        host = copy.deepcopy(probs)  # downloaded parameters, the blobs the solve used
        out = s.reintegrate(probs, NOISE5, np.zeros(3), rows)
    finally:
        s.close()
    opened = 0
    for w, (p, o) in enumerate(zip(host, out)):
        pose, mix, blobs = p["pose"].reshape(K, 7), p["mix"].reshape(K, 9), p["imu_blob"].reshape(-1, 480)
        want = np.array([1 if gate(blobs[k], mix[k]) else 0 for k in range(K - 1)], np.int8)
        assert np.array_equal(o["status"], want), w
        assert o["count"] == int(want.sum())
        opened += int(want.sum())
        for k in np.nonzero(want)[0]:
            st = state16(pose[k], mix[k])
            iw = None if blobs[k, 477] else earth_iewn(np.zeros(3), pose[k, :3])
            bh, eh = imu_preintegrate(st, iw, synth_ba.GRAVITY, NOISE5, rows[w][k])
            got = o["blobs"][k]
            assert got[477] == bh[477]
            assert np.abs(got[:27] - bh[:27]).max() <= 1e-12 * max(1.0, np.abs(bh[:27]).max())
            assert np.abs(got[27:252] - bh[27:252]).max() <= 1e-12 * np.abs(bh[27:252]).max()
            assert np.abs(got[252:477] - bh[252:477]).max() <= 1e-10 * np.abs(bh[252:477]).max()
            assert np.abs(o["end_states"][k] - eh).max() <= 1e-13 * np.abs(eh).max()
    assert 0 < opened < nwin * (K - 1)


def test_chained_after_gvins_optimization_cfg3(olib):
    chained(olib, 10, 300, 4, 10, [410, 411, 412, 413])


def test_chained_after_gvins_optimization_cfg4_split_pipeline(olib):
    chained(olib, 20, 600, 2, 20, [420, 421])


# ---------------------------------------------------------------------------------------------- 5: errors
def test_zero_noise_rejects_every_factor_and_keeps_the_handle(olib):
    from ic_gvins_b200._lib import IcgError
    probs, rows = zip(*[window(olib, 500 + w, lin=lambda k: (np.full(3, 1e-9), np.zeros(3))) for w in range(2)])
    probs = list(probs)
    s = solver_for(probs)
    try:
        s.upload(probs)
        s.run_gvins(20, restart=True)
        sum_ref = s.download()
        ref = copy.deepcopy(probs)
        before = copy.deepcopy(probs)
        with pytest.raises(IcgError) as ei:
            s.reintegrate(probs, np.zeros(5), np.zeros(3), list(rows))
        assert ei.value.code == -1 and "window 0 IMU factor 0" in str(ei.value)
        for o in ei.value.results:
            assert (o["status"] == -1).all() and o["count"] == len(o["status"])
        for a, b in zip(probs, before):
            assert np.array_equal(a["imu_blob"], b["imu_blob"])
        s.run_gvins(20, restart=True)
        assert s.download() == sum_ref
        for a, b in zip(probs, ref):
            for key in ("pose", "mix", "ext", "invdepth"):
                assert np.array_equal(a[key], b[key]), key
    finally:
        s.close()


def test_bad_imu_off_is_refused_before_any_launch(olib):
    from ic_gvins_b200._lib import BaProblem, ReintWindow, lib
    from ic_gvins_b200.ba import to_struct
    prob, rows = window(olib, 510)
    s = solver_for([prob])
    try:
        s.upload([prob])
        imu = np.ascontiguousarray(np.concatenate(rows))
        status = np.full(prob["n_imu"], 7, np.int8)
        blobs = np.zeros((prob["n_imu"], 480))
        arr = (BaProblem * 1)(to_struct(prob))
        nz, stn = np.ascontiguousarray(NOISE5), np.zeros(3)
        for off in ([0] + [101 * (k + 1) for k in range(prob["n_imu"] - 1)] + [101 * (prob["n_imu"] - 1)],  # an empty last interval
                    [0, 101, 90] + [101 * (k + 1) for k in range(2, prob["n_imu"])],                        # decreasing
                    [-5] + [101 * (k + 1) for k in range(prob["n_imu"])]):                                    # negative start
            o = np.ascontiguousarray(off, np.int32)
            assert o.size == prob["n_imu"] + 1
            io = (ReintWindow * 1)()
            io[0].reintegrate, io[0].imu, io[0].imu_off = 1, imu.ctypes.data_as(C.POINTER(C.c_double)), o.ctypes.data_as(C.POINTER(C.c_int32))
            io[0].status, io[0].blob_out = status.ctypes.data_as(C.POINTER(C.c_int8)), blobs.ctypes.data_as(C.POINTER(C.c_double))
            n0 = lib().icg_launch_count()
            rc = lib().icg_ba_reintegrate_resident(s._h, 1, arr, C.c_void_p(nz.ctypes.data), C.c_void_p(stn.ctypes.data), io)
            assert rc == -1 and "imu_off" in lib().icg_last_error().decode()
            assert lib().icg_launch_count() == n0 and (status == 7).all()
    finally:
        s.close()


def test_landmark_sharded_handle_is_refused(olib):
    from ic_gvins_b200._lib import IcgError
    from ic_gvins_b200.ba import WindowSolver
    prob, rows = window(olib, 520)
    solvers = [WindowSolver(max_windows=1, max_K=10, max_L=prob["L"], max_F=prob["F"], max_gnss=16, max_marg_r=64) for _ in range(2)]
    try:
        blobs = [solvers[r].shard_export(r, 2) for r in range(2)]
        for sv in solvers:
            sv.shard_connect(blobs)
        with pytest.raises(IcgError, match="landmark-sharded") as ei:
            solvers[0].reintegrate([prob], NOISE5, np.zeros(3), [rows])
        assert ei.value.code == -4
    finally:
        for sv in solvers:
            sv.close()


# ---------------------------------------------------------------------------------------------- 6: the C++ shim
SRC = r'''
#include <cstdio>
#include <vector>
#include "ic_gvins_b200/host/icg_shims.hpp"

static std::vector<double> rd(FILE *f) {
    long long n = 0;
    if (fread(&n, 8, 1, f) != 1) throw std::runtime_error("short input");
    std::vector<double> v((size_t) n);
    if (n && fread(v.data(), 8, (size_t) n, f) != (size_t) n) throw std::runtime_error("short input");
    return v;
}
template <typename T> static std::vector<T> as(const std::vector<double> &v) { return std::vector<T>(v.begin(), v.end()); }
static void wr(FILE *f, const std::vector<double> &v) {
    long long n = (long long) v.size();
    fwrite(&n, 8, 1, f);
    if (n) fwrite(v.data(), 8, (size_t) n, f);
}

int main(int argc, char **argv) {
    try {
        FILE *in = fopen(argv[1], "rb");
        auto dims = as<int>(rd(in));  // K L F
        const int K = dims[0], L = dims[1], F = dims[2];
        auto pose = rd(in), mix = rd(in), ext = rd(in), rho = rd(in), fc = rd(in), blob = rd(in), scal = rd(in);
        auto f_lm = as<int32_t>(rd(in)), f_ref = as<int32_t>(rd(in)), f_obs = as<int32_t>(rd(in));
        auto gnode = as<int32_t>(rd(in));
        auto gblh = rd(in), gstd = rd(in), lever = rd(in), noise5 = rd(in), imu = rd(in);
        auto off = as<int32_t>(rd(in));
        fclose(in);
        std::vector<uint8_t> act(F, 1);
        icg_ba_problem p{};
        p.K = K, p.L = L, p.F = F, p.pose = pose.data(), p.mix = mix.data(), p.ext = ext.data(), p.invdepth = rho.data();
        p.f_lm = f_lm.data(), p.f_ref = f_ref.data(), p.f_obs = f_obs.data(), p.f_const = fc.data(), p.f_active = act.data();
        p.reproj_std = scal[0], p.reproj_huber = 1, p.n_imu = K - 1, p.imu_blob = blob.data(), p.has_imu_error = 1;
        p.n_gnss = (int) gnode.size(), p.gnss_node = gnode.data(), p.gnss_blh = gblh.data(), p.gnss_std = gstd.data(), p.gnss_huber = 1;
        for (int i = 0; i < 3; i++) p.lever[i] = lever[i];
        icg_b200::WindowSolver solver(K, L, F, 16, 160);
        icg_ba_summary s[2];
        int32_t culled[2];
        solver.gvinsOptimization(p, 20, s, culled);
        const double station[3] = {0, 0, 0};
        std::vector<int8_t> status;
        std::vector<double> ends;
        const int cnt = solver.doReintegration(p, noise5.data(), station, imu, off, status, blob, &ends);
        FILE *out = fopen(argv[2], "wb");
        wr(out, {(double) cnt}), wr(out, std::vector<double>(status.begin(), status.end())), wr(out, blob), wr(out, ends), wr(out, pose);
        fclose(out);
        return 0;
    } catch (const std::exception &e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
}
'''


def _wr(f, arr):
    a = np.ascontiguousarray(arr, np.float64).ravel()
    f.write(np.int64(a.size).tobytes())
    f.write(a.tobytes())


def _rd(f):
    n = int(np.frombuffer(f.read(8), np.int64)[0])
    return np.frombuffer(f.read(8 * n), np.float64).copy()


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_cpp_reintegration_shim_runs_on_the_gpu(olib):
    from ic_gvins_b200.ba import WindowSolver
    lib = os.path.join(ROOT, "ic_gvins_b200", "libicgvins_b200.so")
    prob, rows = window(olib, 530, K=8, L=80, lin=lambda k: (np.array([0, 0, (k % 2) * 9 * NOISE5[2]]), np.zeros(3)))
    py = copy.deepcopy(prob)
    s = WindowSolver(max_windows=1, max_K=prob["K"], max_L=prob["L"], max_F=prob["F"], max_gnss=16, max_marg_r=160)
    try:
        s.gvins_optimization_batch([py], 20)
        o = s.reintegrate([py], NOISE5, np.zeros(3), [rows])[0]
    finally:
        s.close()
    assert o["count"] > 0
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])])
    with tempfile.TemporaryDirectory() as td:
        cpp, exe, fin, fout = (os.path.join(td, x) for x in ("shim.cpp", "shim", "in.bin", "out.bin"))
        open(cpp, "w").write(SRC)
        r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", ROOT, cpp, "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        with open(fin, "wb") as fh:
            for arr in ([prob["K"], prob["L"], prob["F"]], prob["pose"], prob["mix"], prob["ext"], prob["invdepth"], prob["f_const"], prob["imu_blob"],
                        [prob["reproj_std"]], prob["f_lm"], prob["f_ref"], prob["f_obs"], prob["gnss_node"], prob["gnss_blh"], prob["gnss_std"],
                        prob["lever"], NOISE5, np.concatenate(rows), off):
                _wr(fh, arr)
        r = subprocess.run([exe, fin, fout], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, (r.returncode, r.stderr)
        with open(fout, "rb") as fh:
            cnt, status, blob, ends, pose = (_rd(fh) for _ in range(5))
    assert int(cnt[0]) == o["count"] and np.array_equal(status.astype(np.int8), o["status"])
    assert np.array_equal(pose, py["pose"])
    assert np.array_equal(blob, py["imu_blob"])
    assert np.array_equal(ends.reshape(-1, 10), o["end_states"])
