"""The header-only C++ shims EXECUTED on the GPU: a C++ program that includes ic_gvins_b200/host/icg_shims.hpp (OpenCV call signatures) and
icg_factors.hpp (the reference's cost-function classes with the Ceres `Evaluate(double const* const*, double*, double**)` signature) is compiled
with g++, linked against libicgvins_b200.so and run; its outputs are compared with the cv2 golden vectors (KLT) and with the oracle (factors).
This is the C++ side of the drop-in boundary (the Python ctypes mirror is what the other GPU tests drive)."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from datagen import synth_ba
from tests import oracle_api as oa
from tests.test_oracle_klt import assert_px

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r'''
#include <cstdio>
#include <vector>
#include "ic_gvins_b200/host/icg_shims.hpp"
#include "ic_gvins_b200/host/icg_factors.hpp"

static std::vector<double> rd(FILE *f) {
    long long n = 0;
    if (fread(&n, 8, 1, f) != 1) throw std::runtime_error("short input");
    std::vector<double> v((size_t) n);
    if (n && fread(v.data(), 8, (size_t) n, f) != (size_t) n) throw std::runtime_error("short input");
    return v;
}
static void wr(FILE *f, const std::vector<double> &v) {
    long long n = (long long) v.size();
    fwrite(&n, 8, 1, f);
    if (n) fwrite(v.data(), 8, (size_t) n, f);
}

int main(int argc, char **argv) {
    try {
        FILE *in = fopen(argv[1], "rb"), *out = fopen(argv[2], "wb");
        if (!in || !out) return 2;
        // ---------------- Tracking::trackMappoint block through the OpenCV-signature shims (IG/tracking/tracking.cc:385-403)
        std::vector<double> dim = rd(in), img0 = rd(in), img1 = rd(in), p0 = rd(in), init = rd(in);
        const int W = (int) dim[0], H = (int) dim[1], n = (int) p0.size() / 2;
        std::vector<uint8_t> a(img0.begin(), img0.end()), b(img1.begin(), img1.end());
        icg_b200::Mat A{a.data(), H, W, W}, B{b.data(), H, W, W};
        std::vector<icg_b200::Point2f> prev(n), next(n), next2(n);
        for (int k = 0; k < n; k++) prev[k] = {(float) p0[2 * k], (float) p0[2 * k + 1]}, next[k] = next2[k] = {(float) init[2 * k], (float) init[2 * k + 1]};
        std::vector<uint8_t> st, st_fb;
        std::vector<float> err;
        icg_b200::KltContext klt(W, H);
        klt.calcOpticalFlowPyrLK(A, B, prev, next, st, err, icg_b200::Size(21, 21), 3, icg_b200::TermCriteria(3, 30, 0.01), ICG_OPTFLOW_USE_INITIAL_FLOW);
        klt.trackForwardBackward(A, B, prev, next2, st_fb);
        // COUNT-only criteria: OpenCV takes its default epsilon 0.01, so this is the call above
        std::vector<icg_b200::Point2f> next3(n);
        for (int k = 0; k < n; k++) next3[k] = {(float) init[2 * k], (float) init[2 * k + 1]};
        std::vector<uint8_t> st3;
        std::vector<float> err3;
        klt.calcOpticalFlowPyrLK(A, B, prev, next3, st3, err3, icg_b200::Size(21, 21), 3, icg_b200::TermCriteria(1, 30, 0.5), ICG_OPTFLOW_USE_INITIAL_FLOW);
        std::vector<double> o1, o2, o3;
        for (int k = 0; k < n; k++) o1.insert(o1.end(), {next[k].x, next[k].y, (double) st[k]}), o2.insert(o2.end(), {next2[k].x, next2[k].y, (double) st_fb[k]});
        for (int k = 0; k < n; k++) o3.insert(o3.end(), {next3[k].x, next3[k].y, (double) st3[k]});
        wr(out, o1), wr(out, o2), wr(out, o3);
        // ---------------- cv::CLAHE::apply
        icg_b200::Clahe clahe(W, H);
        std::vector<uint8_t> eq(a.size());
        clahe.apply(a.data(), W, eq.data(), W);
        wr(out, std::vector<double>(eq.begin(), eq.end()));
        // ---------------- cost functions, Ceres signature
        std::vector<double> rp = rd(in);  // pose0 7, pose1 7, ext 7, rho 1, td 1, c14, std
        {
            icg_b200::ReprojectionFactor f(&rp[23], &rp[26], &rp[29], &rp[32], rp[35], rp[36], rp[37]);
            const double *params[5] = {&rp[0], &rp[7], &rp[14], &rp[21], &rp[22]};
            std::vector<double> r(2), J0(14), J1(14), J2(14), J3(2), J4(2);
            double *J[5] = {J0.data(), J1.data(), J2.data(), J3.data(), J4.data()};
            if (!f.Evaluate(params, r.data(), J)) return 3;
            wr(out, r), wr(out, J0), wr(out, J1), wr(out, J2), wr(out, J3), wr(out, J4);
            std::vector<double> r2(2);
            if (!f.Evaluate(params, r2.data(), nullptr)) return 3;   // residual-only call (jacobians == NULL), as Ceres makes it
            wr(out, r2);
        }
        std::vector<double> ip = rd(in);  // blob 480, pose0 7, mix0 9, pose1 7, mix1 9
        {
            icg_b200::PreintegrationFactor f(ip.data());
            const double *params[4] = {&ip[480], &ip[487], &ip[496], &ip[503]};
            std::vector<double> r(15), J0(105), J1(135), J2(105), J3(135);
            double *J[4] = {J0.data(), nullptr, J2.data(), J3.data()};   // a NULL block: Ceres skips constant blocks
            if (!f.Evaluate(params, r.data(), J)) return 3;
            wr(out, r), wr(out, J0), wr(out, J2), wr(out, J3);
        }
        std::vector<double> gp = rd(in);  // pose 7, blh 3, std 3, lever 3
        {
            icg_b200::GnssFactor f(&gp[7], &gp[10], &gp[13]);
            const double *params[1] = {&gp[0]};
            std::vector<double> r(3), J0(21);
            double *J[1] = {J0.data()};
            if (!f.Evaluate(params, r.data(), J)) return 3;
            wr(out, r), wr(out, J0);
        }
        fclose(in), fclose(out);
        return 0;
    } catch (const std::exception &e) {
        fprintf(stderr, "shim test: %s\n", e.what());
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
def test_cpp_shims_run_on_the_gpu(oracle, klt_golden):
    oa.declare_ba(oracle)
    lib = os.path.join(ROOT, "ic_gvins_b200", "libicgvins_b200.so")
    g = klt_golden
    name = "small_plain"
    f0, f1, p0, init = g[name + "_f0"], g[name + "_f1"], g[name + "_p0"], g[name + "_init"]
    H, W = f0.shape
    prob, _ = synth_ba.make_window(lambda *a: oa.preintegrate(oracle, *a), K=6, L=40, seed=5)
    pose, mix = prob["pose"].reshape(-1, 7), prob["mix"].reshape(-1, 9)
    f = 7
    i, j, l = int(prob["f_ref"][f]), int(prob["f_obs"][f]), int(prob["f_lm"][f])
    c14 = prob["f_const"][14 * f:14 * f + 14]
    rp = np.concatenate([pose[i], pose[j], prob["ext"][:7], [prob["invdepth"][l]], [prob["ext"][7]], c14, [prob["reproj_std"]]])
    k = 2
    blob = prob["imu_blob"][480 * k:480 * (k + 1)]
    ip = np.concatenate([blob, pose[k], mix[k], pose[k + 1], mix[k + 1]])
    gidx = 1
    nd = int(prob["gnss_node"][gidx])
    gp = np.concatenate([pose[nd], prob["gnss_blh"][3 * gidx:3 * gidx + 3], prob["gnss_std"][3 * gidx:3 * gidx + 3], prob["lever"]])
    with tempfile.TemporaryDirectory() as td:
        cpp, exe, fin, fout = (os.path.join(td, x) for x in ("shim.cpp", "shim", "in.bin", "out.bin"))
        open(cpp, "w").write(SRC)
        r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", ROOT, cpp, "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        with open(fin, "wb") as fh:
            for arr in ([W, H], f0, f1, p0, init, rp, ip, gp):
                _wr(fh, arr)
        r = subprocess.run([exe, fin, fout], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, (r.returncode, r.stderr)
        with open(fout, "rb") as fh:
            lk, fb, lk_count, eq = _rd(fh).reshape(-1, 3), _rd(fh).reshape(-1, 3), _rd(fh).reshape(-1, 3), _rd(fh)
            r_rep, Ji, Jj, Je, Jr, Jt, r_rep2 = (_rd(fh) for _ in range(7))
            r_imu, I0, I2, I3 = (_rd(fh) for _ in range(4))
            r_gn, Jg = _rd(fh), _rd(fh)
    # KLT vs the cv2 golden vectors
    assert np.array_equal(lk[:, 2].astype(np.uint8), g[name + "_st"])
    assert_px(lk[:, :2].astype(np.float32), g[name + "_fwd"], g[name + "_st"] == 1, name)
    assert np.array_equal(lk_count, lk)
    assert np.array_equal(fb[:, 2].astype(np.uint8), g[name + "_good"])
    assert_px(fb[:, :2].astype(np.float32), g[name + "_fwd"], g[name + "_good"] == 1, name)
    # CLAHE vs the oracle (bit-exact with cv2)
    assert np.array_equal(eq.astype(np.uint8).reshape(H, W), oa.clahe_apply(oracle, f0, 3.0, 21, 21))
    # factors vs the oracle
    ro, Jo = oa.reproj_eval(oracle, pose[i], pose[j], prob["ext"][:7], prob["invdepth"][l], prob["ext"][7], c14, prob["reproj_std"])
    assert np.abs(r_rep - ro).max() <= 1e-12 * max(1.0, np.abs(ro).max()) and np.array_equal(r_rep, r_rep2)
    for a, b in zip((Ji, Jj, Je, Jr, Jt), Jo):
        assert np.abs(a - b.ravel()).max() <= 1e-11 * max(1.0, np.abs(b).max())
    off, pn = prob["pn_off"], prob["pn"].reshape(-1, 4)
    ro, Jo = oa.imu_eval(oracle, blob, pn[off[k]:off[k + 1]], pose[k], mix[k], pose[k + 1], mix[k + 1])
    assert np.abs(r_imu - ro).max() <= 1e-7 * max(1.0, np.abs(ro).max())
    for a, b in zip((I0, I2, I3), (Jo[0], Jo[2], Jo[3])):
        assert np.abs(a - b.ravel()).max() <= 1e-7 * max(1.0, np.abs(b).max())
    ro, Jg_o = np.zeros(3), np.zeros((3, 7))
    a = [pose[nd].copy(), prob["gnss_blh"][3 * gidx:3 * gidx + 3].copy(), prob["gnss_std"][3 * gidx:3 * gidx + 3].copy(), np.array(prob["lever"], np.float64)]
    oracle.icgo_gnss_eval(oa._p(a[0]), oa._p(a[1]), oa._p(a[2]), oa._p(a[3]), oa._p(ro), oa._p(Jg_o))
    assert np.abs(r_gn - ro).max() <= 1e-12 * max(1.0, np.abs(ro).max()) and np.abs(Jg - Jg_o.ravel()).max() <= 1e-12 * np.abs(Jg_o).max()
