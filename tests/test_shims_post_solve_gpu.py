"""The C++ shims of the post-solve step EXECUTED on the GPU: a program that includes ic_gvins_b200/host/icg_shims.hpp runs
WindowSolver::gvinsOptimization -> updateAndCull -> marginalization(culled, node_in_map) on one window and must give the same flags,
poses and prior, bit for bit, as the Python binding of the same calls."""
import copy
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import oracle_api as oa
from tests.test_post_solve_gpu import CAMD, STD, cull_inputs, make

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

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
template <typename T> static std::vector<double> dv(const T *p, size_t n) { return std::vector<double>(p, p + n); }

int main(int argc, char **argv) {
    try {
        FILE *in = fopen(argv[1], "rb");
        auto dims = as<int>(rd(in));  // K L F
        const int K = dims[0], L = dims[1], F = dims[2];
        auto pose = rd(in), mix = rd(in), ext = rd(in), rho = rd(in), fc = rd(in), blob = rd(in), scal = rd(in);
        auto f_lm = as<int32_t>(rd(in)), f_ref = as<int32_t>(rd(in)), f_obs = as<int32_t>(rd(in));
        auto gnode = as<int32_t>(rd(in));
        auto gblh = rd(in), gstd = rd(in), lever = rd(in);
        auto Rbc = rd(in), tbc = rd(in);
        auto lm_ref = as<int32_t>(rd(in));
        auto lm_kp = as<float>(rd(in));
        auto off = as<int32_t>(rd(in)), onode = as<int32_t>(rd(in));
        auto okp = as<float>(rd(in));
        auto ofac = as<int32_t>(rd(in));
        auto nim = rd(in);
        fclose(in);
        std::vector<uint8_t> act(F, 1), in_map(nim.begin(), nim.end());
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
        icg_camera cam{scal[1], scal[2], scal[3], scal[4], 0, 0, 0, 0, 0, 0};
        std::vector<double> cam_pose(12 * K), pw(3 * L), depth(L);
        std::vector<uint8_t> lmo(L), obo(onode.size());
        icg_ba_cull_window io{};
        for (int i = 0; i < 9; i++) io.R_bc[i] = Rbc[i];
        for (int i = 0; i < 3; i++) io.t_bc[i] = tbc[i];
        io.estimate_ext = io.estimate_td = 1;
        io.lm_ref_node = lm_ref.data(), io.lm_ref_kp = lm_kp.data(), io.obs_off = off.data(), io.obs_node = onode.data(), io.obs_kp = okp.data();
        io.obs_factor = ofac.data(), io.cam_pose = cam_pose.data(), io.lm_pw = pw.data(), io.lm_depth = depth.data(), io.lm_outlier = lmo.data();
        io.obs_outlier = obo.data();
        solver.updateAndCull(p, cam, scal[5], io);
        auto P = solver.marginalization(p, 1, io, in_map.data());
        FILE *out = fopen(argv[2], "wb");
        wr(out, {(double) io.ext_accepted, (double) io.counts[0], (double) io.counts[1], (double) io.counts[2], (double) io.counts[3], (double) io.counts[4]});
        wr(out, cam_pose), wr(out, pw), wr(out, dv(lmo.data(), lmo.size())), wr(out, dv(obo.data(), obo.size()));
        wr(out, P.J0), wr(out, P.e0), wr(out, pose), wr(out, rho);
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
def test_cpp_post_solve_shims_run_on_the_gpu(oracle):
    from ic_gvins_b200.ba import WindowSolver
    from ic_gvins_b200.camera import Camera
    oa.declare_ba(oracle)
    lib = os.path.join(ROOT, "ic_gvins_b200", "libicgvins_b200.so")
    prob = make(oracle, outliers=10, seed=211, K=8, L=150)
    ci = cull_inputs(prob, prob["ext"].copy(), 212, bad_kp=15)
    nim = np.ones(prob["K"], np.uint8)
    nim[6] = 0
    # the same calls through the Python binding
    py = copy.deepcopy(prob)
    s = WindowSolver(max_windows=1, max_K=prob["K"], max_L=prob["L"], max_F=prob["F"], max_gnss=16, max_marg_r=160)
    try:
        s.gvins_optimization_batch([py], 20)
        g = s.update_and_cull([py], Camera([CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"]], [0.0] * 4), STD, [ci])[0]
        m = s.marginalize([py], 1, resident=True, culled=[g], node_in_map=[nim])[0]
    finally:
        s.close()
    with tempfile.TemporaryDirectory() as td:
        cpp, exe, fin, fout = (os.path.join(td, x) for x in ("shim.cpp", "shim", "in.bin", "out.bin"))
        open(cpp, "w").write(SRC)
        r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", ROOT, cpp, "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        with open(fin, "wb") as fh:
            for arr in ([prob["K"], prob["L"], prob["F"]], prob["pose"], prob["mix"], prob["ext"], prob["invdepth"], prob["f_const"], prob["imu_blob"],
                        [prob["reproj_std"], CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"], STD], prob["f_lm"], prob["f_ref"], prob["f_obs"],
                        prob["gnss_node"], prob["gnss_blh"], prob["gnss_std"], prob["lever"],
                        ci["R_bc"], ci["t_bc"], ci["lm_ref_node"], ci["lm_ref_kp"], ci["obs_off"], ci["obs_node"], ci["obs_kp"], ci["obs_factor"], nim):
                _wr(fh, arr)
        r = subprocess.run([exe, fin, fout], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, (r.returncode, r.stderr)
        with open(fout, "rb") as fh:
            head, cam_pose, pw, lmo, obo, J0, e0, pose, rho = (_rd(fh) for _ in range(9))
    assert head[0] == g["ext_accepted"] and np.array_equal(head[1:].astype(np.int32), g["counts"])
    assert np.array_equal(pose, py["pose"]) and np.array_equal(rho, py["invdepth"])
    assert np.array_equal(cam_pose, g["cam_pose"].ravel()) and np.array_equal(pw, g["lm_pw"].ravel())
    assert np.array_equal(lmo.astype(np.uint8), g["lm_outlier"]) and np.array_equal(obo.astype(np.uint8), g["obs_outlier"])
    assert np.array_equal(J0, m["J0"].ravel()) and np.array_equal(e0, m["e0"])
