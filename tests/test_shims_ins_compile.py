"""The C++ shims of the INS windows and the window solver's IMU sample store (ic_gvins_b200/host/icg_shims.hpp: InsWindows, and
WindowSolver's imuSamplesFromIns / INS slideWindow / stored doReintegration / imuSamples) compile as plain C++17 and link against the
library's exports.  CPU only (no compute calls)."""
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_ins_shims_compile_and_link():
    lib = os.path.join(ROOT, "ic_gvins_b200", "libicgvins_b200.so")
    if not os.path.exists(lib):
        from ic_gvins_b200 import build
        build.build()
    src = r'''
#include "ic_gvins_b200/host/icg_shims.hpp"
// instantiate every new shim member so that its C-ABI symbols are referenced (never executed: no GPU here)
int main(int argc, char **) {
    if (argc > 1000) {
        icg_b200::InsWindows ins(4);
        icg_ins_config cfg[1] = {};
        const int32_t off[2] = {0, 0};
        ins.push(1, cfg, off, nullptr);
        double st[17] = {0}, pose[12], stamp = 0, bc[12] = {0};
        int8_t status = 0;
        int32_t found = 0;
        ins.redo(1, cfg, nullptr, st, 2, &status);
        ins.cameraPose(1, &stamp, bc, pose, pose, &found);
        icg_gins_init in{};
        icg_gins_init_out out{};
        const double noise5[5] = {0}, station[3] = {0};
        ins.ginsInitialize(1, cfg, nullptr, &in, noise5, station, 2, &out);
        std::vector<double> imu8, state17;
        ins.window(0, imu8, state17);
        icg_b200::WindowSolver s(10, 300, 2700);
        icg_ba_problem P{};
        std::vector<double> times(2), blobs, ends, rows;
        s.imuSamplesFromIns(ins, 0, times);
        icg_ba_slide_integrate g{};
        std::vector<int32_t> merge, n_rows, offs;
        s.slideWindow(P, icg_b200::WindowSolver::Carry{}, true, g, ins, 0, times, merge, noise5, station, &n_rows);
        std::vector<int8_t> st8;
        s.doReintegration(P, noise5, station, st8, blobs, &ends);
        s.imuSamples(1, offs, rows);
    }
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as td:
        cpp = os.path.join(td, "shim_ins_test.cpp")
        exe = os.path.join(td, "shim_ins_test")
        open(cpp, "w").write(src)
        r = subprocess.run(["g++", "-std=c++17", "-Wall", "-I", ROOT, cpp, "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        r = subprocess.run([exe], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
