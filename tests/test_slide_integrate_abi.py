"""CPU-only: the layout of icg_ba_slide_integrate and the ICG_SLIDE_* codes as a C compiler sees them match the ctypes image in
ic_gvins_b200/_lib.py, icg_ba_slide_integrate_resident rejects missing arguments before it touches a device, and the C++ shim's
WindowSolver::slideWindow overload compiles and links against the library (never executed: no GPU here)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("imu_from", "state16", "gravity3", "normal", "imu", "imu_off", "node_from_imu", "gnss_node", "gnss_dt", "status", "blob_out",
          "end_state10")


def _lib_path():
    from ic_gvins_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        from ic_gvins_b200 import build
        build.build()
    return _lib.LIB_PATH


@pytest.mark.skipif(shutil.which("gcc") is None, reason="gcc not available")
def test_slide_integrate_layout_matches_ctypes():
    from ic_gvins_b200._lib import SLIDE_CHAIN, SLIDE_ROW, SlideIntegrate
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "include/icgvins_b200.h"\nint main(void) {\n'
    src += '    printf("%d %d\\n", ICG_SLIDE_CHAIN, ICG_SLIDE_ROW);\n'
    src += '    printf("%zu\\n", sizeof(icg_ba_slide_integrate));\n'
    src += "".join(f'    printf("%zu\\n", offsetof(icg_ba_slide_integrate, {f}));\n' for f in FIELDS)
    src += "    return 0;\n}\n"
    with tempfile.TemporaryDirectory() as td:
        c, exe = os.path.join(td, "layout.c"), os.path.join(td, "layout")
        open(c, "w").write(src)
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-I", ROOT, c, "-o", exe], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert out[:2] == [SLIDE_CHAIN, SLIDE_ROW]
    assert out[2] == C.sizeof(SlideIntegrate)
    assert out[3:] == [getattr(SlideIntegrate, f).offset for f in FIELDS]


def test_missing_arguments_are_rejected_without_a_device():
    _lib_path()
    from ic_gvins_b200._lib import SlideIntegrate, SlideWindow, lib
    L = lib()
    integ, carry = SlideIntegrate(), SlideWindow()
    nz = (C.c_double * 5)(1, 1, 1, 1, 1)
    stn = (C.c_double * 3)()
    for args in ((None, 1, None, C.byref(carry), None, nz, stn),             # no integrate array
                 (None, 1, None, C.byref(carry), C.byref(integ), nz, stn)):   # no handle
        assert L.icg_ba_slide_integrate_resident(*args) == -1  # ICG_EINVAL
        assert b"bad arguments" in L.icg_last_error()


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_shim_slide_integrate_compiles_and_links():
    lib = _lib_path()
    src = r'''
#include "ic_gvins_b200/host/icg_shims.hpp"
int main(int argc, char **) {
    if (argc > 1000) {
        icg_b200::WindowSolver s(10, 300, 2700);
        icg_ba_problem P{};
        icg_b200::WindowSolver::Carry c;
        c.node_src = {1, 2, -1};
        std::vector<int32_t> from = {-1, 1}, off = {0, 0, 100};
        std::vector<double> grav = {0, 0, 0, 0, 0, 9.8}, rows(700);
        std::vector<uint8_t> node = {0, 0, 1};
        std::vector<int8_t> status(2);
        icg_ba_slide_integrate g{};
        g.imu_from = from.data(), g.gravity3 = grav.data(), g.imu = rows.data(), g.imu_off = off.data(), g.node_from_imu = node.data();
        g.status = status.data();
        const double noise5[5] = {1, 1, 1, 1, 3600}, station[3] = {0, 0, 0};
        s.slideWindow(P, c, true, g, noise5, station);
        icg_ba_summary o[2];
        int32_t culled[2];
        s.gvinsOptimizationResident(P, 20, o, culled);
    }
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as td:
        cpp, exe = os.path.join(td, "slide_integrate_shim.cpp"), os.path.join(td, "slide_integrate_shim")
        open(cpp, "w").write(src)
        r = subprocess.run(["g++", "-std=c++17", "-Wall", "-I", ROOT, cpp, "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        r = subprocess.run([exe], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
