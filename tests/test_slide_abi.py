"""CPU-only: the layout of icg_ba_slide_window as a C compiler sees it matches the ctypes image in ic_gvins_b200/_lib.py, and the C++ shim's
WindowSolver::slideWindow compiles and links against the library (never executed: no GPU here)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("node_src", "lm_src", "f_src", "imu_src", "gnss_src", "prior_from_marg")


def _lib_path():
    from ic_gvins_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        from ic_gvins_b200 import build
        build.build()
    return _lib.LIB_PATH


@pytest.mark.skipif(shutil.which("gcc") is None, reason="gcc not available")
def test_slide_window_layout_matches_ctypes():
    from ic_gvins_b200._lib import SlideWindow
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "include/icgvins_b200.h"\nint main(void) {\n'
    src += '    printf("%zu\\n", sizeof(icg_ba_slide_window));\n'
    src += "".join(f'    printf("%zu\\n", offsetof(icg_ba_slide_window, {f}));\n' for f in FIELDS)
    src += "    return 0;\n}\n"
    with tempfile.TemporaryDirectory() as td:
        c, exe = os.path.join(td, "layout.c"), os.path.join(td, "layout")
        open(c, "w").write(src)
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-I", ROOT, c, "-o", exe], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert out[0] == C.sizeof(SlideWindow)
    assert out[1:] == [getattr(SlideWindow, f).offset for f in FIELDS]


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_shim_slide_window_compiles_and_links():
    lib = _lib_path()
    src = r'''
#include "ic_gvins_b200/host/icg_shims.hpp"
int main(int argc, char **) {
    if (argc > 1000) {
        icg_b200::WindowSolver s(10, 300, 2700);
        icg_ba_problem P{};
        icg_b200::WindowSolver::Carry c;
        c.node_src = {1, 2, -1};
        s.slideWindow(P, c, true);
        icg_ba_summary o[2];
        int32_t culled[2];
        s.gvinsOptimizationResident(P, 20, o, culled);
    }
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as td:
        cpp, exe = os.path.join(td, "slide_shim.cpp"), os.path.join(td, "slide_shim")
        open(cpp, "w").write(src)
        r = subprocess.run(["g++", "-std=c++17", "-Wall", "-I", ROOT, cpp, "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        r = subprocess.run([exe], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
