"""CPU-only: the layout of icg_ba_ins_cut and icg_ba_slide_ins as a C compiler sees them match the ctypes images in ic_gvins_b200/_lib.py,
and the library exports the four sample-store calls."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ("icg_ba_imu_samples_from_ins", "icg_ba_slide_ins_resident", "icg_ba_reintegrate_stored_resident", "icg_ba_imu_samples")


@pytest.mark.skipif(shutil.which("gcc") is None, reason="gcc not available")
def test_layout_matches_ctypes():
    from ic_gvins_b200._lib import InsCut, SlideIns
    structs = (("icg_ba_ins_cut", InsCut), ("icg_ba_slide_ins", SlideIns))
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "include/icgvins_b200.h"\nint main(void) {\n'
    for name, cls in structs:
        src += f'    printf("%zu\\n", sizeof({name}));\n'
        src += "".join(f'    printf("%zu\\n", offsetof({name}, {f}));\n' for f, _ in cls._fields_)
    src += "    return 0;\n}\n"
    with tempfile.TemporaryDirectory() as td:
        c, exe = os.path.join(td, "layout.c"), os.path.join(td, "layout")
        open(c, "w").write(src)
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-I", ROOT, c, "-o", exe], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    want = []
    for _, cls in structs:
        want += [C.sizeof(cls)] + [getattr(cls, f).offset for f, _ in cls._fields_]
    assert out == want


def test_exports_the_store_calls():
    from ic_gvins_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        from ic_gvins_b200 import build
        build.build()
    L = C.CDLL(_lib.LIB_PATH)
    for name in CALLS:
        assert hasattr(L, name), name
        assert name in _lib.EXPORTS
