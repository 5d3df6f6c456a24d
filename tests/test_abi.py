"""CPU-only: the C-ABI library loads and exports every symbol include/icgvins_b200.h declares (no compute calls)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    text = open(os.path.join(ROOT, "include", "icgvins_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(icg_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from ic_gvins_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        from ic_gvins_b200 import build
        build.build()
    L = C.CDLL(_lib.LIB_PATH)
    names = _declared()
    assert len(names) >= 10
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, missing
    assert set(_lib.EXPORTS) == set(names), (set(_lib.EXPORTS) ^ set(names))


def test_argtypes_match_header_prototypes():
    """Every entry of _lib.ABI has as many argtypes as its prototype in include/icgvins_b200.h has parameters (a missing or extra argtype
    shifts every later argument without an error)."""
    from ic_gvins_b200 import _lib
    text = open(os.path.join(ROOT, "include", "icgvins_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    protos = {name: 0 if params.strip() in ("", "void") else params.count(",") + 1
              for name, params in re.findall(r"\b(icg_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", text)}
    assert set(protos) == set(_lib.ABI), set(protos) ^ set(_lib.ABI)
    wrong = {name: (len(argtypes), protos[name]) for name, (argtypes, _) in _lib.ABI.items() if len(argtypes) != protos[name]}
    assert not wrong, wrong


def test_no_cpu_fallback_without_gpu():
    """Without a CUDA device every create() must fail loudly (ICG_ENODEVICE), never fall back to the oracle."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from ic_gvins_b200 import IcgError
    from ic_gvins_b200.ba import WindowSolver
    from ic_gvins_b200.clahe import Clahe
    from ic_gvins_b200.detect import Detector
    from ic_gvins_b200.klt import KltTracker
    for make in (lambda: KltTracker(320, 240), lambda: Detector(320, 240), lambda: Clahe(320, 240), lambda: WindowSolver(max_windows=1)):
        with pytest.raises(IcgError, match="no CUDA device|no CPU fallback"):
            make()


def test_product_does_not_import_oracle():
    """The package must not reference oracle/ anywhere (the oracle is test infrastructure)."""
    pkg = os.path.join(ROOT, "ic_gvins_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cpp")):
                src = open(os.path.join(dirpath, f)).read()
                assert "icgo_" not in src and "libicg_oracle" not in src, f
                assert not re.search(r"^\s*(from|import)\s+oracle", src, flags=re.M), f
