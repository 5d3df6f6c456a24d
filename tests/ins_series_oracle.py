"""ctypes access to getImuSeriesFromTo of the CPU restatement (tests/ins_series_oracle.cpp, which includes tests/gins_init_oracle.cpp and
tests/ins_oracle.cpp).  TEST INFRASTRUCTURE ONLY.

The library is compiled on first use into a per-user temporary directory, keyed by the sources' hash, so the tree stays read-only."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tests import gins_init_oracle as go
from tests import ins_oracle as io

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "ins_series_oracle.cpp")
HAVE_CXX = io.HAVE_CXX
vp = C.c_void_p
_lib = None
_p = io._p


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        src = open(SRC, "rb").read() + open(go.SRC, "rb").read() + open(io.SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), f"icg_ins_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"ins_series_oracle_{hashlib.sha1(src).hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}"
            subprocess.run([io.CXX, "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-shared", "-o", tmp, SRC], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.icgo_ins_new.restype = vp
        L.icgo_ins_new.argtypes = [C.c_int, C.c_int]
        L.icgo_ins_free.argtypes = [vp]
        L.icgo_ins_free.restype = None
        L.icgo_ins_push.argtypes = [vp, C.c_int, vp, vp, vp]
        L.icgo_ins_redo.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp]
        L.icgo_ins_redo.restype = None
        L.icgo_imu_series.argtypes = [vp, C.c_int, C.c_double, C.c_double, C.c_int, vp]
        _lib = L
    return _lib


class OracleSeries:
    """The oracle's INS windows (push and redo as tests/ins_oracle.py's) and getImuSeriesFromTo on them."""

    def __init__(self, n_streams: int, capacity: int = 1000):
        self.n, self._h = n_streams, lib().icgo_ins_new(n_streams, capacity)

    def close(self):
        if self._h:
            lib().icgo_ins_free(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def push(self, rows, cfg) -> int:
        n = len(rows)
        parts = [np.asarray(r, np.float64).reshape(-1, 8) for r in rows]
        off = np.zeros(n + 1, np.int32)
        off[1:] = np.cumsum([p.shape[0] for p in parts])
        imu = np.ascontiguousarray(np.concatenate(parts) if n else np.zeros((0, 8)))
        return lib().icgo_ins_push(self._h, n, _p(io.cfg7(cfg, n)), _p(off), _p(imu))

    def redo(self, state17, cfg, reserved: int = 2) -> np.ndarray:
        st = np.ascontiguousarray(np.asarray(state17, np.float64).reshape(-1, 17))
        status = np.zeros(st.shape[0], np.int8)
        lib().icgo_ins_redo(self._h, st.shape[0], _p(io.cfg7(cfg, st.shape[0])), None, _p(st), int(reserved), _p(status))
        return status

    def series(self, stream: int, start: float, end: float):
        """(m, 7) rows (dt, dtheta, dvel) of getImuSeriesFromTo(start, end), or None where the product refuses the interval"""
        out = np.zeros((1100, 8))
        m = lib().icgo_imu_series(self._h, int(stream), float(start), float(end), out.shape[0], _p(out))
        return None if m < 0 else out[:m, 1:].copy()
