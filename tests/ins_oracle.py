"""ctypes access to the CPU restatement of the INS window (tests/ins_oracle.cpp).  TEST INFRASTRUCTURE ONLY.

The library is compiled on first use into a per-user temporary directory, keyed by the source's hash, so the tree stays read-only."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "ins_oracle.cpp")
CXX = os.environ.get("CXX", "g++")
HAVE_CXX = shutil.which(CXX) is not None  # the tests that need the restatement skip without a host C++ compiler
vp = C.c_void_p
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        src = open(SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), f"icg_ins_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"ins_oracle_{hashlib.sha1(src).hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}"
            subprocess.run([CXX, "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-shared", "-o", tmp,
                            SRC], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.icgo_ins_new.restype = vp
        L.icgo_ins_new.argtypes = [C.c_int, C.c_int]
        L.icgo_ins_free.argtypes = [vp]
        L.icgo_ins_free.restype = None
        L.icgo_ins_push.argtypes = [vp, C.c_int, vp, vp, vp]
        L.icgo_ins_redo.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp]
        L.icgo_ins_redo.restype = None
        L.icgo_ins_camera_pose.argtypes = [vp, C.c_int, vp, vp, vp, vp]
        L.icgo_ins_camera_pose.restype = None
        L.icgo_ins_window.argtypes = [vp, C.c_int, C.c_int, vp, vp]
        L.icgo_ins_mechanize.argtypes = [vp, vp, vp, vp]
        L.icgo_ins_mechanize.restype = None
        L.icgo_ins_window_index.argtypes = [C.c_int, vp, C.c_double]
        L.icgo_ins_need_interpolation.argtypes = [C.c_double, C.c_double, C.c_double]
        L.icgo_ins_interpolate.argtypes = [vp, C.c_double, vp, vp]
        L.icgo_ins_interpolate.restype = None
        L.icgo_ins_pose_interpolate.argtypes = [vp, vp, C.c_double, vp, vp]
        L.icgo_ins_pose_interpolate.restype = None
        _lib = L
    return _lib


def _p(a: np.ndarray):
    return vp(a.ctypes.data) if a is not None and a.size else None


def cfg7(cfg, n: int) -> np.ndarray:
    """configuration dict(s) as the oracle's n x 7 rows (with_earth, gravity[3], iewn[3])"""
    cs = [cfg] * n if isinstance(cfg, dict) else list(cfg)
    return np.ascontiguousarray(np.array([[1.0 if c.get("with_earth") else 0.0, *c["gravity"], *c.get("iewn", (0, 0, 0))] for c in cs],
                                         np.float64).reshape(n, 7))


class OracleIns:
    """The oracle's multi-stream INS windows: the same calls as ic_gvins_b200.ins.InsWindow, on std::deque."""

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
        c7 = cfg7(cfg, n)  # kept alive across the call
        return lib().icgo_ins_push(self._h, n, _p(c7), _p(off), _p(imu))

    def push_packed(self, c7: np.ndarray, off: np.ndarray, imu: np.ndarray) -> int:
        return lib().icgo_ins_push(self._h, off.shape[0] - 1, _p(c7), _p(off), _p(imu))

    def redo(self, state17, cfg, redo=None, reserved: int = 2) -> np.ndarray:
        st = np.ascontiguousarray(np.asarray(state17, np.float64).reshape(-1, 17))
        n = st.shape[0]
        status = np.zeros(n, np.int8)
        sel = None if redo is None else np.ascontiguousarray(np.asarray(redo, np.uint8))
        c7 = cfg7(cfg, n)
        lib().icgo_ins_redo(self._h, n, _p(c7), _p(sel), _p(st), int(reserved), _p(status))
        return status

    def camera_pose(self, stamp, pose_b_c):
        t = np.ascontiguousarray(np.asarray(stamp, np.float64).reshape(-1))
        n = t.shape[0]
        bc = np.ascontiguousarray(np.asarray(pose_b_c, np.float64).reshape(-1, 12))
        if bc.shape[0] == 1 and n > 1:
            bc = np.ascontiguousarray(np.repeat(bc, n, axis=0))
        pose = np.zeros((n, 12))
        found = np.zeros(n, np.int32)
        lib().icgo_ins_camera_pose(self._h, n, _p(t), _p(bc), _p(pose), _p(found))
        return pose, found

    def window(self, stream: int):
        n = lib().icgo_ins_window(self._h, stream, 0, None, None)
        imu, st = np.zeros((n, 8)), np.zeros((n, 17))
        lib().icgo_ins_window(self._h, stream, n, _p(imu), _p(st))
        return imu, st


def mechanize(cfg, pre8, cur8, state17) -> np.ndarray:
    st = np.ascontiguousarray(np.array(state17, np.float64))
    c7, pre, cur = cfg7(cfg, 1), np.ascontiguousarray(pre8, np.float64), np.ascontiguousarray(cur8, np.float64)
    lib().icgo_ins_mechanize(_p(c7), _p(pre), _p(cur), _p(st))
    return st


def window_index(times, t) -> int:
    tt = np.ascontiguousarray(np.asarray(times, np.float64))
    return lib().icgo_ins_window_index(tt.shape[0], _p(tt), float(t))


def need_interpolation(t0, t1, mid) -> int:
    return lib().icgo_ins_need_interpolation(float(t0), float(t1), float(mid))


def interpolate(row8, mid):
    a, b, row = np.zeros(8), np.zeros(8), np.ascontiguousarray(row8, np.float64)
    lib().icgo_ins_interpolate(_p(row), float(mid), _p(a), _p(b))
    return a, b


def pose_interpolate(state0, state1, mid, pose_b_c) -> np.ndarray:
    out = np.zeros(12)
    s0, s1, bc = (np.ascontiguousarray(v, np.float64) for v in (state0, state1, pose_b_c))
    lib().icgo_ins_pose_interpolate(_p(s0), _p(s1), float(mid), _p(bc), _p(out))
    return out
