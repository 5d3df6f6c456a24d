"""ctypes access to the CPU restatement of the GNSS/INS initialization (tests/gins_init_oracle.cpp, which includes tests/ins_oracle.cpp).
TEST INFRASTRUCTURE ONLY.

The library is compiled on first use into a per-user temporary directory, keyed by both sources' hash, so the tree stays read-only."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tests import ins_oracle as io

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "gins_init_oracle.cpp")
HAVE_CXX = io.HAVE_CXX
MAX_SERIES = 1002  # an unmechanized window's 1000 rows + the two interpolated ends
vp = C.c_void_p
_lib = None
_p = io._p
IN_FIELDS = ("gnss_time", "gnss_blh", "last_time", "last_blh", "last_yaw_valid", "last_yaw", "origin_blh", "gravity", "antlever", "imudatarate")


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        src = open(SRC, "rb").read() + open(io.SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), f"icg_ins_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"gins_init_oracle_{hashlib.sha1(src).hexdigest()[:16]}.so")
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
        L.icgo_ins_window.argtypes = [vp, C.c_int, C.c_int, vp, vp]
        L.icgo_ins_redo.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp]
        L.icgo_ins_redo.restype = None
        L.icgo_gins_initialize.argtypes = [vp, C.c_int, vp, vp, vp, C.c_double, C.c_int, vp, vp, vp, vp, C.c_int, vp, vp]
        L.icgo_gins_initialize.restype = None
        L.icgo_earth_iewn.argtypes = [vp, vp, vp]
        L.icgo_earth_iewn.restype = None
        L.icgo_euler2quaternion.argtypes = [vp, vp]
        L.icgo_euler2quaternion.restype = None
        _lib = L
    return _lib


def pack_in(inits) -> np.ndarray:
    """initialization inputs (dicts as InsWindow.gins_initialize takes them) as the oracle's n x 24 rows"""
    out = np.zeros((len(inits), 24))
    for s, g in enumerate(inits):
        out[s, :18] = [g["gnss_time"], *g["gnss_blh"], g["last_time"], *g["last_blh"], 1.0 if g.get("last_yaw_valid") else 0.0,
                       g.get("last_yaw", 0.0), *g.get("origin_blh", (0, 0, 0)), g["gravity"], *g.get("antlever", (0, 0, 0)), g["imudatarate"]]
    return out


class OracleGins:
    """The oracle's INS windows with gvinsInitialization's function statics kept per stream (bg, initatt, has_zero_velocity)."""

    def __init__(self, n_streams: int, capacity: int = 1000):
        self.n, self._h = n_streams, lib().icgo_ins_new(n_streams, capacity)
        self.slot7 = np.zeros((n_streams, 7))

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
        c7 = io.cfg7(cfg, n)
        return lib().icgo_ins_push(self._h, n, _p(c7), _p(off), _p(imu))

    def redo(self, state17, cfg, redo=None, reserved: int = 2) -> np.ndarray:
        st = np.ascontiguousarray(np.asarray(state17, np.float64).reshape(-1, 17))
        n = st.shape[0]
        status = np.zeros(n, np.int8)
        sel = None if redo is None else np.ascontiguousarray(np.asarray(redo, np.uint8))
        c7 = io.cfg7(cfg, n)
        lib().icgo_ins_redo(self._h, n, _p(c7), _p(sel), _p(st), int(reserved), _p(status))
        return status

    def window(self, stream: int):
        n = lib().icgo_ins_window(self._h, stream, 0, None, None)
        imu, st = np.zeros((n, 8)), np.zeros((n, 17))
        lib().icgo_ins_window(self._h, stream, n, _p(imu), _p(st))
        return imu, st

    def gins_initialize(self, inits, cfg, gyr_bias_std: float, sel=None, reserved: int = 2):
        """returns a dict: status, has_zero_velocity, bg, initatt, state17 (statedatalist_[0]), pose_prior, pose_prior_std, mix_prior,
        mix_prior_std, series (list of k x 8 arrays, the time column included), n_series; and the configurations as left (list of dicts)"""
        n = len(inits)
        c7 = io.cfg7(cfg, n)
        g24 = np.ascontiguousarray(pack_in(inits))
        s = None if sel is None else np.ascontiguousarray(np.asarray(sel, np.uint8))
        status, nser = np.zeros(n, np.int32), np.zeros(n, np.int32)
        st, pr = np.zeros((n, 17)), np.zeros((n, 31))
        ser = np.zeros((n, MAX_SERIES, 8))
        slot = np.ascontiguousarray(self.slot7[:n].copy())
        lib().icgo_gins_initialize(self._h, n, _p(c7), _p(s), _p(g24), float(gyr_bias_std), int(reserved), _p(slot), _p(status), _p(st), _p(pr),
                                   MAX_SERIES, _p(ser), _p(nser))
        self.slot7[:n] = slot
        out = {"status": status, "has_zero_velocity": slot[:, 6].astype(np.int32), "bg": slot[:, :3].copy(), "initatt": slot[:, 3:6].copy(),
               "state17": st, "pose_prior": pr[:, :7], "pose_prior_std": pr[:, 7:13], "mix_prior": pr[:, 13:22], "mix_prior_std": pr[:, 22:31],
               "series": [ser[k, :nser[k]].copy() for k in range(n)], "n_series": nser}
        cfg_out = [{"with_earth": bool(c7[k, 0]), "gravity": tuple(c7[k, 1:4]), "iewn": tuple(c7[k, 4:7])} for k in range(n)]
        return out, cfg_out


def earth_iewn(origin3, local3) -> np.ndarray:
    o, l3, out = np.ascontiguousarray(origin3, np.float64), np.ascontiguousarray(local3, np.float64), np.zeros(3)
    lib().icgo_earth_iewn(_p(o), _p(l3), _p(out))
    return out


def euler2quaternion(euler3) -> np.ndarray:
    e, q = np.ascontiguousarray(euler3, np.float64), np.zeros(4)
    lib().icgo_euler2quaternion(_p(e), _p(q))
    return q
