"""Device INS windows for B streams (csrc/ins.cu): the per-sample mechanization of GVINS::runFusion (ic_gvins.cc:249-293), the post-solve
redo (MISC::redoInsMechanization, misc.cc:208-261) and each frame's prior camera pose (MISC::getCameraPoseFromInsWindow, misc.cc:67-108).

Rows are (time, dt, dtheta[3], dvel[3]); states are (time, p[3], q_xyzw[4], v[3], bg[3], ba[3]); poses are (R row-major, t), 12 doubles.
A configuration is a dict {"with_earth": bool, "gravity": (3,), "iewn": (3,)} or a list of them, one per stream.

InsWindow.gins_initialize is GVINS::gvinsInitialization (ic_gvins.cc:584-692) for B streams: an initialization input is a dict with the
fields of icg_gins_init (gnss_time, gnss_blh, last_time, last_blh, last_yaw_valid, last_yaw, origin_blh, gravity, antlever, imudatarate;
gnss_std / last_std optional)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import GinsInit, GinsInitOut, InsConfig, check, lib, vp

RESERVED_INS_NUM = 2  # GVINS::reserved_ins_num_ (ic_gvins.cc:82)


def _configs(cfg, n: int):
    cs = [cfg] * n if isinstance(cfg, dict) else list(cfg)
    assert len(cs) == n, "one configuration per stream"
    arr = (InsConfig * max(n, 1))()
    for s, c in enumerate(cs):
        arr[s].with_earth = 1 if c.get("with_earth", False) else 0
        arr[s].gravity[:] = [float(x) for x in c["gravity"]]
        arr[s].iewn[:] = [float(x) for x in c.get("iewn", (0.0, 0.0, 0.0))]
    return arr


def _f64(a, cols: int) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, np.float64).reshape(-1, cols))


class InsWindow:
    def __init__(self, max_streams: int, capacity: int = 1000, device: int = 0, stream=None):
        self.max_streams, self.capacity = max_streams, capacity
        self._h = vp()
        check(lib().icg_ins_create(C.byref(self._h), max_streams, capacity, device, vp(stream) if stream else None), "icg_ins_create")

    def close(self):
        if getattr(self, "_h", None):
            lib().icg_ins_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def push(self, rows, cfg) -> None:
        """rows: a list of n_streams arrays (k_s x 8), one per stream (k_s may be 0).  Asynchronous; raises IcgError on rejection."""
        n = len(rows)
        parts = [_f64(r, 8) for r in rows]
        off = np.zeros(n + 1, np.int32)
        off[1:] = np.cumsum([p.shape[0] for p in parts])
        imu = np.ascontiguousarray(np.concatenate(parts) if n else np.zeros((0, 8)))
        c = _configs(cfg, n)
        check(lib().icg_ins_push(self._h, n, c, vp(off.ctypes.data), vp(imu.ctypes.data) if imu.size else None), "icg_ins_push")

    def redo(self, state17, cfg, redo=None, reserved: int = RESERVED_INS_NUM) -> np.ndarray:
        """state17: n x 17 optimized states; returns status (n,) int8: 1 redone, 0 not selected, -1 time outside the window."""
        st = _f64(state17, 17)
        n = st.shape[0]
        status = np.zeros(n, np.int8)
        sel = None if redo is None else np.ascontiguousarray(np.asarray(redo, np.uint8))
        check(lib().icg_ins_redo(self._h, n, _configs(cfg, n), vp(sel.ctypes.data) if sel is not None else None, vp(st.ctypes.data), int(reserved),
                                 vp(status.ctypes.data)), "icg_ins_redo")
        return status

    def gins_initialize(self, inits, cfg, noise5, station3=(0.0, 0.0, 0.0), sel=None, reserved: int = RESERVED_INS_NUM):
        """gvinsInitialization of the selected streams (sel: n flags, None: all).  Returns (out, cfg): out is a dict of numpy arrays over the
        n streams -- status (1 initialized, 0 not selected, -1 .. -5 as icg_ins_gins_initialize), has_zero_velocity, bg (n, 3), initatt (n, 3),
        state17 (n, 2, 17), pose_prior (n, 7), pose_prior_std (n, 6), mix_prior (n, 9), mix_prior_std (n, 9), imu_blob (n, 480), n_series --
        and cfg the configurations as the call left them (gravity and, in the Earth form, iewn set where status == 1)."""
        n = len(inits)
        c = _configs(cfg, n)
        arr = (GinsInit * max(n, 1))()
        for s, g in enumerate(inits):
            a = arr[s]
            for k in ("gnss_time", "last_time", "last_yaw", "gravity", "imudatarate"):
                setattr(a, k, float(g.get(k, 0.0)))
            a.last_yaw_valid = 1 if g.get("last_yaw_valid", False) else 0
            for k in ("gnss_blh", "gnss_std", "last_blh", "last_std", "origin_blh", "antlever"):
                getattr(a, k)[:] = [float(x) for x in g.get(k, (0.0, 0.0, 0.0))]
        res = (GinsInitOut * max(n, 1))()
        nz = np.ascontiguousarray(np.asarray(noise5, np.float64).reshape(5))
        stn = np.ascontiguousarray(np.asarray(station3, np.float64).reshape(3))
        sl = None if sel is None else np.ascontiguousarray(np.asarray(sel, np.uint8).reshape(n))
        check(lib().icg_ins_gins_initialize(self._h, n, c, vp(sl.ctypes.data) if sl is not None else None, arr, vp(nz.ctypes.data),
                                            vp(stn.ctypes.data), int(reserved), res), "icg_ins_gins_initialize")
        out = {k: np.array([getattr(res[s], k) for s in range(n)], np.int32) for k in ("status", "has_zero_velocity", "n_series")}
        for k, shape in (("bg", (3,)), ("initatt", (3,)), ("state17", (2, 17)), ("pose_prior", (7,)), ("pose_prior_std", (6,)),
                         ("mix_prior", (9,)), ("mix_prior_std", (9,)), ("imu_blob", (480,))):
            out[k] = np.array([np.ctypeslib.as_array(getattr(res[s], k)) for s in range(n)], np.float64).reshape((n,) + shape)
        cfg_out = [{"with_earth": bool(c[s].with_earth), "gravity": tuple(c[s].gravity), "iewn": tuple(c[s].iewn)} for s in range(n)]
        return out, cfg_out

    def camera_pose(self, stamp, pose_b_c, dev_pose=None):
        """Prior camera poses at stamp (n,) with pose_b_c (n x 12 or one 12-vector for all).  dev_pose: a torch float64 CUDA tensor (n, 12)
        or None (one is allocated).  Returns (host_pose (n, 12), found (n,) int32, dev_pose).  The handle writes dev_pose on its own stream,
        so the work torch has queued on its current stream (an allocation, a fill of dev_pose) completes first."""
        import torch
        t = np.ascontiguousarray(np.asarray(stamp, np.float64).reshape(-1))
        n = t.shape[0]
        bc = _f64(pose_b_c, 12)
        if bc.shape[0] == 1 and n > 1:
            bc = np.ascontiguousarray(np.repeat(bc, n, axis=0))
        if dev_pose is None:
            dev_pose = torch.empty((max(n, 1), 12), dtype=torch.float64, device="cuda")
        torch.cuda.current_stream(dev_pose.device).synchronize()
        host = np.zeros((n, 12))
        found = np.zeros(n, np.int32)
        check(lib().icg_ins_camera_pose(self._h, n, vp(t.ctypes.data), vp(bc.ctypes.data), vp(dev_pose.data_ptr()), vp(host.ctypes.data),
                                        vp(found.ctypes.data)), "icg_ins_camera_pose")
        return host, found, dev_pose

    def window(self, stream: int):
        """(rows (count x 8), states (count x 17)) of one stream, oldest first."""
        count = C.c_int32(0)
        check(lib().icg_ins_window(self._h, stream, 0, C.byref(count), None, None), "icg_ins_window")
        imu = np.zeros((count.value, 8))
        st = np.zeros((count.value, 17))
        check(lib().icg_ins_window(self._h, stream, count.value, C.byref(count), vp(imu.ctypes.data), vp(st.ctypes.data)), "icg_ins_window")
        return imu, st

    def sync(self) -> None:
        check(lib().icg_ins_sync(self._h), "icg_ins_sync")
