"""Host-side mirror of the reference's KLT call sites (IG/tracking/tracking.cc:385-403, 487-506).

`KltTracker.calcOpticalFlowPyrLK` keeps OpenCV's argument list and return convention (as cv2 exposes it), so the
parity tests read like calls into the reference's own dependency.  Everything runs in libicgvins_b200.so.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import check, lib, vp
from .camera import CameraStruct

OPTFLOW_USE_INITIAL_FLOW = 4
TERM_COUNT, TERM_EPS = 1, 2


def _ptr(a: np.ndarray):
    return C.c_void_p(a.ctypes.data)


class TrackFrameStruct(C.Structure):
    """ctypes image of `icg_track_frame` (per-stream parameters of trackMappoint / trackReferenceFrame)."""
    _fields_ = [("prev_slot", C.c_int32), ("cur_slot", C.c_int32), ("camera", CameraStruct), ("R_pre", C.c_double * 9), ("R_cur", C.c_double * 9),
                ("R_ref", C.c_double * 9), ("t_cur", C.c_double * 3), ("dt", C.c_double), ("ref_id", C.c_int64), ("fm_threshold", C.c_double)]


MAP_IN = ("prev_xy", "prev_undis_xy", "pw", "ref_kp_xy")
MAP_OUT = ("fwd_xy", "fwd_undis_xy", "keep", "cur_xy", "cur_undis_xy", "velocity", "src")
REF_IN = ("new_xy", "ref_xy", "ref_frame_id", "velocity_ref")
REF_OUT = ("fwd_xy", "fwd_undis_xy", "keep", "cur_xy", "cur_undis_xy", "velocity", "ref_out_xy", "ref_frame_id_out", "velocity_ref_out", "src")


class TrackMapStruct(C.Structure):
    """ctypes image of `icg_track_map` (all pointers)."""
    _fields_ = [(k, C.c_void_p) for k in MAP_IN + MAP_OUT]


class TrackRefStruct(C.Structure):
    """ctypes image of `icg_track_ref` (all pointers)."""
    _fields_ = [(k, C.c_void_p) for k in REF_IN + REF_OUT]


# numpy (dtype, columns) of every list array; columns 1 = flat
_SPEC = {"prev_xy": (np.float32, 2), "prev_undis_xy": (np.float32, 2), "pw": (np.float64, 3), "ref_kp_xy": (np.float32, 2),
         "new_xy": (np.float32, 2), "ref_xy": (np.float32, 2), "ref_frame_id": (np.int64, 1), "velocity_ref": (np.float64, 2),
         "fwd_xy": (np.float32, 2), "fwd_undis_xy": (np.float32, 2), "keep": (np.uint8, 1), "cur_xy": (np.float32, 2),
         "cur_undis_xy": (np.float32, 2), "velocity": (np.float64, 2), "ref_out_xy": (np.float32, 2), "ref_frame_id_out": (np.int64, 1),
         "velocity_ref_out": (np.float64, 2), "src": (np.int32, 1)}


class TriFrameStruct(C.Structure):
    """ctypes image of `icg_tri_frame` (per-stream parameters of Tracking::triangulation)."""
    _fields_ = [("camera", CameraStruct), ("R_cur", C.c_double * 9), ("t_cur", C.c_double * 3), ("cur_id", C.c_int64), ("ref_id", C.c_int64),
                ("window_normal", C.c_int32), ("triangulate", C.c_int32), ("reprojection_error_std", C.c_double)]


class TriKeyframeStruct(C.Structure):
    """ctypes image of `icg_tri_keyframe` (a frame the reference list can name)."""
    _fields_ = [("id", C.c_int64), ("R", C.c_double * 9), ("t", C.c_double * 3), ("in_map", C.c_int32)]


TRI_LIST = ("ref_out_xy", "ref_frame_id_out", "cur_xy", "velocity_ref_out", "velocity", "src")
TRI_NEW = ("pw", "depth", "ref_undis_xy", "ref_xy", "cur_undis_xy", "cur_xy", "velocity_cur", "velocity_ref", "ref_frame_id", "src")
TRI_COUNTS = ("kept", "succeeded", "outlier", "reset", "outtime")


class TriListStruct(C.Structure):
    """ctypes image of `icg_tri_list` (all pointers)."""
    _fields_ = [(k, C.c_void_p) for k in TRI_LIST]


class TriNewStruct(C.Structure):
    """ctypes image of `icg_tri_new` (all pointers)."""
    _fields_ = [(k, C.c_void_p) for k in TRI_NEW]


# numpy (dtype, columns) of the new map points' arrays (the list arrays are in _SPEC)
_TRI_NEW_SPEC = {"pw": (np.float64, 3), "depth": (np.float64, 1), "ref_undis_xy": (np.float32, 2), "ref_xy": (np.float32, 2),
                 "cur_undis_xy": (np.float32, 2), "cur_xy": (np.float32, 2), "velocity_cur": (np.float64, 2), "velocity_ref": (np.float64, 2),
                 "ref_frame_id": (np.int64, 1), "src": (np.int32, 1)}


def tri_frame_params(intrinsic, distortion, R_cur, t_cur, cur_id, ref_id, window_normal, reprojection_error_std, triangulate=True) -> TriFrameStruct:
    """icg_tri_frame from Camera::createCamera's lists and frame_cur_'s camera-to-world pose"""
    i, d = list(map(float, intrinsic)), list(map(float, distortion))
    cam = CameraStruct(i[0], i[1], i[2], i[3], i[4] if len(i) == 5 else 0.0, d[0], d[1], d[2], d[3], d[4] if len(d) == 5 else 0.0)
    m = lambda a, n: (C.c_double * n)(*np.asarray(a, np.float64).reshape(n).tolist())  # noqa: E731
    return TriFrameStruct(cam, m(R_cur, 9), m(t_cur, 3), int(cur_id), int(ref_id), int(bool(window_normal)), int(bool(triangulate)),
                          float(reprojection_error_std))


def tri_keyframes(frames) -> C.Array:
    """icg_tri_keyframe array from an iterable of (id, R (3 x 3 camera-to-world), t (3), in_map)"""
    frames = list(frames)
    arr = (TriKeyframeStruct * max(len(frames), 1))()
    for e, (fid, R, t, in_map) in enumerate(frames):
        arr[e].id, arr[e].in_map = int(fid), int(bool(in_map))
        arr[e].R[:] = np.asarray(R, np.float64).reshape(9).tolist()
        arr[e].t[:] = np.asarray(t, np.float64).reshape(3).tolist()
    return arr


def track_frame_params(prev_slot, cur_slot, intrinsic, distortion, R_pre, R_cur, R_ref, t_cur, dt, ref_id, fm_threshold) -> TrackFrameStruct:
    """icg_track_frame from Camera::createCamera's intrinsic / distortion lists and camera-to-world attitudes (Pose::R, 3 x 3)."""
    i, d = list(map(float, intrinsic)), list(map(float, distortion))
    cam = CameraStruct(i[0], i[1], i[2], i[3], i[4] if len(i) == 5 else 0.0, d[0], d[1], d[2], d[3], d[4] if len(d) == 5 else 0.0)
    m = lambda a, n: (C.c_double * n)(*np.asarray(a, np.float64).reshape(n).tolist())  # noqa: E731
    return TrackFrameStruct(int(prev_slot), int(cur_slot), cam, m(R_pre, 9), m(R_cur, 9), m(R_ref, 9), m(t_cur, 3), float(dt), int(ref_id),
                            float(fm_threshold))


class KltTracker:
    """One tracker handle == one image geometry on one GPU (the reference has one Tracking object per camera)."""

    def __init__(self, width: int, height: int, n_slots: int = 4, max_points: int = 4096, device: int = 0, stream=None):
        self.W, self.H, self.n_slots, self.max_points = width, height, n_slots, max_points
        self._h = vp()
        check(lib().icg_klt_create(C.byref(self._h), width, height, n_slots, max_points, device,
                                   vp(stream) if stream else None), "icg_klt_create")

    def close(self):
        if getattr(self, "_h", None):
            lib().icg_klt_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ drop-in: cv2.calcOpticalFlowPyrLK
    def calcOpticalFlowPyrLK(self, prevImg, nextImg, prevPts, nextPts, winSize=(21, 21), maxLevel=3,
                             criteria=(TERM_COUNT + TERM_EPS, 30, 0.01), flags=0):
        prevImg = np.ascontiguousarray(prevImg, dtype=np.uint8)
        nextImg = np.ascontiguousarray(nextImg, dtype=np.uint8)
        if prevImg.shape != (self.H, self.W) or nextImg.shape != (self.H, self.W):
            raise ValueError("image size does not match the tracker")
        p = np.ascontiguousarray(prevPts, dtype=np.float32).reshape(-1, 2)
        n = p.shape[0]
        if flags & OPTFLOW_USE_INITIAL_FLOW:
            q = np.array(nextPts, dtype=np.float32).reshape(-1, 2).copy()
        else:
            q = p.copy()
        status = np.zeros(n, np.uint8)
        err = np.zeros(n, np.float32)
        # cv::calcOpticalFlowPyrLK's defaults for a criterion the type leaves out: 30 iterations, epsilon 0.01
        max_iter = criteria[1] if criteria[0] & TERM_COUNT else 30
        eps = criteria[2] if criteria[0] & TERM_EPS else 0.01
        check(lib().icg_klt_calc_optical_flow_pyr_lk(self._h, _ptr(prevImg), _ptr(nextImg), self.W, _ptr(p), _ptr(q),
                                                     _ptr(status), _ptr(err), n, winSize[0], maxLevel, max_iter,
                                                     float(eps), flags), "icg_klt_calc_optical_flow_pyr_lk")
        return q, status, err

    # ------------------------------------------------------------------ fused fwd+bwd+gates (tracking.cc:385-403)
    def track_fb(self, prevImg, nextImg, prevPts, predicted):
        prevImg = np.ascontiguousarray(prevImg, dtype=np.uint8)
        nextImg = np.ascontiguousarray(nextImg, dtype=np.uint8)
        p = np.ascontiguousarray(prevPts, dtype=np.float32).reshape(-1, 2)
        q = np.array(predicted, dtype=np.float32).reshape(-1, 2).copy()
        n = p.shape[0]
        back = np.zeros((n, 2), np.float32)
        status = np.zeros(n, np.uint8)
        check(lib().icg_klt_track_fb(self._h, _ptr(prevImg), _ptr(nextImg), self.W, _ptr(p), _ptr(q), _ptr(back),
                                     _ptr(status), n), "icg_klt_track_fb")
        return q, back, status

    # ------------------------------------------------------------------ device-resident API
    def upload(self, slot: int, img: np.ndarray, build: bool = True):
        img = np.ascontiguousarray(img, dtype=np.uint8)
        f = lib().icg_klt_upload if build else lib().icg_klt_upload_level0
        check(f(self._h, slot, _ptr(img), img.strides[0]), "icg_klt_upload")

    def upload_ptr(self, slot: int, host_ptr: int, stride: int, build: bool = True):
        f = lib().icg_klt_upload if build else lib().icg_klt_upload_level0
        check(f(self._h, slot, vp(host_ptr), stride), "icg_klt_upload")

    def upload_batch_ptrs(self, first_slot: int, host_ptrs, stride: int):
        """One call for the new frame of every stream: host_ptrs = iterable of host addresses (pinned), slots first_slot ...; no pyramid build."""
        arr = (C.c_void_p * len(host_ptrs))(*host_ptrs)
        check(lib().icg_klt_upload_batch(self._h, first_slot, len(host_ptrs), arr, stride), "icg_klt_upload_batch")

    def build_pyramids(self, first_slot: int, count: int):
        check(lib().icg_klt_build_pyramids(self._h, first_slot, count), "icg_klt_build_pyramids")

    def level_shape(self, level: int):
        w, h, pitch, ptr = C.c_int(), C.c_int(), C.c_int(), vp()
        check(lib().icg_klt_slot_level(self._h, 0, level, C.byref(ptr), C.byref(pitch), C.byref(w), C.byref(h)), "slot_level")
        return h.value, w.value

    def download_level(self, slot: int, level: int) -> np.ndarray:
        h, w = self.level_shape(level)
        out = np.zeros((h, w), np.uint8)
        check(lib().icg_klt_download_level(self._h, slot, level, _ptr(out), w), "icg_klt_download_level")
        return out

    def track_batch_dev(self, n_total: int, slots_ptr: int, prev_ptr: int, init_ptr: int, fwd_ptr: int, bwd_ptr: int,
                        status_ptr: int, mode: int = 1):
        check(lib().icg_klt_track_batch_dev(self._h, n_total, vp(slots_ptr), vp(prev_ptr), vp(init_ptr), vp(fwd_ptr),
                                            vp(bwd_ptr) if bwd_ptr else None, vp(status_ptr), mode), "icg_klt_track_batch_dev")

    # ------------------------------------------------------------------ trackMappoint + trackReferenceFrame (tracking.cc:351-574)
    def track_frame(self, params: TrackFrameStruct, map_lists=None, ref_lists=None):
        """One stream from host arrays (icg_klt_track_frame, synchronous).  map_lists: dict with prev_xy, prev_undis_xy (n, 2) float32, pw (n, 3),
        ref_kp_xy (n, 2) float32 (NaN = no feature in frame_ref_); ref_lists: dict with new_xy, ref_xy (m, 2) float32, ref_frame_id (m,) int64,
        velocity_ref (m, 2).  Either may be None (empty).  Returns (map_out, ref_out, n_out[2], parallax[2], parallax_n[2]); the outputs are the
        per-input fwd_xy / fwd_undis_xy / keep and the compacted lists cut to their counts."""
        def prep(lists, names_in, names_out, struct):
            lists = lists or {}
            n = len(lists[names_in[0]]) if names_in[0] in lists else 0
            arrs = {}
            for k in names_in:
                dt, c = _SPEC[k]
                arrs[k] = np.ascontiguousarray(np.asarray(lists[k], dt).reshape(n, c) if n else np.zeros((1, c), dt))
            for k in names_out:
                dt, c = _SPEC[k]
                arrs[k] = np.zeros((max(n, 1), c), dt)
            return n, arrs, struct(*[a.ctypes.data for a in (arrs[k] for k in names_in + names_out)])
        nm, am, sm = prep(map_lists, MAP_IN, MAP_OUT, TrackMapStruct)
        nr, ar, sr = prep(ref_lists, REF_IN, REF_OUT, TrackRefStruct)
        n_out, par, par_n = np.zeros(2, np.int32), np.zeros(2), np.zeros(2, np.int32)
        check(lib().icg_klt_track_frame(self._h, C.byref(params), nm, C.byref(sm), nr, C.byref(sr), _ptr(n_out), _ptr(par), _ptr(par_n)),
              "icg_klt_track_frame")

        def cut(arrs, names_out, n, k_out):
            out = {}
            for k in names_out:
                a = arrs[k][:n] if k in ("fwd_xy", "fwd_undis_xy", "keep") else arrs[k][:k_out]
                out[k] = a.reshape(-1) if _SPEC[k][1] == 1 else a
            return out
        return cut(am, MAP_OUT, nm, int(n_out[0])), cut(ar, REF_OUT, nr, int(n_out[1])), n_out, par, par_n

    def track_frames_dev(self, params, map_off, map_ptrs, ref_off, ref_ptrs, dev_n_out, dev_parallax, dev_parallax_n):
        """B streams in one asynchronous call (icg_klt_track_frames_dev).  params: sequence of TrackFrameStruct; map_off / ref_off: host sequences
        of B + 1; map_ptrs / ref_ptrs: dicts name -> device address (MAP_IN + MAP_OUT / REF_IN + REF_OUT; None or {} for a list with no points);
        dev_n_out / dev_parallax / dev_parallax_n: device addresses of 2 B int32 / float64 / int32."""
        B = len(params)
        par = (TrackFrameStruct * B)(*params)
        mo = np.ascontiguousarray(np.asarray(map_off, np.int32).reshape(-1))
        ro = np.ascontiguousarray(np.asarray(ref_off, np.int32).reshape(-1))
        if mo.size != B + 1 or ro.size != B + 1:
            raise ValueError("map_off and ref_off need len(params) + 1 entries")
        sm = TrackMapStruct(*[map_ptrs.get(k) for k in MAP_IN + MAP_OUT]) if map_ptrs else None
        sr = TrackRefStruct(*[ref_ptrs.get(k) for k in REF_IN + REF_OUT]) if ref_ptrs else None
        check(lib().icg_klt_track_frames_dev(self._h, B, par, _ptr(mo), C.byref(sm) if sm is not None else None, _ptr(ro),
                                             C.byref(sr) if sr is not None else None, vp(dev_n_out), vp(dev_parallax), vp(dev_parallax_n)),
              "icg_klt_track_frames_dev")

    # ------------------------------------------------------------------ Tracking::triangulation (tracking.cc:690-798)
    def triangulate(self, params: TriFrameStruct, keyframes, lists):
        """One stream from host arrays (icg_klt_triangulate, synchronous).  keyframes: iterable of (id, R, t, in_map); lists: dict with
        ref_out_xy, cur_xy (n, 2) float32, ref_frame_id_out (n,) int64, velocity_ref_out, velocity (n, 2) float64 (None or {} = empty).
        Returns (list_out, new, counts): list_out = the compacted ref_out_xy / ref_frame_id_out / cur_xy / velocity_ref_out / src cut to the
        kept count, new = the new map points (TRI_NEW) cut to the succeeded count, counts = int32[5] (TRI_COUNTS)."""
        kfs = list(keyframes)
        kf = tri_keyframes(kfs)
        lists = lists or {}
        n = len(lists["cur_xy"]) if "cur_xy" in lists else 0
        la = {}
        for k in TRI_LIST:
            dt, c = _SPEC[k]
            la[k] = np.ascontiguousarray(np.asarray(lists[k], dt).reshape(n, c)).copy() if (n and k != "src") else np.zeros((max(n, 1), c), dt)
        na = {k: np.zeros((max(n, 1), c), dt) for k, (dt, c) in _TRI_NEW_SPEC.items()}
        sl = TriListStruct(*[la[k].ctypes.data for k in TRI_LIST])
        sn = TriNewStruct(*[na[k].ctypes.data for k in TRI_NEW])
        counts = np.zeros(5, np.int32)
        check(lib().icg_klt_triangulate(self._h, C.byref(params), len(kfs), kf, n, C.byref(sl), C.byref(sn), _ptr(counts)), "icg_klt_triangulate")
        k_out, m_out = max(int(counts[0]), 0), max(int(counts[1]), 0) if counts[0] >= 0 else 0
        flat = lambda a, c: a.reshape(-1) if c == 1 else a  # noqa: E731
        lo = {k: flat(la[k][:k_out], _SPEC[k][1]) for k in TRI_LIST if k != "velocity"}
        no = {k: flat(na[k][:m_out], _TRI_NEW_SPEC[k][1]) for k in TRI_NEW}
        return lo, no, counts

    def triangulate_dev(self, params, kf_off, keyframes, ref_off, dev_n_in, n_in_stride, list_ptrs, new_ptrs, dev_counts):
        """B streams in one asynchronous call (icg_klt_triangulate_dev).  params: sequence of TriFrameStruct; kf_off: host sequence of B + 1;
        keyframes: iterable of (id, R, t, in_map) for all streams in kf_off order (or a prebuilt tri_keyframes array; params likewise may be a
        prebuilt TriFrameStruct array); ref_off: host sequence of B + 1; dev_n_in: device address of
        the live counts (dev_n_in[s * n_in_stride]) or 0 for the segment lengths; list_ptrs / new_ptrs: dicts name -> device address (TRI_LIST /
        TRI_NEW; None when no stream has points); dev_counts: device address of 5 B int32."""
        B = len(params)
        par = params if isinstance(params, C.Array) else (TriFrameStruct * B)(*params)
        ko = np.ascontiguousarray(np.asarray(kf_off, np.int32).reshape(-1))
        ro = np.ascontiguousarray(np.asarray(ref_off, np.int32).reshape(-1))
        if ko.size != B + 1 or ro.size != B + 1:
            raise ValueError("kf_off and ref_off need len(params) + 1 entries")
        kf = keyframes if isinstance(keyframes, C.Array) else tri_keyframes(list(keyframes))
        sl = TriListStruct(*[list_ptrs.get(k) for k in TRI_LIST]) if list_ptrs else None
        sn = TriNewStruct(*[new_ptrs.get(k) for k in TRI_NEW]) if new_ptrs else None
        check(lib().icg_klt_triangulate_dev(self._h, B, par, _ptr(ko), kf if ko[-1] else None, _ptr(ro), vp(dev_n_in) if dev_n_in else None,
                                            int(n_in_stride), C.byref(sl) if sl is not None else None, C.byref(sn) if sn is not None else None,
                                            vp(dev_counts)), "icg_klt_triangulate_dev")

    def sync(self):
        check(lib().icg_klt_sync(self._h), "icg_klt_sync")
