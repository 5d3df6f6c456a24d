"""Device versions of the point-wise front-end geometry and of the IMU propagation (SURVEY.md 8f ranks 2-4), batched: same argument
conventions as the host mirrors in camera.py / ba.py, arithmetic in CUDA kernels of libicgvins_b200.so (csrc/geom.cu)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import check, lib, vp
from .camera import CameraStruct


class Geometry:
    def __init__(self, device: int = 0, stream=None):
        self._h = vp()
        check(lib().icg_geom_create(C.byref(self._h), device, vp(stream) if stream else None), "icg_geom_create")

    def close(self):
        if getattr(self, "_h", None):
            lib().icg_geom_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _cam(intrinsic, distortion) -> CameraStruct:
        i, d = list(map(float, intrinsic)), list(map(float, distortion))
        return CameraStruct(i[0], i[1], i[2], i[3], i[4] if len(i) == 5 else 0.0, d[0], d[1], d[2], d[3], d[4] if len(d) == 5 else 0.0)

    def undistortPoints(self, intrinsic, distortion, pts):
        """Camera::undistortPoints (camera.cc:72-74) on any number of points"""
        c = self._cam(intrinsic, distortion)
        p = np.ascontiguousarray(np.array(pts, np.float32).reshape(-1, 2))
        check(lib().icg_geom_undistort_points(self._h, C.byref(c), vp(p.ctypes.data), p.shape[0]), "icg_geom_undistort_points")
        return p

    def distortPoints(self, intrinsic, distortion, pts):
        c = self._cam(intrinsic, distortion)
        p = np.ascontiguousarray(np.array(pts, np.float32).reshape(-1, 2))
        check(lib().icg_geom_distort_points(self._h, C.byref(c), vp(p.ctypes.data), p.shape[0]), "icg_geom_distort_points")
        return p

    def findFundamentalMat(self, points1, points2, ransacReprojThreshold=3.0, confidence=0.99, maxIters=1000):
        """cv2.findFundamentalMat(p1, p2, cv2.FM_RANSAC, thr, conf) -> (F, status): hypotheses solved and scored on the device"""
        p1 = np.ascontiguousarray(np.array(points1, np.float32).reshape(-1, 2))
        p2 = np.ascontiguousarray(np.array(points2, np.float32).reshape(-1, 2))
        st = np.zeros(p1.shape[0], np.uint8)
        F = np.zeros(9)
        check(lib().icg_geom_find_fundamental_mat_ransac(self._h, vp(p1.ctypes.data), vp(p2.ctypes.data), p1.shape[0], float(ransacReprojThreshold),
                                                         float(confidence), int(maxIters), vp(st.ctypes.data), vp(F.ctypes.data)),
              "icg_geom_find_fundamental_mat_ransac")
        return F.reshape(3, 3), st

    def findFundamentalMat_batch_dev(self, set_off, dev_pts1, dev_pts2, dev_mask, dev_n_inliers, thresholds=None, confidences=None, maxIters=1000,
                                     dev_F=0, dev_stats=0):
        """cv2.findFundamentalMat(FM_RANSAC) on S device-resident point sets in one asynchronous call (icg_geom_find_fundamental_mat_ransac_batch):
        set s = pairs set_off[s] .. set_off[s + 1] (host sequence of S + 1) of the float2 device arrays at dev_pts1 / dev_pts2; thresholds /
        confidences: host sequences of S (None = 3 / 0.99).  Writes one u8 per pair at dev_mask, S int32 inlier counts at dev_n_inliers, and
        optionally 9 doubles per set at dev_F and 3 int64 per set at dev_stats (subsets drawn, draw cycles, total cycles)."""
        off = np.ascontiguousarray(np.asarray(set_off, np.int32).reshape(-1))
        S = off.size - 1
        th = np.ascontiguousarray(np.broadcast_to(np.asarray(thresholds, np.float64), (S,))) if thresholds is not None else None
        cf = np.ascontiguousarray(np.broadcast_to(np.asarray(confidences, np.float64), (S,))) if confidences is not None else None
        check(lib().icg_geom_find_fundamental_mat_ransac_batch(self._h, S, vp(off.ctypes.data), vp(dev_pts1) if dev_pts1 else None,
                                                               vp(dev_pts2) if dev_pts2 else None, vp(th.ctypes.data) if th is not None else None,
                                                               vp(cf.ctypes.data) if cf is not None else None, int(maxIters), vp(dev_mask),
                                                               vp(dev_n_inliers), vp(dev_F) if dev_F else None, vp(dev_stats) if dev_stats else None),
              "icg_geom_find_fundamental_mat_ransac_batch")

    def triangulatePoints(self, Tcw0, Tcw1, pc0, pc1):
        a = np.ascontiguousarray(np.array(Tcw0, np.float64).reshape(-1, 12))
        b = np.ascontiguousarray(np.array(Tcw1, np.float64).reshape(12))
        p0 = np.ascontiguousarray(np.array(pc0, np.float64).reshape(a.shape[0], -1)[:, :2])
        p1 = np.ascontiguousarray(np.array(pc1, np.float64).reshape(a.shape[0], -1)[:, :2])
        out = np.zeros((a.shape[0], 3))
        check(lib().icg_geom_triangulate_points(self._h, vp(a.ctypes.data), vp(b.ctypes.data), vp(p0.ctypes.data), vp(p1.ctypes.data), a.shape[0],
                                                vp(out.ctypes.data)), "icg_geom_triangulate_points")
        return out

    def imu_preintegrate_batch(self, states16, iewn, gravity, noise5, imu_list):
        """Preintegration of many intervals in one launch (doReintegration over a window, IG/ic_gvins.cc:1680-1695): states16 (n, 16), imu_list = n
        arrays of (m_k, 7) rows (dt, dtheta, dvel).  iewn None: PreintegrationNormal.  Returns (blobs (n, 480), end_states (n, 10))."""
        st = np.ascontiguousarray(np.array(states16, np.float64).reshape(-1, 16))
        n = st.shape[0]
        off = np.zeros(n + 1, np.int32)
        off[1:] = np.cumsum([len(x) for x in imu_list])
        imu = np.ascontiguousarray(np.concatenate([np.asarray(x, np.float64).reshape(-1, 7) for x in imu_list], axis=0))
        g, nz = np.ascontiguousarray(gravity, np.float64), np.ascontiguousarray(noise5, np.float64)
        iw = np.ascontiguousarray(iewn, np.float64) if iewn is not None else None
        blobs, ends = np.zeros((n, 480)), np.zeros((n, 10))
        check(lib().icg_geom_imu_preintegrate_batch(self._h, n, vp(st.ctypes.data), vp(iw.ctypes.data) if iw is not None else None, vp(g.ctypes.data),
                                                    vp(nz.ctypes.data), vp(imu.ctypes.data), vp(off.ctypes.data), vp(blobs.ctypes.data), vp(ends.ctypes.data)),
              "icg_geom_imu_preintegrate_batch")
        return blobs, ends
