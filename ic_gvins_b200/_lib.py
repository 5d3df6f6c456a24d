"""ctypes loader for libicgvins_b200.so (the C ABI declared in include/icgvins_b200.h).

There is no CPU fallback: if the library is missing this raises, and every create() call fails without an H100 (sm_90).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# ICG_LIB_VARIANT=prof loads libicgvins_b200_prof.so: the same sources built with -DICG_BA_PHASE_CLOCKS (`python -m ic_gvins_b200.build --prof`),
# an instrumented build for the profiling scripts only -- never the measured or shipped library
LIB_PATH = os.path.join(_HERE, "libicgvins_b200_prof.so" if os.environ.get("ICG_LIB_VARIANT") == "prof" else "libicgvins_b200.so")

u8p = C.POINTER(C.c_uint8)
f32p = C.POINTER(C.c_float)
f64p = C.POINTER(C.c_double)
i32p = C.POINTER(C.c_int32)
vp = C.c_void_p

_lib = None


class IcgError(RuntimeError):
    pass


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise IcgError(f"{LIB_PATH} not built: run `python -m ic_gvins_b200.build` (there is no CPU fallback)")
        _lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        _declare(_lib)
        _declare_r2(_lib)
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().icg_last_error().decode("utf-8", "replace")
        raise IcgError(f"{what} failed with code {rc}: {msg}")


def _declare(L: C.CDLL) -> None:
    L.icg_last_error.restype = C.c_char_p
    L.icg_version.restype = C.c_int
    L.icg_launch_count.restype = C.c_uint64
    L.icg_launch_count_reset.restype = None
    # ---- KLT
    L.icg_klt_create.argtypes = [C.POINTER(vp), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    L.icg_klt_destroy.argtypes = [vp]
    L.icg_klt_destroy.restype = None
    L.icg_klt_calc_optical_flow_pyr_lk.argtypes = [vp, vp, vp, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int,
                                                   C.c_double, C.c_int]
    L.icg_klt_track_fb.argtypes = [vp, vp, vp, C.c_int, vp, vp, vp, vp, C.c_int]
    L.icg_klt_upload.argtypes = [vp, C.c_int, vp, C.c_int]
    L.icg_klt_upload_level0.argtypes = [vp, C.c_int, vp, C.c_int]
    L.icg_klt_upload_batch.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int]
    L.icg_klt_slot_level0.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(C.c_int)]
    L.icg_klt_slot_level.argtypes = [vp, C.c_int, C.c_int, C.POINTER(vp), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.icg_klt_build_pyramids.argtypes = [vp, C.c_int, C.c_int]
    L.icg_klt_track_batch_dev.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_int]
    L.icg_klt_sync.argtypes = [vp]
    L.icg_klt_download_level.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int]
    # ---- detection
    L.icg_detect_create.argtypes = [C.POINTER(vp), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    L.icg_detect_destroy.argtypes = [vp]
    L.icg_detect_destroy.restype = None
    L.icg_detect_blocks.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, vp, C.c_double, C.c_double, C.c_int, vp, vp]
    L.icg_detect_blocks_dev.argtypes = [vp, C.c_int, vp, C.c_int, C.c_size_t, vp, C.c_int, vp, vp, C.c_double, C.c_double, C.c_int, vp, vp]
    L.icg_corner_subpix.argtypes = [vp, vp, C.c_int, vp, C.c_int]
    L.icg_detect_features.argtypes = [vp, vp, C.c_int, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]
    L.icg_detect_features_dev.argtypes = [vp, C.c_int, vp, C.c_int, C.c_size_t, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int, vp, vp]
    L.icg_detect_mask_dev.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(C.c_int)]
    # ---- camera model (host functions)
    L.icg_camera_undistort_points.argtypes = [vp, vp, C.c_int]
    L.icg_camera_distort_points.argtypes = [vp, vp, C.c_int]
    L.icg_camera_distort_camera_points.argtypes = [vp, vp, vp, C.c_int]
    L.icg_camera_pixel2cam.argtypes = [vp, vp, vp, C.c_int]
    L.icg_camera_world2pixel.argtypes = [vp, vp, vp, vp, vp, C.c_int]
    L.icg_tracking_histogram.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp]
    L.icg_triangulate_points.argtypes = [vp, vp, vp, vp, C.c_int, vp]
    L.icg_find_fundamental_mat_ransac.argtypes = [vp, vp, C.c_int, C.c_double, C.c_double, C.c_int, vp, vp]
    # ---- CLAHE
    L.icg_clahe_create.argtypes = [C.POINTER(vp), C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, vp]
    L.icg_clahe_destroy.argtypes = [vp]
    L.icg_clahe_destroy.restype = None
    L.icg_clahe_apply.argtypes = [vp, vp, C.c_int, vp, C.c_int]
    L.icg_clahe_apply_dev.argtypes = [vp, vp, C.c_int, vp, C.c_int]
    L.icg_clahe_sync.argtypes = [vp]
    # ---- BA
    L.icg_imu_preintegrate.argtypes = [vp, vp, vp, vp, vp, C.c_int, vp, vp]
    L.icg_ba_create.argtypes = [C.POINTER(vp), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    L.icg_ba_destroy.argtypes = [vp]
    L.icg_ba_destroy.restype = None
    L.icg_ba_solve.argtypes = [vp, C.c_int, vp, C.c_int, vp]
    L.icg_ba_upload.argtypes = [vp, C.c_int, vp]
    L.icg_ba_run.argtypes = [vp, C.c_int, C.c_int]
    L.icg_ba_download.argtypes = [vp, C.c_int, vp, vp]
    L.icg_ba_sync.argtypes = [vp]
    L.icg_ba_shard_export.argtypes = [vp, C.c_int, C.c_int, vp]
    L.icg_ba_shard_connect.argtypes = [vp, vp]
    L.icg_ba_shard_error.argtypes = [vp]
    L.icg_ba_shard_leave.argtypes = [vp]
    L.icg_ba_gvins_optimization.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp]
    L.icg_ba_run_gvins.argtypes = [vp, C.c_int, C.c_int]
    L.icg_ba_gvins_optimization_begin.argtypes = [vp, C.c_int, vp, C.c_int]
    L.icg_ba_gvins_optimization_end.argtypes = [vp, C.c_int, vp, vp, vp]
    L.icg_ba_residual_costs.argtypes = [vp, vp, vp, vp]
    L.icg_ba_reproj_evaluate.argtypes = [vp, vp, vp, vp, vp, vp, vp, C.c_double, vp, vp]
    L.icg_ba_reproj_evaluate_frames.argtypes = [vp, vp, vp, vp, vp, vp, vp, C.c_double, vp, vp]
    L.icg_ba_imu_evaluate.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    L.icg_ba_marginalize.argtypes = [vp, C.c_int, vp, vp, vp]
    L.icg_ba_marginalize_resident.argtypes = [vp, C.c_int, vp, vp, vp]
    L.icg_ba_gnss_evaluate.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.icg_ba_pose_prior_evaluate.argtypes = [vp, vp, vp, vp, vp, vp]
    L.icg_ba_mix_prior_evaluate.argtypes = [vp, vp, vp, vp, vp, vp]
    L.icg_ba_imu_error_evaluate.argtypes = [vp, vp, vp, vp]
    L.icg_ba_marg_factor_evaluate.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp]


def _declare_r2(L: C.CDLL) -> None:
    L.icg_clahe_apply_batch_dev.argtypes = [vp, C.c_int, vp, C.c_int, C.c_size_t, vp, C.c_int, C.c_size_t, vp]
    L.icg_geom_create.argtypes = [C.POINTER(vp), C.c_int, vp]
    L.icg_geom_destroy.argtypes = [vp]
    L.icg_geom_destroy.restype = None
    L.icg_geom_undistort_points.argtypes = [vp, vp, vp, C.c_int]
    L.icg_geom_distort_points.argtypes = [vp, vp, vp, C.c_int]
    L.icg_geom_find_fundamental_mat_ransac.argtypes = [vp, vp, vp, C.c_int, C.c_double, C.c_double, C.c_int, vp, vp]
    L.icg_geom_triangulate_points.argtypes = [vp, vp, vp, vp, vp, C.c_int, vp]
    L.icg_geom_imu_preintegrate_batch.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.icg_geom_find_fundamental_mat_ransac_batch.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp]
    L.icg_klt_track_frames_dev.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.icg_klt_track_frame.argtypes = [vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp]
    L.icg_klt_triangulate_dev.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp]
    L.icg_klt_triangulate.argtypes = [vp, vp, C.c_int, vp, C.c_int, vp, vp, vp]
    L.icg_ba_update_and_cull_resident.argtypes = [vp, C.c_int, vp, vp, C.c_double, vp]
    L.icg_ba_marginalize_resident_culled.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp]
    L.icg_ba_reintegrate_resident.argtypes = [vp, C.c_int, vp, vp, vp, vp]
    L.icg_ba_slide_resident.argtypes = [vp, C.c_int, vp, vp]
    L.icg_ba_slide_integrate_resident.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp]
    L.icg_ba_slide_vision_resident.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp]
    L.icg_ba_shard_reintegrate_resident.argtypes = [vp, C.c_int, vp, vp, vp, vp]
    L.icg_ba_shard_slide_resident.argtypes = [vp, C.c_int, vp, vp]
    L.icg_ba_shard_slide_integrate_resident.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp]
    L.icg_ba_shard_slide_vision_resident.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp]
    # ---- INS windows
    L.icg_ins_create.argtypes = [C.POINTER(vp), C.c_int, C.c_int, C.c_int, vp]
    L.icg_ins_destroy.argtypes = [vp]
    L.icg_ins_destroy.restype = None
    L.icg_ins_push.argtypes = [vp, C.c_int, vp, vp, vp]
    L.icg_ins_redo.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp]
    L.icg_ins_camera_pose.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp]
    L.icg_ins_window.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp]
    L.icg_ins_sync.argtypes = [vp]
    L.icg_ins_gins_initialize.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, C.c_int, vp]
    # ---- the window solver's IMU sample store, filled from the INS windows
    L.icg_ba_imu_samples_from_ins.argtypes = [vp, vp, C.c_int, vp]
    L.icg_ba_slide_ins_resident.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, vp, vp]
    L.icg_ba_reintegrate_stored_resident.argtypes = [vp, C.c_int, vp, vp, vp, vp]
    L.icg_ba_imu_samples.argtypes = [vp, C.c_int, C.c_int, vp, vp]


class InsConfig(C.Structure):
    """ctypes image of `icg_ins_config`."""
    _fields_ = [("with_earth", C.c_int32), ("gravity", C.c_double * 3), ("iewn", C.c_double * 3)]


class GinsInit(C.Structure):
    """ctypes image of `icg_gins_init`."""
    _fields_ = [("gnss_time", C.c_double), ("gnss_blh", C.c_double * 3), ("gnss_std", C.c_double * 3),
                ("last_time", C.c_double), ("last_blh", C.c_double * 3), ("last_std", C.c_double * 3),
                ("last_yaw_valid", C.c_int32), ("last_yaw", C.c_double), ("origin_blh", C.c_double * 3), ("gravity", C.c_double),
                ("antlever", C.c_double * 3), ("imudatarate", C.c_double)]


class GinsInitOut(C.Structure):
    """ctypes image of `icg_gins_init_out`."""
    _fields_ = [("status", C.c_int32), ("has_zero_velocity", C.c_int32), ("bg", C.c_double * 3), ("initatt", C.c_double * 3),
                ("state17", C.c_double * 34), ("pose_prior", C.c_double * 7), ("pose_prior_std", C.c_double * 6), ("mix_prior", C.c_double * 9),
                ("mix_prior_std", C.c_double * 9), ("imu_blob", C.c_double * 480), ("n_series", C.c_int32)]


class SlideWindow(C.Structure):
    """ctypes image of `icg_ba_slide_window`."""
    _fields_ = [("node_src", i32p), ("lm_src", i32p), ("f_src", i32p), ("imu_src", i32p), ("gnss_src", i32p), ("prior_from_marg", C.c_int32)]


SLIDE_CHAIN, SLIDE_ROW = -2, -3  # ICG_SLIDE_CHAIN, ICG_SLIDE_ROW


class SlideIntegrate(C.Structure):
    """ctypes image of `icg_ba_slide_integrate`."""
    _fields_ = [("imu_from", i32p), ("state16", f64p), ("gravity3", f64p), ("normal", u8p), ("imu", f64p), ("imu_off", i32p),
                ("node_from_imu", u8p), ("gnss_node", i32p), ("gnss_dt", f64p),
                ("status", C.POINTER(C.c_int8)), ("blob_out", f64p), ("end_state10", f64p)]


class InsCut(C.Structure):
    """ctypes image of `icg_ba_ins_cut`."""
    _fields_ = [("stream", C.c_int32), ("node_time", f64p)]


class SlideIns(C.Structure):
    """ctypes image of `icg_ba_slide_ins`."""
    _fields_ = [("integ", SlideIntegrate), ("stream", C.c_int32), ("node_time", f64p), ("merge_src", i32p), ("n_rows", i32p)]


class SlideVision(C.Structure):
    """ctypes image of `icg_ba_slide_vision` (device pointers as void *)."""
    _fields_ = [("num_marg", C.c_int32), ("node_in_map", u8p), ("obs_factor", i32p), ("cam", C.c_double * 10), ("node_td", f64p),
                ("cur_node", C.c_int32), ("n_frames", C.c_int32), ("frame_id", C.POINTER(C.c_int64)), ("frame_node", i32p),
                ("n_obs", C.c_int32), ("n_in", C.c_int32), ("dev_n", vp), ("obs_src", vp), ("obs_lm", vp), ("obs_node", vp), ("obs_undis_xy", vp),
                ("obs_vel", vp), ("n_new", C.c_int32), ("dev_new_n", vp), ("new_depth", vp), ("new_vel_ref", vp), ("new_vel_cur", vp),
                ("new_ref_undis_xy", vp), ("new_cur_undis_xy", vp), ("new_ref_frame_id", vp),
                ("L", C.c_int32), ("F", C.c_int32), ("nan_dropped", C.c_int32),
                ("lm_src", i32p), ("f_src", i32p), ("f_lm", i32p), ("f_ref", i32p), ("f_obs", i32p), ("lm_origin", i32p), ("nan_flags", u8p),
                ("invdepth", f64p), ("f_const", f64p)]


# every symbol include/icgvins_b200.h declares (checked by tests/test_abi.py against the header text)
EXPORTS = [
    "icg_last_error", "icg_version", "icg_launch_count", "icg_launch_count_reset",
    "icg_klt_create", "icg_klt_destroy", "icg_klt_calc_optical_flow_pyr_lk", "icg_klt_track_fb", "icg_klt_upload",
    "icg_klt_upload_level0", "icg_klt_upload_batch", "icg_klt_slot_level0", "icg_klt_slot_level", "icg_klt_build_pyramids",
    "icg_klt_track_batch_dev", "icg_klt_sync", "icg_klt_download_level",
    "icg_detect_create", "icg_detect_destroy", "icg_detect_blocks", "icg_detect_blocks_dev", "icg_corner_subpix",
    "icg_detect_features", "icg_detect_features_dev", "icg_detect_mask_dev",
    "icg_camera_undistort_points", "icg_camera_distort_points", "icg_camera_distort_camera_points", "icg_camera_pixel2cam", "icg_camera_world2pixel", "icg_tracking_histogram", "icg_find_fundamental_mat_ransac", "icg_triangulate_points",
    "icg_clahe_create", "icg_clahe_destroy", "icg_clahe_apply", "icg_clahe_apply_dev", "icg_clahe_apply_batch_dev", "icg_geom_create", "icg_geom_destroy", "icg_geom_undistort_points", "icg_geom_distort_points", "icg_geom_find_fundamental_mat_ransac", "icg_geom_triangulate_points", "icg_geom_imu_preintegrate_batch", "icg_clahe_sync",
    "icg_geom_find_fundamental_mat_ransac_batch", "icg_klt_track_frames_dev", "icg_klt_track_frame",
    "icg_klt_triangulate_dev", "icg_klt_triangulate",
    "icg_imu_preintegrate", "icg_ba_create", "icg_ba_destroy", "icg_ba_solve", "icg_ba_upload", "icg_ba_run", "icg_ba_download",
    "icg_ba_sync", "icg_ba_shard_export", "icg_ba_shard_connect", "icg_ba_shard_error", "icg_ba_shard_leave", "icg_ba_gvins_optimization", "icg_ba_run_gvins", "icg_ba_gvins_optimization_begin", "icg_ba_gvins_optimization_end", "icg_ba_residual_costs", "icg_ba_reproj_evaluate", "icg_ba_reproj_evaluate_frames", "icg_ba_imu_evaluate", "icg_ba_marginalize", "icg_ba_marginalize_resident", "icg_ba_update_and_cull_resident", "icg_ba_marginalize_resident_culled", "icg_ba_reintegrate_resident", "icg_ba_slide_resident", "icg_ba_slide_integrate_resident", "icg_ba_slide_vision_resident", "icg_ba_shard_reintegrate_resident", "icg_ba_shard_slide_resident", "icg_ba_shard_slide_integrate_resident", "icg_ba_shard_slide_vision_resident", "icg_ba_gnss_evaluate", "icg_ba_pose_prior_evaluate", "icg_ba_mix_prior_evaluate", "icg_ba_imu_error_evaluate", "icg_ba_marg_factor_evaluate",
    "icg_ins_create", "icg_ins_destroy", "icg_ins_push", "icg_ins_redo", "icg_ins_gins_initialize", "icg_ins_camera_pose", "icg_ins_window", "icg_ins_sync",
    "icg_ba_imu_samples_from_ins", "icg_ba_slide_ins_resident", "icg_ba_reintegrate_stored_resident", "icg_ba_imu_samples",
]
