"""ctypes loader for libicgvins_b200.so (the C ABI declared in include/icgvins_b200.h).

There is no CPU fallback: if the library is missing this raises, and every create() call fails without an H100 (sm_90).
"""
from __future__ import annotations

import ctypes as C
import os
from ctypes import c_double, c_int, c_size_t

_HERE = os.path.dirname(os.path.abspath(__file__))
# ICG_LIB_VARIANT=prof loads libicgvins_b200_prof.so: the same sources built with -DICG_BA_PHASE_CLOCKS (`python -m ic_gvins_b200.build --prof`),
# an instrumented build for the profiling scripts only -- never the measured or shipped library
LIB_PATH = os.path.join(_HERE, "libicgvins_b200_prof.so" if os.environ.get("ICG_LIB_VARIANT") == "prof" else "libicgvins_b200.so")

u8p = C.POINTER(C.c_uint8)
i8p = C.POINTER(C.c_int8)
i32p = C.POINTER(C.c_int32)
i64p = C.POINTER(C.c_int64)
f32p = C.POINTER(C.c_float)
f64p = C.POINTER(C.c_double)
vp = C.c_void_p
vpp = C.POINTER(vp)

# every function include/icgvins_b200.h declares: name -> (argtypes, restype).  ctypes converts Python ints and floats by these argtypes.
ABI = {
    # ---- library
    "icg_last_error": ([], C.c_char_p),
    "icg_version": ([], c_int),
    "icg_launch_count": ([], C.c_uint64),
    "icg_launch_count_reset": ([], None),
    # ---- KLT and the per-stream tracking / triangulation on its handle
    "icg_klt_create": ([vpp, c_int, c_int, c_int, c_int, c_int, vp], c_int),
    "icg_klt_destroy": ([vp], None),
    "icg_klt_calc_optical_flow_pyr_lk": ([vp, vp, vp, c_int, vp, vp, vp, vp, c_int, c_int, c_int, c_int, c_double, c_int], c_int),
    "icg_klt_track_fb": ([vp, vp, vp, c_int, vp, vp, vp, vp, c_int], c_int),
    "icg_klt_upload": ([vp, c_int, vp, c_int], c_int),
    "icg_klt_upload_level0": ([vp, c_int, vp, c_int], c_int),
    "icg_klt_upload_batch": ([vp, c_int, c_int, vp, c_int], c_int),
    "icg_klt_download_level": ([vp, c_int, c_int, vp, c_int], c_int),
    "icg_klt_slot_level0": ([vp, c_int, vpp, i32p], c_int),
    "icg_klt_slot_level": ([vp, c_int, c_int, vpp, i32p, i32p, i32p], c_int),
    "icg_klt_build_pyramids": ([vp, c_int, c_int], c_int),
    "icg_klt_track_batch_dev": ([vp, c_int, vp, vp, vp, vp, vp, vp, c_int], c_int),
    "icg_klt_sync": ([vp], c_int),
    "icg_klt_track_frames_dev": ([vp, c_int, vp, vp, vp, vp, vp, vp, vp, vp], c_int),
    "icg_klt_track_frame": ([vp, vp, c_int, vp, c_int, vp, vp, vp, vp], c_int),
    "icg_klt_triangulate_dev": ([vp, c_int, vp, vp, vp, vp, vp, c_int, vp, vp, vp], c_int),
    "icg_klt_triangulate": ([vp, vp, c_int, vp, c_int, vp, vp, vp], c_int),
    # ---- detection
    "icg_detect_create": ([vpp, c_int, c_int, c_int, c_int, c_int, c_int, vp], c_int),
    "icg_detect_destroy": ([vp], None),
    "icg_detect_blocks": ([vp, vp, vp, c_int, c_int, vp, vp, c_double, c_double, c_int, vp, vp], c_int),
    "icg_detect_blocks_dev": ([vp, c_int, vp, c_int, c_size_t, vp, c_int, vp, vp, c_double, c_double, c_int, vp, vp], c_int),
    "icg_detect_features": ([vp, vp, c_int, vp, c_int, vp, c_int, c_int, c_int, c_int, vp, vp], c_int),
    "icg_detect_features_dev": ([vp, c_int, vp, c_int, c_size_t, vp, vp, vp, vp, vp, vp, vp, vp, c_int, vp, vp], c_int),
    "icg_detect_mask_dev": ([vp, c_int, vpp, i32p], c_int),
    "icg_corner_subpix": ([vp, vp, c_int, vp, c_int], c_int),
    # ---- camera model and geometry (host functions)
    "icg_camera_undistort_points": ([vp, vp, c_int], c_int),
    "icg_camera_distort_points": ([vp, vp, c_int], c_int),
    "icg_camera_distort_camera_points": ([vp, vp, vp, c_int], c_int),
    "icg_camera_pixel2cam": ([vp, vp, vp, c_int], c_int),
    "icg_camera_world2pixel": ([vp, vp, vp, vp, vp, c_int], c_int),
    "icg_find_fundamental_mat_ransac": ([vp, vp, c_int, c_double, c_double, c_int, vp, vp], c_int),
    "icg_triangulate_points": ([vp, vp, vp, vp, c_int, vp], c_int),
    "icg_tracking_histogram": ([vp, c_int, c_int, c_int, vp], c_int),
    # ---- geometry on the device
    "icg_geom_create": ([vpp, c_int, vp], c_int),
    "icg_geom_destroy": ([vp], None),
    "icg_geom_undistort_points": ([vp, vp, vp, c_int], c_int),
    "icg_geom_distort_points": ([vp, vp, vp, c_int], c_int),
    "icg_geom_find_fundamental_mat_ransac": ([vp, vp, vp, c_int, c_double, c_double, c_int, vp, vp], c_int),
    "icg_geom_triangulate_points": ([vp, vp, vp, vp, vp, c_int, vp], c_int),
    "icg_geom_imu_preintegrate_batch": ([vp, c_int, vp, vp, vp, vp, vp, vp, vp, vp], c_int),
    "icg_geom_find_fundamental_mat_ransac_batch": ([vp, c_int, vp, vp, vp, vp, vp, c_int, vp, vp, vp, vp], c_int),
    # ---- CLAHE
    "icg_clahe_create": ([vpp, c_int, c_int, c_int, c_int, c_double, c_int, vp], c_int),
    "icg_clahe_destroy": ([vp], None),
    "icg_clahe_apply": ([vp, vp, c_int, vp, c_int], c_int),
    "icg_clahe_apply_dev": ([vp, vp, c_int, vp, c_int], c_int),
    "icg_clahe_apply_batch_dev": ([vp, c_int, vp, c_int, c_size_t, vp, c_int, c_size_t, vp], c_int),
    "icg_clahe_sync": ([vp], c_int),
    # ---- window solver: solve, marginalization, read-outs
    "icg_imu_preintegrate": ([vp, vp, vp, vp, vp, c_int, vp, vp], c_int),
    "icg_ba_create": ([vpp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, vp], c_int),
    "icg_ba_destroy": ([vp], None),
    "icg_ba_solve": ([vp, c_int, vp, c_int, vp], c_int),
    "icg_ba_upload": ([vp, c_int, vp], c_int),
    "icg_ba_run": ([vp, c_int, c_int], c_int),
    "icg_ba_download": ([vp, c_int, vp, vp], c_int),
    "icg_ba_sync": ([vp], c_int),
    "icg_ba_gvins_optimization": ([vp, c_int, vp, c_int, vp, vp], c_int),
    "icg_ba_run_gvins": ([vp, c_int, c_int], c_int),
    "icg_ba_gvins_optimization_begin": ([vp, c_int, vp, c_int], c_int),
    "icg_ba_gvins_optimization_end": ([vp, c_int, vp, vp, vp], c_int),
    "icg_ba_residual_costs": ([vp, vp, vp, vp], c_int),
    "icg_ba_marginalize": ([vp, c_int, vp, vp, vp], c_int),
    "icg_ba_marginalize_resident": ([vp, c_int, vp, vp, vp], c_int),
    "icg_ba_peek_linearization": ([vp, c_int, vp], c_int),
    "icg_ba_peek_structure": ([vp, c_int, vp], c_int),
    # ---- window solver: landmark-shard group
    "icg_ba_shard_export": ([vp, c_int, c_int, vp], c_int),
    "icg_ba_shard_connect": ([vp, vp], c_int),
    "icg_ba_shard_error": ([vp], c_int),
    "icg_ba_shard_leave": ([vp], c_int),
    # ---- window solver: the resident keyframe cycle (culling, reintegration, slides)
    "icg_ba_update_and_cull_resident": ([vp, c_int, vp, vp, c_double, vp], c_int),
    "icg_ba_update_and_cull_built": ([vp, c_int, vp, vp, c_double, vp, vp], c_int),
    "icg_ba_shard_update_and_cull_built": ([vp, c_int, vp, vp, c_double, vp, vp], c_int),
    "icg_ba_marginalize_resident_culled": ([vp, c_int, vp, vp, vp, vp, vp], c_int),
    "icg_ba_marginalize_built": ([vp, c_int, vp, vp, vp, vp], c_int),
    "icg_ba_reintegrate_resident": ([vp, c_int, vp, vp, vp, vp], c_int),
    "icg_ba_shard_reintegrate_resident": ([vp, c_int, vp, vp, vp, vp], c_int),
    "icg_ba_slide_resident": ([vp, c_int, vp, vp], c_int),
    "icg_ba_shard_slide_resident": ([vp, c_int, vp, vp], c_int),
    "icg_ba_slide_integrate_resident": ([vp, c_int, vp, vp, vp, vp, vp], c_int),
    "icg_ba_shard_slide_integrate_resident": ([vp, c_int, vp, vp, vp, vp, vp], c_int),
    "icg_ba_slide_vision_resident": ([vp, c_int, vp, vp, vp, vp, vp, vp], c_int),
    "icg_ba_shard_slide_vision_resident": ([vp, c_int, vp, vp, vp, vp, vp, vp], c_int),
    # ---- window solver: the IMU sample store, filled from the INS windows
    "icg_ba_imu_samples_from_ins": ([vp, vp, c_int, vp], c_int),
    "icg_ba_slide_ins_resident": ([vp, vp, c_int, vp, vp, vp, vp, vp, vp], c_int),
    "icg_ba_reintegrate_stored_resident": ([vp, c_int, vp, vp, vp, vp], c_int),
    "icg_ba_imu_samples": ([vp, c_int, c_int, vp, vp], c_int),
    # ---- window solver: single-factor Evaluate
    "icg_ba_reproj_evaluate": ([vp, vp, vp, vp, vp, vp, vp, c_double, vp, vp], c_int),
    "icg_ba_reproj_evaluate_frames": ([vp, vp, vp, vp, vp, vp, vp, c_double, vp, vp], c_int),
    "icg_ba_imu_evaluate": ([vp, vp, vp, vp, vp, vp, vp, vp], c_int),
    "icg_ba_gnss_evaluate": ([vp, vp, vp, vp, vp, vp, vp], c_int),
    "icg_ba_pose_prior_evaluate": ([vp, vp, vp, vp, vp, vp], c_int),
    "icg_ba_mix_prior_evaluate": ([vp, vp, vp, vp, vp, vp], c_int),
    "icg_ba_imu_error_evaluate": ([vp, vp, vp, vp], c_int),
    "icg_ba_marg_factor_evaluate": ([vp, c_int, c_int, vp, vp, vp, vp, vp, vp, vp], c_int),
    # ---- INS windows
    "icg_ins_create": ([vpp, c_int, c_int, c_int, vp], c_int),
    "icg_ins_destroy": ([vp], None),
    "icg_ins_push": ([vp, c_int, vp, vp, vp], c_int),
    "icg_ins_redo": ([vp, c_int, vp, vp, vp, c_int, vp], c_int),
    "icg_ins_gins_initialize": ([vp, c_int, vp, vp, vp, vp, vp, c_int, vp], c_int),
    "icg_ins_camera_pose": ([vp, c_int, vp, vp, vp, vp, vp], c_int),
    "icg_ins_window": ([vp, c_int, c_int, vp, vp, vp], c_int),
    "icg_ins_sync": ([vp], c_int),
}
EXPORTS = list(ABI)

_lib = None


class IcgError(RuntimeError):
    """A failed library call.  Raised by check(): `code` is the call's return code, `results` (where the call has any) what it wrote
    before it failed."""


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise IcgError(f"{LIB_PATH} not built: run `python -m ic_gvins_b200.build` (there is no CPU fallback)")
        L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        for name, (argtypes, restype) in ABI.items():
            fn = getattr(L, name)
            fn.argtypes, fn.restype = argtypes, restype
        _lib = L
    return _lib


def check(rc: int, what: str = "", results=None) -> None:
    if rc != 0:
        err = IcgError(f"{what} failed with code {rc}: {lib().icg_last_error().decode('utf-8', 'replace')}")
        err.code = rc
        if results is not None:
            err.results = results
        raise err


# ---- struct images
class BaProblem(C.Structure):
    """ctypes image of `icg_ba_problem`."""
    _fields_ = [
        ("K", C.c_int32), ("L", C.c_int32), ("F", C.c_int32),
        ("pose", f64p), ("mix", f64p), ("ext", f64p), ("invdepth", f64p),
        ("ext_const", C.c_int32), ("td_const", C.c_int32),
        ("f_lm", i32p), ("f_ref", i32p), ("f_obs", i32p), ("f_const", f64p), ("f_active", u8p),
        ("reproj_std", C.c_double), ("reproj_huber", C.c_int32),
        ("n_imu", C.c_int32), ("imu_blob", f64p), ("has_imu_error", C.c_int32),
        ("has_pose_prior", C.c_int32), ("pose_prior", f64p), ("pose_prior_std", f64p),
        ("has_mix_prior", C.c_int32), ("mix_prior", f64p), ("mix_prior_std", f64p),
        ("n_gnss", C.c_int32), ("gnss_node", i32p), ("gnss_blh", f64p), ("gnss_std", f64p), ("lever", C.c_double * 3),
        ("gnss_huber", C.c_int32),
        ("marg_r", C.c_int32), ("marg_nblocks", C.c_int32), ("marg_block_type", i32p), ("marg_block_node", i32p),
        ("marg_x0", f64p), ("marg_J0", f64p), ("marg_e0", f64p),
    ]


class BaPrior(C.Structure):
    """ctypes image of `icg_ba_prior`."""
    _fields_ = [("m", C.c_int32), ("r", C.c_int32), ("nblocks", C.c_int32), ("rcap", C.c_int32), ("block_type", i32p), ("block_node", i32p),
                ("x0", f64p), ("J0", f64p), ("e0", f64p), ("Hp", f64p), ("bp", f64p)]


class BaSummary(C.Structure):
    """ctypes image of `icg_ba_summary`."""
    _fields_ = [("iterations", C.c_int32), ("num_successful_steps", C.c_int32), ("termination", C.c_int32), ("reserved", C.c_int32),
                ("initial_cost", C.c_double), ("final_cost", C.c_double), ("final_radius", C.c_double)]


class CullWindow(C.Structure):
    """ctypes image of `icg_ba_cull_window`."""
    _fields_ = [("R_bc", C.c_double * 9), ("t_bc", C.c_double * 3), ("td_bc", C.c_double), ("estimate_ext", C.c_int32), ("estimate_td", C.c_int32),
                ("lm_ref_node", i32p), ("lm_ref_kp", f32p), ("obs_off", i32p), ("obs_node", i32p), ("obs_kp", f32p), ("obs_factor", i32p),
                ("R_bc_out", C.c_double * 9), ("t_bc_out", C.c_double * 3), ("td_bc_out", C.c_double), ("ext_accepted", C.c_int32),
                ("cam_pose", f64p), ("lm_pw", f64p), ("lm_depth", f64p), ("lm_outlier", u8p), ("obs_outlier", u8p), ("counts", C.c_int32 * 5)]


class CullLists(C.Structure):
    """ctypes image of `icg_ba_cull_lists`."""
    _fields_ = [("n_obs", C.c_int32), ("lm_ref_node", i32p), ("obs_off", i32p), ("obs_node", i32p), ("obs_factor", i32p),
                ("lm_ref_kp", f32p), ("obs_kp", f32p)]


class ReintWindow(C.Structure):
    """ctypes image of `icg_ba_reint_window`."""
    _fields_ = [("reintegrate", C.c_int32), ("imu", f64p), ("imu_off", i32p), ("status", i8p), ("blob_out", f64p), ("end_state10", f64p),
                ("count", C.c_int32)]


class SlideWindow(C.Structure):
    """ctypes image of `icg_ba_slide_window`."""
    _fields_ = [("node_src", i32p), ("lm_src", i32p), ("f_src", i32p), ("imu_src", i32p), ("gnss_src", i32p), ("prior_from_marg", C.c_int32)]


SLIDE_CHAIN, SLIDE_ROW = -2, -3  # ICG_SLIDE_CHAIN, ICG_SLIDE_ROW


class SlideIntegrate(C.Structure):
    """ctypes image of `icg_ba_slide_integrate`."""
    _fields_ = [("imu_from", i32p), ("state16", f64p), ("gravity3", f64p), ("normal", u8p), ("imu", f64p), ("imu_off", i32p),
                ("node_from_imu", u8p), ("gnss_node", i32p), ("gnss_dt", f64p),
                ("status", i8p), ("blob_out", f64p), ("end_state10", f64p)]


class InsCut(C.Structure):
    """ctypes image of `icg_ba_ins_cut`."""
    _fields_ = [("stream", C.c_int32), ("node_time", f64p)]


class SlideIns(C.Structure):
    """ctypes image of `icg_ba_slide_ins`."""
    _fields_ = [("integ", SlideIntegrate), ("stream", C.c_int32), ("node_time", f64p), ("merge_src", i32p), ("n_rows", i32p)]


class SlideVision(C.Structure):
    """ctypes image of `icg_ba_slide_vision` (device pointers as void *)."""
    _fields_ = [("num_marg", C.c_int32), ("node_in_map", u8p), ("obs_factor", i32p), ("cam", C.c_double * 10), ("node_td", f64p),
                ("cur_node", C.c_int32), ("n_frames", C.c_int32), ("frame_id", i64p), ("frame_node", i32p),
                ("n_obs", C.c_int32), ("n_in", C.c_int32), ("dev_n", vp), ("obs_src", vp), ("obs_lm", vp), ("obs_node", vp), ("obs_undis_xy", vp),
                ("obs_vel", vp), ("n_new", C.c_int32), ("dev_new_n", vp), ("new_depth", vp), ("new_vel_ref", vp), ("new_vel_cur", vp),
                ("new_ref_undis_xy", vp), ("new_cur_undis_xy", vp), ("new_ref_frame_id", vp),
                ("L", C.c_int32), ("F", C.c_int32), ("nan_dropped", C.c_int32),
                ("lm_src", i32p), ("f_src", i32p), ("f_lm", i32p), ("f_ref", i32p), ("f_obs", i32p), ("lm_origin", i32p), ("nan_flags", u8p),
                ("invdepth", f64p), ("f_const", f64p)]


class Linearization(C.Structure):
    """ctypes image of `icg_ba_linearization`."""
    _fields_ = [("K", C.c_int32), ("L", C.c_int32), ("F", C.c_int32), ("n_pairs", C.c_int32), ("lin_buf", C.c_int32), ("radius", C.c_double), ("pair_ro", i32p), ("Mp", f64p), ("A_W", f64p),
                ("h_l", f64p), ("g_l", f64p), ("H_c", f64p), ("g_c", f64p), ("costf", f64p), ("scale_l", f64p), ("Hs", f64p), ("visv", f64p)]


class Structure(C.Structure):
    """ctypes image of `icg_ba_structure`."""
    _fields_ = [("K", C.c_int32), ("L", C.c_int32), ("F", C.c_int32), ("n_runs", C.c_int32), ("npairs", C.c_int32), ("lm_perm", i32p),
                ("lm_off", i32p), ("f_meta_s", i32p), ("vb_lm0", i32p), ("ref_nrun", i32p), ("part_off", i32p), ("pair_ro", i32p),
                ("vis_ord", i32p), ("f_active", u8p)]


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
