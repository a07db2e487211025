"""ctypes binding of the C-ABI in include/gslam_b200.h (gslam_b200/lib/libgslam_b200_kernels.so).

This is the same boundary the C++ GSLAM plugins link against; Python is only the harness language of tests and
bench.py.  There is no CPU fallback: if the CUDA library is missing or no device is usable, loading / context creation
raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libgslam_b200_kernels.so")
_LIB = None

GB_OK, GB_ERR_INVALID, GB_ERR_CUDA, GB_ERR_CAPACITY, GB_ERR_NODEVICE, GB_ERR_NUMERIC = range(6)

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])
assert KP_DTYPE.itemsize == 28

f64p = C.POINTER(C.c_double)
u8p = C.POINTER(C.c_uint8)
i32p = C.POINTER(C.c_int32)


class OrbCfg(C.Structure):
    _fields_ = [("nfeatures", C.c_int32), ("scale_factor", C.c_float), ("nlevels", C.c_int32),
                ("edge_threshold", C.c_int32), ("first_level", C.c_int32), ("wta_k", C.c_int32),
                ("score_type", C.c_int32), ("patch_size", C.c_int32), ("fast_threshold", C.c_int32)]


class BaProblem(C.Structure):
    _fields_ = [("n_cams", C.c_int32), ("n_points", C.c_int32), ("n_obs", C.c_int32),
                ("cam_pose_wc", f64p), ("cam_dof", u8p), ("points", f64p), ("point_free", u8p),
                ("obs_cam", i32p), ("obs_point", i32p), ("obs_xyz", f64p), ("obs_info", f64p)]


class PoseEdges(C.Structure):
    _fields_ = [("n_se3", C.c_int32), ("se3_first", i32p), ("se3_second", i32p), ("se3_meas", f64p), ("se3_info", f64p),
                ("n_gps", C.c_int32), ("gps_frame", i32p), ("gps_meas", f64p), ("gps_info", f64p)]


class BaOptions(C.Structure):
    _fields_ = [("projection", C.c_int32), ("huber_delta", C.c_double), ("max_iterations", C.c_int32),
                ("verbose", C.c_int32), ("function_tolerance", C.c_double), ("lambda_init", C.c_double),
                ("pcg_max_iters", C.c_int32), ("pcg_tol", C.c_double), ("linear_solver", C.c_int32)]


class BaResult(C.Structure):
    _fields_ = [("initial_cost", C.c_double), ("final_cost", C.c_double), ("iterations", C.c_int32),
                ("accepted", C.c_int32), ("pcg_iterations", C.c_int32), ("status", C.c_int32),
                ("lambda_final", C.c_double), ("gpu_ms", C.c_float)]


class PnpStats(C.Structure):
    _fields_ = [("hypotheses", C.c_int32), ("best_hypothesis", C.c_int32), ("best_root", C.c_int32), ("inliers_minimal", C.c_int32),
                ("inliers_refined", C.c_int32)]


# every symbol include/gslam_b200.h declares: (name, restype, argtypes)
_VP = C.c_void_p
_SIGNATURES = [
    ("gb_version", C.c_int, []),
    ("gb_device_count", C.c_int, [C.POINTER(C.c_int)]),
    ("gb_ctx_create", C.c_int, [C.c_int, C.POINTER(_VP)]),
    ("gb_ctx_create_priority", C.c_int, [C.c_int, C.c_int, C.POINTER(_VP)]),
    ("gb_ctx_destroy", C.c_int, [_VP]),
    ("gb_last_error", C.c_char_p, [_VP]),
    ("gb_ctx_stream", _VP, [_VP]),
    ("gb_ctx_sync", C.c_int, [_VP]),
    ("gb_ctx_wait_for", C.c_int, [_VP, _VP]),
    ("gb_timer_begin", C.c_int, [_VP]),
    ("gb_timer_end", C.c_int, [_VP, C.POINTER(C.c_float)]),
    ("gb_launch_count", C.c_int64, [_VP]),
    ("gb_orb_cfg_default", None, [C.POINTER(OrbCfg)]),
    ("gb_orb_extract", C.c_int, [_VP, _VP, C.c_int, C.c_int, C.POINTER(OrbCfg), _VP, _VP, C.POINTER(C.c_int)]),
    ("gb_orb_extract_image", C.c_int, [_VP, _VP, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(OrbCfg), _VP, _VP, C.POINTER(C.c_int)]),
    ("gb_features_create", C.c_int, [_VP, C.c_int, C.POINTER(_VP)]),
    ("gb_features_destroy", C.c_int, [_VP, _VP]),
    ("gb_orb_extract_to", C.c_int, [_VP, _VP, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(OrbCfg), _VP]),
    ("gb_features_count", C.c_int, [_VP, _VP, C.POINTER(C.c_int)]),
    ("gb_features_upload", C.c_int, [_VP, _VP, _VP, _VP, C.c_int]),
    ("gb_features_download", C.c_int, [_VP, _VP, _VP, _VP, C.POINTER(C.c_int)]),
    ("gb_match_hamming", C.c_int, [_VP, _VP, C.c_int, _VP, C.c_int, _VP, _VP, _VP]),
    ("gb_match_features", C.c_int, [_VP, _VP, _VP]),
    ("gb_match_download", C.c_int, [_VP, _VP, _VP, _VP, _VP, C.POINTER(C.c_int)]),
    ("gb_match_stereo", C.c_int, [_VP, _VP, _VP, C.c_int, _VP, _VP, C.c_int, C.c_float, C.c_float, C.c_float, _VP, _VP, _VP]),
    ("gb_match_stereo_features", C.c_int, [_VP, _VP, _VP, C.c_float, C.c_float, C.c_float]),
    ("gb_remap_create", C.c_int, [_VP, C.c_int, C.c_int, C.c_int, C.c_int, _VP, _VP, _VP, C.POINTER(_VP)]),
    ("gb_remap_destroy", C.c_int, [_VP, _VP]),
    ("gb_remap_apply", C.c_int, [_VP, _VP, _VP, C.c_int, _VP]),
    ("gb_remap_apply_to", C.c_int, [_VP, _VP, _VP, C.c_int, C.c_int, C.c_int, _VP, C.c_int]),
    ("gb_orb_extract_undistorted_to", C.c_int, [_VP, _VP, _VP, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(OrbCfg), _VP]),
    ("gb_orb_extract_undistorted", C.c_int, [_VP, _VP, _VP, C.c_int, C.c_int, C.POINTER(OrbCfg), _VP, _VP, C.POINTER(C.c_int)]),
    ("gb_voc_create", C.c_int, [_VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint32, _VP, _VP, _VP, C.POINTER(_VP)]),
    ("gb_voc_destroy", C.c_int, [_VP, _VP]),
    ("gb_bow_transform", C.c_int, [_VP, _VP, _VP, C.c_int, C.c_int, _VP, _VP, C.POINTER(C.c_int), _VP, _VP, C.POINTER(C.c_int)]),
    ("gb_bow_transform_features", C.c_int, [_VP, _VP, _VP, C.c_int, _VP, _VP, C.POINTER(C.c_int), _VP, _VP, C.POINTER(C.c_int)]),
    ("gb_ba_options_default", None, [C.POINTER(BaOptions)]),
    ("gb_ba_solve", C.c_int, [_VP, C.POINTER(BaProblem), C.POINTER(BaOptions), C.POINTER(BaResult)]),
    ("gb_ba_pnp", C.c_int, [_VP, C.c_int, _VP, _VP, _VP, C.c_int, _VP, C.POINTER(BaOptions), C.POINTER(BaResult)]),
    ("gb_ba_graph_create", C.c_int, [_VP, C.POINTER(BaProblem), C.POINTER(_VP)]),
    ("gb_ba_graph_create_ex", C.c_int, [_VP, C.POINTER(BaProblem), C.POINTER(PoseEdges), C.POINTER(_VP)]),
    ("gb_ba_solve_posegraph", C.c_int, [_VP, C.POINTER(BaProblem), C.POINTER(PoseEdges), C.POINTER(BaOptions), C.POINTER(BaResult)]),
    ("gb_ba_graph_destroy", C.c_int, [_VP, _VP]),
    ("gb_ba_graph_reset", C.c_int, [_VP, _VP]),
    ("gb_ba_graph_solve", C.c_int, [_VP, _VP, C.POINTER(BaOptions), C.POINTER(BaResult)]),
    ("gb_ba_graph_download", C.c_int, [_VP, _VP, _VP, _VP]),
    ("gb_ba_graph_sweep", C.c_int, [_VP, _VP, C.c_double]),
    ("gb_ba_graph_reduce_size", C.c_int, [_VP, _VP, C.POINTER(C.c_size_t)]),
    ("gb_ba_graph_begin", C.c_int, [_VP, _VP, C.POINTER(BaOptions)]),
    ("gb_ba_graph_reduce_local", C.c_int, [_VP, _VP, _VP]),
    ("gb_ba_graph_step", C.c_int, [_VP, _VP, _VP, _VP]),
    ("gb_ba_graph_commit", C.c_int, [_VP, _VP, _VP, _VP]),
    ("gb_ba_graph_finish", C.c_int, [_VP, _VP, C.POINTER(BaResult)]),
    ("gb_pnp_ransac", C.c_int, [_VP, C.c_int, _VP, _VP, C.c_double, C.c_double, C.c_int, C.c_uint64, _VP, _VP, C.POINTER(PnpStats)]),
    ("gb_comm_unique_id", C.c_int, [_VP]),
    ("gb_comm_create", C.c_int, [_VP, C.c_int, C.c_int, _VP, C.POINTER(_VP)]),
    ("gb_comm_create_all", C.c_int, [C.c_int, C.POINTER(_VP), C.POINTER(_VP)]),
    ("gb_comm_destroy", C.c_int, [_VP]),
    ("gb_comm_rank", C.c_int, [_VP]),
    ("gb_comm_world", C.c_int, [_VP]),
    ("gb_comm_allreduce_sum_f64", C.c_int, [_VP, _VP, C.c_size_t]),
    ("gb_ba_shard_create", C.c_int, [_VP, C.POINTER(BaProblem), C.POINTER(_VP)]),
    ("gb_ba_shard_range", C.c_int, [_VP, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    ("gb_ba_shard_reduce_bytes", C.c_int, [_VP, C.POINTER(C.c_size_t)]),
    ("gb_ba_shard_solve", C.c_int, [_VP, _VP, C.POINTER(BaOptions), C.POINTER(BaResult)]),
    ("gb_ba_solve_multi", C.c_int, [C.c_int, C.POINTER(_VP), C.POINTER(BaProblem), C.POINTER(BaOptions), C.POINTER(BaResult)]),
]
# test hooks (not part of the reference-facing surface)
_DEBUG_SIGNATURES = [
    ("gb_dbg_ba_linearize", C.c_int, [_VP, _VP, C.c_double, _VP, _VP, _VP, _VP, _VP, _VP]),
    ("gb_dbg_ba_reduced", C.c_int, [_VP, _VP, C.POINTER(BaOptions), _VP, _VP, _VP, C.POINTER(C.c_int)]),
    ("gb_dbg_ba_system", C.c_int, [_VP, _VP, C.POINTER(BaOptions), _VP, _VP, _VP, C.POINTER(C.c_double), _VP, C.POINTER(C.c_int)]),
    ("gb_dbg_ba_last_step", C.c_int, [_VP, _VP, _VP, _VP, _VP]),
    ("gb_dbg_ba_force_generic_pcg", C.c_int, [_VP, _VP, C.c_int]),
    ("gb_dbg_ba_pcg_cluster_size", C.c_int, [_VP, _VP]),
    ("gb_dbg_ba_pcg_sparse", C.c_int, [_VP, _VP]),
    ("gb_dbg_ba_paths", C.c_int, [_VP, _VP]),
    ("gb_dbg_ba_set_cam_split", C.c_int, [_VP, _VP, C.c_int]),
    ("gb_dbg_ba_sweep_part", C.c_int, [_VP, _VP, C.c_int]),
    ("gb_dbg_ba_set_sweep", C.c_int, [_VP, _VP, C.c_int]),
    ("gb_dbg_ba_sweep_plan", C.c_int, [C.c_int, C.c_int, C.c_int, _VP, _VP, C.c_int, _VP, C.c_int, _VP, C.POINTER(C.c_int)]),
    ("gb_dbg_pnp_p3p_host", C.c_int, [_VP, _VP, _VP]),
    ("gb_dbg_pnp_minimal_host", C.c_int, [C.c_int, _VP, _VP, C.c_double, C.c_double, C.c_int, C.c_uint64, _VP, C.POINTER(PnpStats)]),
    ("gb_dbg_pnp_hypotheses_host", C.c_int, [C.c_int, _VP, _VP, C.c_double, C.c_uint64, C.c_int, _VP, _VP, _VP]),
    ("gb_dbg_pnp_hypotheses", C.c_int, [_VP, C.c_int, _VP, _VP, C.c_double, C.c_uint64, C.c_int, _VP, _VP, _VP]),
    ("gb_dbg_pnp_p3p_device", C.c_int, [_VP, C.c_int, _VP, _VP, _VP, _VP]),
    ("gb_dbg_ba_last_paths", C.c_int, [_VP]),
    ("gb_dbg_ba_shard_bounds", C.c_int, [C.c_int, C.c_int, _VP, C.c_int, _VP]),
    ("gb_dbg_comm_create_local", C.c_int, [_VP, C.c_int, C.POINTER(_VP), C.POINTER(_VP)]),
    ("gb_dbg_ba_shard_reduced", C.c_int, [_VP, _VP, C.POINTER(BaOptions), C.c_int, _VP, _VP, _VP, _VP]),
    ("gb_dbg_popc_peak", C.c_int, [_VP, C.POINTER(C.c_double)]),
    ("gb_dbg_match_last_plan", C.c_int, [_VP, _VP]),
    ("gb_dbg_features_set_pending", C.c_int, [_VP, _VP, C.c_int, C.c_int, C.c_int]),
    ("gb_dbg_bow_last_plan", C.c_int, [_VP, _VP]),
    ("gb_dbg_orb_level_size", C.c_int, [C.c_int, C.c_int, C.c_float, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    ("gb_dbg_orb_candidates", C.c_int, [_VP, C.c_int, _VP, _VP, _VP, _VP, C.c_int, C.POINTER(C.c_int), _VP, C.c_int, C.POINTER(C.c_int)]),
]

EXPORTED_SYMBOLS = [s[0] for s in _SIGNATURES]


class GbError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"gslam_b200 error {code}: {msg}")
        self.code = code


def lib() -> C.CDLL:
    """Load the CUDA library.  Raises (loudly) when it has not been built — there is no fallback implementation."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -m gslam_b200.build` (needs nvcc). "
                              "gslam_b200 has no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        for name, res, args in _SIGNATURES + _DEBUG_SIGNATURES:
            fn = getattr(L, name)  # AttributeError if the ABI and the header disagree
            fn.restype = res
            fn.argtypes = args
        _LIB = L
    return _LIB


def ptr(a):
    if a is None:
        return None
    return a.ctypes.data_as(C.c_void_p)
