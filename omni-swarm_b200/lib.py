"""ctypes binding of csrc/libomniswarm_b200.so (the C ABI declared in include/omniswarm_b200.h).

There is no CPU fallback: `load()` raises if the library has not been built, and every `create`
returns OSB_ERR_NO_DEVICE without a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(CSRC, "libomniswarm_b200.so")

OK, ERR_INVALID, ERR_CUDA, ERR_CAPACITY, ERR_NO_DEVICE = 0, 1, 2, 3, 4
PRECISION_SPLIT_FP16, PRECISION_FP16 = 0, 1
MAIN_CAMERA_UP, MAIN_CAMERA_DOWN = 0, 1
DB_STORAGE_FP32, DB_STORAGE_FP16 = 0, 1
MAX_DIRS, MAX_KPTS, FEATURE_DESC_SIZE, DEEP_DESC_SIZE = 4, 200, 64, 4096
REMOTE_MAGIN_NUMBER = 1000000
SWARM_ID_BYTES = 128
PAYLOAD_LEN = 24


class OsbError(RuntimeError):
    def __init__(self, status, text):
        super().__init__(f"libomniswarm_b200 status {status}: {text}")
        self.status = status


class SolveOptions(C.Structure):
    _fields_ = [("max_iterations", C.c_int32), ("max_pcg_iterations", C.c_int32), ("max_time_s", C.c_double),
                ("function_tolerance", C.c_double), ("gradient_tolerance", C.c_double),
                ("parameter_tolerance", C.c_double), ("pcg_tolerance", C.c_double),
                ("initial_trust_radius", C.c_double), ("preconditioner", C.c_int32), ("inner_precision", C.c_int32)]


class SolveSummary(C.Structure):
    _fields_ = [("initial_cost", C.c_double), ("final_cost", C.c_double), ("solve_ms", C.c_double),
                ("iterations", C.c_int32), ("pcg_iterations", C.c_int32), ("n_residuals", C.c_int32),
                ("termination", C.c_int32)]


class MultistartOptions(C.Structure):
    _fields_ = [("n_trials", C.c_int32), ("normalise", C.c_int32), ("window_size", C.c_int32), ("seed", C.c_uint64),
                ("rand_xy", C.c_double), ("rand_z", C.c_double), ("acpt_cost", C.c_double)]


class KeyframeRecord(C.Structure):
    _fields_ = [("drone_id", C.c_int32), ("msg_id", C.c_int32), ("n_dirs", C.c_int32), ("reserved", C.c_int32),
                ("n_kpts", C.c_int32 * MAX_DIRS), ("n_kpts_down", C.c_int32 * MAX_DIRS),
                ("global_desc", (C.c_float * DEEP_DESC_SIZE) * MAX_DIRS),
                ("local_desc", ((C.c_float * FEATURE_DESC_SIZE) * MAX_KPTS) * MAX_DIRS),
                ("kpts", ((C.c_float * 2) * MAX_KPTS) * MAX_DIRS),
                ("stereo_match", (C.c_int32 * MAX_KPTS) * MAX_DIRS),
                ("landmarks_3d", ((C.c_float * 3) * MAX_KPTS) * MAX_DIRS),
                ("landmarks_flag", (C.c_int32 * MAX_KPTS) * MAX_DIRS)]


class LoopResult(C.Structure):
    _fields_ = [("hit_id", C.c_int32), ("hit_dir", C.c_int32), ("hit_score", C.c_float), ("accepted", C.c_int32),
                ("swapped", C.c_int32), ("hit_msg_id", C.c_int32), ("hit_drone_id", C.c_int32), ("dir_new", C.c_int32 * MAX_DIRS), ("dir_old", C.c_int32 * MAX_DIRS),
                ("n_matches", C.c_int32 * MAX_DIRS), ("match_new", (C.c_int32 * MAX_KPTS) * MAX_DIRS),
                ("match_old", (C.c_int32 * MAX_KPTS) * MAX_DIRS),
                ("geo_valid", C.c_int32 * MAX_DIRS), ("n_geo", C.c_int32 * MAX_DIRS),
                ("geo_new", (C.c_int32 * MAX_KPTS) * MAX_DIRS), ("geo_old", (C.c_int32 * MAX_KPTS) * MAX_DIRS)]


class LoopEdge(C.Structure):
    _fields_ = [("id_a", C.c_int32), ("id_b", C.c_int32), ("rel_pose", C.c_double * 7), ("cov", C.c_double * 36),
                ("odom_a", C.c_double * 7), ("odom_b", C.c_double * 7), ("len_a", C.c_double), ("len_b", C.c_double)]


class PcmStateParams(C.Structure):
    _fields_ = [("self_id", C.c_int32), ("redundant", C.c_int32), ("max_pairs", C.c_int32), ("pair_capacity", C.c_int32),
                ("pcm_thres", C.c_double), ("odom_pos_cov_per_m", C.c_double), ("odom_ang_cov_per_m", C.c_double)]


class AnchorParams(C.Structure):
    _fields_ = [("max_drones", C.c_int32), ("max_traj_samples", C.c_int32), ("max_measurements", C.c_int32),
                ("max_window_entries", C.c_int32), ("begin_min_loop_dt_s", C.c_double), ("det_dpos_thres", C.c_double),
                ("odom_pos_cov_per_m", C.c_double), ("odom_ang_cov_per_m", C.c_double), ("huber", C.c_int32),
                ("reserved", C.c_int32)]


MEAS_LOOP, MEAS_DET4D, MEAS_DET6D = 0, 1, 2
# numpy views of osb_measurement, osb_window_entry, osb_loop_edge and osb_anchor_result (include/omniswarm_b200.h)
MEASUREMENT_DTYPE = np.dtype([("id", "<i8"), ("type", "<i4"), ("id_a", "<i4"), ("id_b", "<i4"), ("reserved", "<i4"),
                              ("stamp_a", "<i8"), ("stamp_b", "<i8"), ("relative_pose", "<f8", 7), ("cov", "<f8", (6, 6)),
                              ("self_pose_a", "<f8", 7), ("self_pose_b", "<f8", 7)])
WINDOW_ENTRY_DTYPE = np.dtype([("drone_id", "<i4"), ("vo_available", "<i4"), ("block", "<i4"), ("reserved", "<i4"),
                               ("stamp", "<i8"), ("self_pose", "<f8", 7)])
LOOP_EDGE_DTYPE = np.dtype([("id_a", "<i4"), ("id_b", "<i4"), ("rel_pose", "<f8", 7), ("cov", "<f8", (6, 6)),
                            ("odom_a", "<f8", 7), ("odom_b", "<f8", 7), ("len_a", "<f8"), ("len_b", "<f8")])
ANCHOR_RESULT_DTYPE = np.dtype([("id", "<i8"), ("type", "<i4"), ("status", "<i4"), ("frame_a", "<i4"), ("frame_b", "<i4"),
                                ("node_a", "<i4"), ("node_b", "<i4"), ("stamp_a", "<i8"), ("stamp_b", "<i8"),
                                ("dt_err_ns", "<i8"), ("dpos", "<f8"), ("edge", LOOP_EDGE_DTYPE), ("skip", "<i4"),
                                ("factor_type", "<i4"), ("ia", "<i4"), ("ib", "<i4"), ("huber", "<i4"), ("reserved", "<i4"),
                                ("payload", "<f8", PAYLOAD_LEN)])
ANCHOR_OK, ANCHOR_EMPTY_WINDOW, ANCHOR_BEFORE_WINDOW, ANCHOR_NO_FRAME, ANCHOR_NO_TRAJECTORY, ANCHOR_DPOS, ANCHOR_VOID = range(7)


class PnpParams(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("reproj_thresh", C.c_float), ("seed", C.c_uint32), ("is_4dof", C.c_int32),
                ("min_loop_num", C.c_int32), ("same_drone", C.c_int32), ("rperr_thres", C.c_double),
                ("accept_loop_yaw_rad", C.c_double), ("max_loop_dis", C.c_double),
                ("odometry_consistency_threshold", C.c_double), ("prior", C.c_double * 7), ("extrinsic", C.c_double * 7),
                ("drone_pose_now", C.c_double * 7), ("drone_pose_old", C.c_double * 7), ("odom_rel", C.c_double * 7),
                ("odom_edge_cov", C.c_double * 36)]


class PnpResult(C.Structure):
    _fields_ = [("pnp_success", C.c_int32), ("n_inliers", C.c_int32), ("winner", C.c_int32), ("verified", C.c_int32),
                ("odometry_consistent", C.c_int32), ("reserved", C.c_int32), ("rperr", C.c_double), ("md", C.c_double),
                ("pose_cam", C.c_double * 7), ("dp_old_to_new", C.c_double * 4)]


(LOOP_ACCEPTED, LOOP_NO_HIT, LOOP_NO_FRAME, LOOP_FEW_LANDMARKS, LOOP_CORRESPONDENCE_FAILED, LOOP_TOO_FEW_COMMON,
 LOOP_PNP_FAILED, LOOP_NOT_VERIFIED, LOOP_ODOMETRY_INCONSISTENT) = range(9)
LOOP_MAXN = MAX_DIRS * MAX_KPTS


class LoopParams(C.Structure):
    _fields_ = [("min_loop_num", C.c_int32), ("init_mode_min_loop_num", C.c_int32), ("min_match_per_dir", C.c_int32),
                ("min_direction_loop", C.c_int32), ("is_4dof", C.c_int32), ("reproj_thresh", C.c_float),
                ("seed", C.c_uint32), ("reserved", C.c_int32), ("rperr_thres", C.c_double),
                ("accept_loop_yaw_rad", C.c_double), ("max_loop_dis", C.c_double),
                ("odometry_consistency_threshold", C.c_double)]


class LoopCandidate(C.Structure):
    _fields_ = [("init_mode", C.c_int32), ("reserved", C.c_int32), ("pose_query", C.c_double * 7),
                ("pose_hit", C.c_double * 7), ("odom_rel", C.c_double * 7), ("odom_edge_cov", C.c_double * 36)]


class LoopEdgeResult(C.Structure):
    _fields_ = [("status", C.c_int32), ("drone_id_a", C.c_int32), ("drone_id_b", C.c_int32), ("msg_id_a", C.c_int32),
                ("msg_id_b", C.c_int32), ("main_dir_new", C.c_int32), ("main_dir_old", C.c_int32),
                ("matched_dir_count", C.c_int32), ("n_corr", C.c_int32), ("reserved", C.c_int32), ("pnp", PnpResult),
                ("relative_pose", C.c_double * 7), ("corr_dir_new", C.c_int32 * LOOP_MAXN),
                ("corr_idx_new", C.c_int32 * LOOP_MAXN), ("corr_dir_old", C.c_int32 * LOOP_MAXN),
                ("corr_idx_old", C.c_int32 * LOOP_MAXN), ("inlier", C.c_uint8 * LOOP_MAXN)]


class LoopStamps(C.Structure):
    _fields_ = [("stamp_query_ns", C.c_int64), ("stamp_hit_ns", C.c_int64)]


LOOP_PAIR_DRONES = 256         # inter_drone_loop_count is kept for drone ids 0..255 (osb_frontend_loop_counts)


class FrontendConfig(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("n_dirs", C.c_int32), ("max_num", C.c_int32),
                ("sp_thres", C.c_float), ("self_id", C.c_int32), ("db_capacity", C.c_int32),
                ("inner_product_thres", C.c_double), ("init_mode_product_thres", C.c_double),
                ("match_index_dist", C.c_int32), ("query_dir", C.c_int32), ("zero_bottom_quarter", C.c_int32),
                ("accept_min_3d_pts", C.c_int32), ("geometric_filter", C.c_int32), ("ransac_seed", C.c_int32)]


RECORD_BYTES = C.sizeof(KeyframeRecord)
RESULT_BYTES = C.sizeof(LoopResult)
EDGE_BYTES = C.sizeof(LoopEdgeResult)

_P = C.c_void_p
_SIG = {
    "osb_last_error": (C.c_char_p, []),
    "osb_version": (C.c_char_p, []),
    "osb_device_count": (C.c_int, []),
    "osb_launch_count": (C.c_int64, []),
    "osb_live_resources": (C.c_int64, []),
    "osb_set_sm_budget": (None, [C.c_int]),
    "osb_superpoint_create": (C.c_int, [C.POINTER(_P), _P, C.c_size_t, C.c_int, C.c_int, C.c_float, C.c_int, _P, _P, C.c_int]),
    "osb_superpoint_destroy": (C.c_int, [_P]),
    "osb_superpoint_infer": (C.c_int, [_P, _P, C.c_int, _P, _P, _P]),
    "osb_superpoint_infer_dev": (C.c_int, [_P, _P, C.c_int, _P, _P, _P, _P]),
    "osb_superpoint_postprocess": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P]),
    "osb_superpoint_read": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_size_t]),
    "osb_superpoint_set_profiling": (C.c_int, [_P, C.c_int]),
    "osb_superpoint_layer_ms": (C.c_int, [_P, _P, C.c_int]),
    "osb_superpoint_set_precision": (C.c_int, [_P, C.c_int]),
    "osb_superpoint_band_geometry": (C.c_int, [C.c_int, C.c_int, C.c_int, _P]),
    "osb_conv_layer_parity": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_float, _P, _P, C.c_int, C.c_int, C.c_int,
                                        C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P,
                                        C.c_float, _P]),
    "osb_conv_first_parity": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_float, _P, _P, _P]),
    "osb_dwconv_parity": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, _P, _P,
                                    _P]),
    "osb_conv_layer_fp16_parity": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_float, _P, C.c_int, C.c_int, C.c_int,
                                             C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P,
                                             C.c_float, _P]),
    "osb_conv_first_fp16_parity": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_float, _P, _P]),
    "osb_dwconv_fp16_parity": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, _P,
                                         _P]),
    "osb_netvlad_create": (C.c_int, [C.POINTER(_P), _P, C.c_size_t, C.c_int, C.c_int, C.c_int]),
    "osb_netvlad_destroy": (C.c_int, [_P]),
    "osb_netvlad_infer": (C.c_int, [_P, _P, C.c_int, _P]),
    "osb_netvlad_infer_dev": (C.c_int, [_P, _P, C.c_int, _P, _P]),
    "osb_netvlad_set_precision": (C.c_int, [_P, C.c_int]),
    "osb_conv_ffma_parity": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                       _P, _P]),
    "osb_conv_first_ffma_parity": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "osb_dwconv_ffma_parity": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "osb_maxpool_parity": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "osb_nv_block0_parity": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "osb_nv_head_parity": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P]),
    "osb_db_create": (C.c_int, [C.POINTER(_P), C.c_int, C.c_int64]),
    "osb_db_create_storage": (C.c_int, [C.POINTER(_P), C.c_int, C.c_int64, C.c_int]),
    "osb_db_destroy": (C.c_int, [_P]),
    "osb_db_add": (C.c_int, [_P, C.c_int64, _P, C.POINTER(C.c_int64)]),
    "osb_db_add_dev": (C.c_int, [_P, C.c_int64, _P, C.POINTER(C.c_int64), _P]),
    "osb_db_search": (C.c_int, [_P, C.c_int64, _P, C.c_int, _P, _P]),
    "osb_db_search_dev": (C.c_int, [_P, C.c_int64, _P, C.c_int, _P, _P, _P]),
    "osb_topk_merge_dev": (C.c_int, [C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P]),
    "osb_db_size": (C.c_int64, [_P]),
    "osb_db_reset": (C.c_int, [_P]),
    "osb_homography_ransac": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_float, C.c_uint32, _P, _P, _P]),
    "osb_homography_ransac_dev": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_float, C.c_uint32, _P, _P, _P, _P]),
    "osb_matcher_create": (C.c_int, [C.POINTER(_P), C.c_int, C.c_int, C.c_int]),
    "osb_matcher_destroy": (C.c_int, [_P]),
    "osb_matcher_match": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P]),
    "osb_matcher_match_dev": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "osb_solve_default_options": (None, [C.POINTER(SolveOptions)]),
    "osb_solver_create": (C.c_int, [C.POINTER(_P), C.c_int, C.c_int]),
    "osb_solver_destroy": (C.c_int, [_P]),
    "osb_solver_solve": (C.c_int, [_P, C.c_int, _P, _P, C.c_int, _P, _P, _P, _P, _P, C.POINTER(SolveOptions), C.POINTER(SolveSummary)]),
    "osb_solver_solve_multistart": (C.c_int, [_P, C.c_int, _P, _P, _P, C.c_int, _P, _P, _P, _P, _P,
                                              C.POINTER(SolveOptions), C.POINTER(MultistartOptions), _P, _P,
                                              C.POINTER(C.c_int32)]),
    "osb_solver_graph_clear": (C.c_int, [_P]),
    "osb_solver_graph_add_nodes": (C.c_int, [_P, C.c_int, _P, _P, C.POINTER(C.c_int32)]),
    "osb_solver_graph_add_factors": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P]),
    "osb_solver_graph_set_fixed": (C.c_int, [_P, C.c_int, C.c_int]),
    "osb_solver_graph_set_poses": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "osb_solver_graph_get_poses": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "osb_solver_graph_size": (C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "osb_solver_graph_drop_oldest": (C.c_int, [_P, C.c_int]),
    "osb_solver_solve_resident": (C.c_int, [_P, _P, _P]),
    "osb_solver_solve_resident_dev": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P]),
    "osb_solver_last_summary": (C.c_int, [_P, _P]),
    "osb_solver_phase_cycles": (C.c_int, [_P, _P]),
    "osb_solver_chain_cycles": (C.c_int, [_P, _P]),
    "osb_solver_chain_plan": (C.c_int, [C.c_int, _P, C.c_int, _P, _P, _P, _P, _P, _P]),
    "osb_solver_linearize": (C.c_int, [_P, C.c_int, _P, C.c_int, _P, _P, _P, _P, _P, _P, _P]),
    "osb_frontend_create": (C.c_int, [C.POINTER(_P), C.POINTER(FrontendConfig), _P, C.c_size_t, _P, _P, _P, C.c_size_t]),
    "osb_frontend_destroy": (C.c_int, [_P]),
    "osb_frontend_extract": (C.c_int, [_P, _P, _P, C.c_int32, _P, _P]),
    "osb_frontend_extract_dev": (C.c_int, [_P, _P, _P, C.c_int32, _P, _P]),
    "osb_frontend_ingest": (C.c_int, [_P, _P, C.c_int, C.c_int, _P]),
    "osb_frontend_ingest_own": (C.c_int, [_P, _P, _P]),
    "osb_frontend_query": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P]),
    "osb_frontend_query_received": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "osb_frontend_set_loop_params": (C.c_int, [_P, C.POINTER(LoopParams)]),
    "osb_frontend_compute_loop": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P]),
    "osb_frontend_loop_measurements": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, C.c_double, C.c_double, _P, _P, _P]),
    "osb_frontend_loop_counts": (C.c_int, [_P, C.POINTER(C.c_int64), _P]),
    "osb_frontend_process": (C.c_int, [_P, _P, _P, C.c_int32, _P, _P]),
    "osb_frontend_finish": (C.c_int, [_P, _P]),
    "osb_frontend_set_profiling": (C.c_int, [_P, C.c_int]),
    "osb_frontend_stage_ms": (C.c_int, [_P, _P]),
    "osb_frontend_set_precision": (C.c_int, [_P, C.c_int]),
    "osb_frontend_set_main_camera": (C.c_int, [_P, C.c_int]),
    "osb_frontend_set_db_storage": (C.c_int, [_P, C.c_int]),
    "osb_frontend_db_size": (C.c_int64, [_P, C.c_int]),
    "osb_frontend_db_reset": (C.c_int, [_P]),
    "osb_frontend_db_load": (C.c_int, [_P, C.c_int, C.c_int64, _P, _P, _P]),
    "osb_frontend_db_set_geometry": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int64, _P, _P]),
    "osb_stereo_lift": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P, C.c_double, C.c_int, _P, _P, _P]),
    "osb_stereo_lift_dev": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P, C.c_double, C.c_int, _P, _P, _P, _P]),
    "osb_depth_lift": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P, _P, C.c_double, C.c_double, C.c_int, _P, _P]),
    "osb_depth_lift_dev": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P, _P, C.c_double, C.c_double, C.c_int, _P, _P, _P]),
    "osb_frontend_set_cameras": (C.c_int, [_P, _P, _P, _P, C.c_double]),
    "osb_frontend_set_drone_pose": (C.c_int, [_P, _P]),
    "osb_frontend_set_depth_camera": (C.c_int, [_P, _P, _P, C.c_double, C.c_double]),
    "osb_frontend_extract_depth": (C.c_int, [_P, _P, _P, C.c_int32, _P, _P]),
    "osb_frontend_extract_depth_dev": (C.c_int, [_P, _P, _P, C.c_int32, _P, _P]),
    "osb_frontend_process_depth": (C.c_int, [_P, _P, _P, C.c_int32, _P, _P]),
    "osb_pnp_ransac": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "osb_pnp_ransac_dev": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P, _P]),
    "osb_pcm": (C.c_int, [_P, C.c_int, C.c_double, C.c_double, C.c_double, _P, _P, _P, _P]),
    "osb_pcm_dev": (C.c_int, [_P, C.c_int, C.c_double, C.c_double, C.c_double, _P, _P, _P, _P, _P]),
    "osb_pcm_state_create": (C.c_int, [C.POINTER(_P), C.POINTER(PcmStateParams)]),
    "osb_pcm_state_destroy": (C.c_int, [_P]),
    "osb_pcm_state_reject": (C.c_int, [_P, _P, _P, C.c_int, _P]),
    "osb_pcm_state_inliers": (C.c_int, [_P, C.c_int32, C.c_int32, _P, C.c_int, C.POINTER(C.c_int32)]),
    "osb_pcm_state_set_inliers": (C.c_int, [_P, C.c_int32, C.c_int32, _P, C.c_int]),
    "osb_pcm_state_pair": (C.c_int, [_P, C.c_int32, C.c_int32, C.POINTER(C.c_int32), _P, _P, _P, C.POINTER(C.c_int32)]),
    "osb_pcm_state_reject_anchored": (C.c_int, [_P, _P, C.c_int, _P, _P]),
    "osb_pcm_state_status": (C.c_int, [_P, C.POINTER(C.c_int)]),
    "osb_anchor_create": (C.c_int, [C.POINTER(_P), C.POINTER(AnchorParams)]),
    "osb_anchor_destroy": (C.c_int, [_P]),
    "osb_anchor_push_odometry": (C.c_int, [_P, C.c_int32, C.c_int, _P, _P]),
    "osb_anchor_add_measurements": (C.c_int, [_P, C.c_int, _P]),
    "osb_anchor_size": (C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "osb_anchor_set_window": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "osb_anchor_run": (C.c_int, [_P, _P, _P, C.POINTER(C.c_int32)]),
    "osb_anchor_run_dev": (C.c_int, [_P, _P, _P, C.POINTER(C.c_int32), _P]),
    "osb_anchor_compact_factors_dev": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P]),
    "osb_anchor_add_measurements_dev": (C.c_int, [_P, _P, _P, C.c_int, C.c_float, _P]),
    "osb_anchor_status": (C.c_int, [_P, C.POINTER(C.c_int)]),
    "osb_swarm_unique_id": (C.c_int, [_P]),
    "osb_swarm_init": (C.c_int, [C.POINTER(_P), _P, C.c_int, C.c_int]),
    "osb_swarm_destroy": (C.c_int, [_P]),
    "osb_swarm_exchange": (C.c_int, [_P, _P, _P, _P]),
    "osb_swarm_exchange_async": (C.c_int, [_P, _P, _P, _P]),
    "osb_swarm_wait": (C.c_int, [_P, _P]),
    "osb_swarm_rank": (C.c_int, [_P]),
    "osb_swarm_transport": (C.c_int, [_P]),
    "osb_swarm_world": (C.c_int, [_P]),
}

_lib = None


def build(verbose: bool = False) -> str:
    """Compile csrc/*.cu for sm_90a into csrc/libomniswarm_b200.so (nvcc cross-compiles without a GPU)."""
    r = subprocess.run(["make", "-C", CSRC, "-j8"], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout[-4000:])
        print(r.stderr[-4000:])
    if r.returncode != 0:
        raise RuntimeError("building libomniswarm_b200.so failed")
    return LIB_PATH


def exported_symbols():
    return sorted(_SIG)


def load():
    """Load the shared library and attach the signatures.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIG.items():
        fn = getattr(lib, name)          # AttributeError here = symbol missing from the build
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int):
    if status != OK:
        raise OsbError(status, load().osb_last_error().decode(errors="replace"))


def ptr(a):
    """numpy array / ctypes object / int (device pointer) -> c_void_p"""
    import numpy as np
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"], "array must be C-contiguous"
        return a.ctypes.data_as(C.c_void_p)
    return C.cast(C.byref(a), C.c_void_p)
