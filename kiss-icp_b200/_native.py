"""ctypes binding of the C-ABI (include/kiss_icp_b200.h) + the in-tree build recipe.

The shared library is built IN-TREE (kiss-icp_b200/libkiss_icp_b200.so) with nvcc for sm_90a (H100)
so that a checkout that was built once runs on any H100 machine it is copied to. There is no CPU fallback: if the
library is missing it is an ImportError-grade failure, and without a CUDA device every compute
entry point returns KB_ERR_NO_DEVICE, surfaced here as ``NoDeviceError``.
"""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
LIB_PATH = os.environ.get("KB_LIB") or os.path.join(_HERE, "libkiss_icp_b200.so")  # KB_LIB: A/B builds side by side
CSRC = os.path.join(_HERE, "csrc")
HEADER = os.path.join(ROOT, "include", "kiss_icp_b200.h")
DEBUG_HEADER = os.path.join(ROOT, "include", "kiss_icp_b200_debug.h")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-fmad=false",  # FP64 products/sums round like the x86-64 reference build (no FMA contraction)
    "-shared", "-Xcompiler", "-fPIC",
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def sources():
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))] + [HEADER, DEBUG_HEADER]


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every csrc/*.cu -> libkiss_icp_b200.so (sm_90a). No-op when up to date."""
    stale = (not os.path.exists(LIB_PATH)) or any(os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in sources())
    if force or stale:
        cmd = [_nvcc(), *NVCC_FLAGS, "-o", LIB_PATH, *(s for s in sources() if s.endswith(".cu"))]
        if verbose:
            print(" ".join(cmd))
        env = dict(os.environ)
        env.pop("CXX", None)  # the image's CXX wrapper is not usable as nvcc host compiler
        env.pop("CC", None)
        subprocess.check_call(cmd, env=env)
    return LIB_PATH


class KissB200Error(RuntimeError):
    pass


class NoDeviceError(KissB200Error):
    pass


KB_OK, KB_ERR_INVALID_ARG, KB_ERR_NOT_SE3, KB_ERR_OUT_OF_RANGE, KB_ERR_CUDA, KB_ERR_CAPACITY, KB_ERR_NO_DEVICE = range(7)

_lib = None
vp, dbl, sz, i32, u32 = C.c_void_p, C.c_double, C.c_size_t, C.c_int, C.c_uint


class Config(C.Structure):
    """kb_config == KISSConfig (cpp/kiss_icp/pipeline/KissICP.hpp:36-54)."""
    _fields_ = [("voxel_size", dbl), ("max_range", dbl), ("min_range", dbl), ("max_points_per_voxel", i32),
                ("min_motion_th", dbl), ("initial_threshold", dbl), ("max_num_iterations", i32),
                ("convergence_criterion", dbl), ("max_num_threads", i32), ("deskew", i32)]


class FrameStats(C.Structure):
    """kb_frame_stats"""
    _fields_ = [("pose", dbl * 16), ("phase_us", dbl * 6), ("icp_queries", dbl), ("icp_candidates", dbl),
                ("iterations", i32), ("n_points_in", i32), ("n_preprocessed", i32), ("n_downsampled", i32),
                ("n_source", i32), ("map_points", i32), ("map_voxels", i32), ("team", i32)]


class PipelineState(C.Structure):
    """kb_pipeline_state: pose / delta in Sophus::SE3d::params() order {qx,qy,qz,qw,tx,ty,tz}"""
    _fields_ = [("pose", dbl * 7), ("delta", dbl * 7), ("model_sse", dbl), ("num_samples", i32)]


class Fit(C.Structure):
    """kb_fit: the fit of one localized frame at its final pose"""
    _fields_ = [("n_correspondences", i32), ("n_source", i32), ("sum_sq_residual", dbl), ("JTJ", dbl * 36)]


class Constraints(C.Structure):
    """kb_constraints: the plane constraints of one source at one pose"""
    _fields_ = [("n_planes", i32), ("weight_sum", dbl), ("sum_sq_plane_residual", dbl), ("information", dbl * 36)]


class Degeneracy(C.Structure):
    """kb_degeneracy: the degeneracy-aware ICP's eigen-decomposition of one frame"""
    _fields_ = [("n_planes", i32), ("weight_sum", dbl), ("translation_eigenvalues", dbl * 3),
                ("translation_axes", dbl * 9), ("rotation_eigenvalues", dbl * 3), ("rotation_axes", dbl * 9),
                ("translation_held", i32 * 3), ("rotation_held", i32 * 3)]


class Motion(C.Structure):
    """kb_motion: sampled poses of the LiDAR that deskew and predict one frame"""
    _fields_ = [("times", vp), ("poses", vp), ("m", sz), ("stamp_offset", dbl), ("end_time", dbl)]


class Sensor(C.Structure):
    """kb_sensor: one LiDAR of a rig, its extrinsic (base <- sensor) and its range crop"""
    _fields_ = [("extrinsic", dbl * 16), ("min_range", dbl), ("max_range", dbl)]


class RigCalibrationOptions(C.Structure):
    """kb_rig_calibration_options"""
    _fields_ = [("max_correspondence_distance", dbl), ("kernel_scale", dbl), ("max_iterations", i32),
                ("convergence_criterion", dbl)]


class SensorCalibration(C.Structure):
    """kb_sensor_calibration: one sensor's result of kb_calibrate_rig"""
    _fields_ = [("iterations", i32), ("converged", i32), ("fit", Fit), ("constraints", Constraints)]


class RigClockCalibrationOptions(C.Structure):
    """kb_rig_clock_calibration_options"""
    _fields_ = [("max_correspondence_distance", dbl), ("kernel_scale", dbl), ("max_iterations", i32),
                ("convergence_criterion", dbl), ("time_convergence_criterion", dbl)]


class SensorClockCalibration(C.Structure):
    """kb_sensor_clock_calibration: one sensor's result of kb_calibrate_rig_clocks"""
    _fields_ = [("iterations", i32), ("converged", i32), ("fit", Fit), ("constraints", Constraints),
                ("time_row", dbl * 7), ("time_schur", dbl)]


class RelocSearch(C.Structure):
    """kb_reloc_search: the hypothesis grid of kb_relocalize"""
    _fields_ = [("center", dbl * 16), ("half_cells_x", i32), ("half_cells_y", i32), ("step", dbl), ("n_yaw", i32),
                ("yaw_step", dbl), ("top_k", i32), ("max_correspondence_distance", dbl), ("kernel_scale", dbl)]


class RelocResult(C.Structure):
    """kb_reloc_result"""
    _fields_ = [("pose", dbl * 16), ("inliers", i32), ("iterations", i32), ("rank", i32), ("n_source", i32),
                ("n_hypotheses", i32), ("n_peaks", i32), ("n_candidates", i32), ("runner_up_pose", dbl * 16),
                ("runner_up_inliers", i32)]


class PlaceParams(C.Structure):
    """kb_place_params: the Scan Context grid"""
    _fields_ = [("n_rings", i32), ("n_sectors", i32), ("max_radius", dbl), ("z_offset", dbl)]


class PlaceMatch(C.Structure):
    """kb_place_match: one candidate of a place query"""
    _fields_ = [("entry", i32), ("shift", i32), ("yaw", dbl), ("distance", dbl), ("guess", dbl * 16)]


class PlaceMatchReport(C.Structure):
    """kb_place_match_report: the counts of a kb_place_db_match"""
    _fields_ = [("queries", sz), ("entries", sz), ("pairs", sz), ("fallbacks", sz), ("chunks", sz)]


class PlaceSearch(C.Structure):
    """kb_place_search: the query and refinement of kb_place_relocalize"""
    _fields_ = [("top_k", i32), ("max_entry", i32), ("separation", dbl), ("max_correspondence_distance", dbl),
                ("kernel_scale", dbl)]


class PlaceResult(C.Structure):
    """kb_place_result"""
    _fields_ = [("pose", dbl * 16), ("inliers", i32), ("iterations", i32), ("rank", i32), ("n_source", i32),
                ("n_entries", i32), ("n_candidates", i32), ("runner_up_pose", dbl * 16), ("runner_up_inliers", i32)]


class PoseGraphOptions(C.Structure):
    """kb_pose_graph_options"""
    _fields_ = [("max_iterations", i32), ("function_tolerance", dbl), ("parameter_tolerance", dbl),
                ("initial_lambda", dbl), ("max_cg_iterations", i32), ("cg_tolerance", dbl)]


class PoseGraphReport(C.Structure):
    """kb_pose_graph_report"""
    _fields_ = [("iterations", i32), ("accepted", i32), ("cg_iterations", i32), ("termination", i32),
                ("initial_cost", dbl), ("final_cost", dbl), ("lambda_", dbl)]


class FreeSpaceParams(C.Structure):
    """kb_free_space_params"""
    _fields_ = [("pass_radius", dbl), ("end_margin", dbl), ("min_incidence", dbl), ("min_planarity", dbl),
                ("min_passes", u32), ("ratio", dbl)]


class FreeSpaceReport(C.Structure):
    """kb_free_space_report"""
    _fields_ = [(f, C.c_ulonglong) for f in ("rays", "scans", "points", "voxels", "points_removed", "voxels_removed",
                                             "ray_point_tests")]


class PlaneAdjustParams(C.Structure):
    """kb_plane_adjust_params"""
    _fields_ = [("voxel_size", dbl), ("min_points", i32), ("planarity", dbl), ("sigma", dbl), ("robust_scale", dbl),
                ("rounds", i32), ("round_tolerance", dbl)]


class PlaneRound(C.Structure):
    """kb_plane_round: one round of kb_pose_graph_adjust_planes"""
    _fields_ = [("planar_pairs", C.c_ulonglong), ("points_used", C.c_ulonglong), ("initial_cost", dbl),
                ("final_cost", dbl), ("final_plane_cost", dbl), ("iterations", i32), ("accepted", i32),
                ("termination", i32), ("max_change", dbl)]


class PlaneAdjustReport(C.Structure):
    """kb_plane_adjust_report"""
    _fields_ = [("rounds", i32), ("converged", i32), ("initial_cost", dbl), ("final_cost", dbl)]


class PoseGraphFactorInfo(C.Structure):
    """kb_pose_graph_factor_info"""
    _fields_ = [("free_nodes", sz), ("h_blocks", sz), ("l_blocks", sz), ("etree_height", sz), ("flops", dbl)]


# every exported symbol of include/kiss_icp_b200.h: name -> (restype, argtypes)
SIGNATURES = {
    "kb_last_error": (C.c_char_p, []),
    "kb_version": (C.c_char_p, []),
    "kb_device_count": (i32, []),
    "kb_set_device": (i32, [i32]),
    "kb_set_stream": (i32, [vp]),
    "kb_set_grid_blocks": (i32, [i32]),
    "kb_map_create": (i32, [dbl, dbl, u32, C.POINTER(vp)]),
    "kb_map_destroy": (i32, [vp]),
    "kb_map_clear": (i32, [vp]),
    "kb_map_empty": (i32, [vp, C.POINTER(i32)]),
    "kb_map_update_origin": (i32, [vp, vp, sz, vp]),
    "kb_map_update_pose": (i32, [vp, vp, sz, vp]),
    "kb_map_add_points": (i32, [vp, vp, sz]),
    "kb_map_remove_far": (i32, [vp, vp]),
    "kb_map_pointcloud": (i32, [vp, vp, sz, C.POINTER(sz)]),
    "kb_map_num_points": (i32, [vp, C.POINTER(sz)]),
    "kb_map_num_voxels": (i32, [vp, C.POINTER(sz)]),
    "kb_map_dump": (i32, [vp, vp, vp, vp, sz, sz, C.POINTER(sz), C.POINTER(sz)]),
    "kb_map_closest_neighbors": (i32, [vp, vp, sz, vp, vp]),
    "kb_map_closest_neighbors_dev": (i32, [vp, vp, sz, vp, vp]),
    "kb_map_compact": (i32, [vp]),
    "kb_map_params": (i32, [vp, C.POINTER(dbl), C.POINTER(dbl), C.POINTER(u32)]),
    "kb_map_query_bytes_dev": (i32, [vp, vp, sz, C.POINTER(dbl)]),
    "kb_map_sync": (i32, [vp]),
    "kb_registration_create": (i32, [i32, dbl, i32, C.POINTER(vp)]),
    "kb_registration_destroy": (i32, [vp]),
    "kb_registration_align_points_to_map": (i32, [vp, vp, sz, vp, vp, dbl, dbl, vp]),
    "kb_registration_last_iterations": (i32, [vp, C.POINTER(i32)]),
    "kb_registration_build_system": (i32, [vp, vp, sz, vp, dbl, dbl, vp, vp, C.POINTER(i32)]),
    "kb_registration_align_batch": (i32, [vp, vp, sz, vp, vp, sz, vp, vp, vp, vp, vp, vp, vp]),
    "kb_registration_align_batch_dev": (i32, [vp, vp, sz, vp, vp, sz, vp, vp, vp, vp, vp, vp, vp]),
    "kb_preprocessor_create": (i32, [dbl, dbl, i32, i32, C.POINTER(vp)]),
    "kb_preprocessor_destroy": (i32, [vp]),
    "kb_preprocessor_preprocess": (i32, [vp, vp, sz, vp, sz, vp, vp, sz, C.POINTER(sz)]),
    "kb_threshold_create": (i32, [dbl, dbl, dbl, C.POINTER(vp)]),
    "kb_threshold_destroy": (i32, [vp]),
    "kb_threshold_compute": (i32, [vp, C.POINTER(dbl)]),
    "kb_threshold_update_model_deviation": (i32, [vp, vp]),
    "kb_voxel_down_sample": (i32, [vp, sz, dbl, vp, sz, C.POINTER(sz)]),
    "kb_correct_kitti_scan": (i32, [vp, sz, vp]),
    "kb_correct_kitti_scan_dev": (i32, [vp, sz, vp]),
    "kb_config_default": (None, [C.POINTER(Config)]),
    "kb_pipeline_create": (i32, [C.POINTER(Config), C.POINTER(vp)]),
    "kb_pipeline_destroy": (i32, [vp]),
    "kb_pipeline_register_frame": (i32, [vp, vp, sz, vp, sz]),
    "kb_pipeline_register_frame_f32": (i32, [vp, vp, sz, vp, sz]),
    "kb_pipeline_register_frame_dev": (i32, [vp, vp, sz, vp, sz]),
    "kb_pipeline_register_frames": (i32, [vp, vp, vp, vp, vp, sz, i32, vp]),
    "kb_pipeline_grow_retries": (i32, [vp, C.POINTER(C.c_ulonglong)]),
    "kb_pipeline_last_cloud_sizes": (i32, [vp, C.POINTER(sz), C.POINTER(sz)]),
    "kb_pipeline_last_clouds": (i32, [vp, vp, sz, vp, sz]),
    "kb_pipeline_voxelize": (i32, [vp, vp, sz, vp, sz, C.POINTER(sz), vp, sz, C.POINTER(sz)]),
    "kb_pipeline_pose": (i32, [vp, vp]),
    "kb_pipeline_delta": (i32, [vp, vp]),
    "kb_pipeline_set_pose": (i32, [vp, vp]),
    "kb_pipeline_set_delta": (i32, [vp, vp]),
    "kb_pipeline_voxel_map": (vp, [vp]),
    "kb_pipeline_last_sigma": (i32, [vp, C.POINTER(dbl)]),
    "kb_pipeline_debug_stamps": (i32, [vp, vp, i32]),
    "kb_pipeline_history_stamps": (i32, [vp, vp, sz, C.POINTER(sz)]),
    "kb_pipeline_history_grid_stamps": (i32, [vp, vp, sz, C.POINTER(sz)]),
    "kb_pipeline_debug_prefetch": (i32, [vp, i32]),
    "kb_debug_icp_solve_fast": (i32, [vp, vp, vp, vp]),
    "kb_debug_icp_schur": (i32, [vp, vp, vp, C.POINTER(i32)]),
    "kb_debug_nn_reuse": (i32, [vp, vp, vp, sz, i32, vp, vp, vp]),
    "kb_debug_icp_solve_dev": (i32, [vp, dbl, sz, vp, vp, vp, vp]),
    "kb_debug_se3_exp_dev": (i32, [vp, sz, vp]),
    "kb_debug_fast_rcp_dev": (i32, [vp, sz, vp]),
    "kb_debug_barrier_ns": (i32, [i32, C.POINTER(dbl)]),
    "kb_pipeline_last_ds_profile": (i32, [vp, vp]),
    "kb_pipeline_last_map_profile": (i32, [vp, vp]),
    "kb_pipeline_last_cache_stats": (i32, [vp, vp]),
    "kb_pipeline_last_icp_work": (i32, [vp, C.POINTER(dbl), C.POINTER(dbl)]),
    "kb_pipeline_threshold": (i32, [vp, C.POINTER(dbl)]),
    "kb_pipeline_last_iterations": (i32, [vp, C.POINTER(i32)]),
    "kb_pipeline_last_profile": (i32, [vp, vp, i32]),
    "kb_pipeline_set_profiling": (i32, [vp, i32]),
    "kb_any_device_stuck": (i32, []),
    "kb_pipeline_set_history": (i32, [vp, sz]),
    "kb_pipeline_get_history": (i32, [vp, vp, sz, C.POINTER(sz)]),
    "kb_pipeline_launch_count": (i32, [vp, C.POINTER(C.c_ulonglong)]),
    "kb_map_load": (i32, [vp, vp, vp, vp, sz, sz]),
    "kb_map_load_dev": (i32, [vp, vp, vp, vp, sz, sz]),
    "kb_pipeline_get_state": (i32, [vp, C.POINTER(PipelineState)]),
    "kb_pipeline_set_state": (i32, [vp, C.POINTER(PipelineState)]),
    "kb_threshold_get_state": (i32, [vp, C.POINTER(dbl), C.POINTER(i32)]),
    "kb_threshold_set_state": (i32, [vp, dbl, i32]),
    "kb_pipeline_create_localizer": (i32, [C.POINTER(Config), vp, C.POINTER(vp)]),
    "kb_map_readers": (i32, [vp, C.POINTER(i32)]),
    "kb_pipeline_last_fit": (i32, [vp, C.POINTER(Fit)]),
    "kb_pipeline_register_frames_fit": (i32, [vp, vp, vp, vp, vp, sz, i32, vp, vp]),
    "kb_pipeline_set_fit_reporting": (i32, [vp, i32]),
    "kb_pipeline_fit_reporting": (i32, [vp, C.POINTER(i32)]),
    "kb_reloc_hypotheses": (i32, [C.POINTER(RelocSearch), vp, sz, C.POINTER(sz)]),
    "kb_relocalize": (i32, [vp, vp, sz, vp, C.POINTER(RelocSearch), C.POINTER(RelocResult), vp, vp, vp]),
    "kb_debug_reloc_score_ms": (i32, [vp, C.POINTER(C.c_float)]),
    "kb_registration_constraints": (i32, [vp, vp, sz, vp, vp, dbl, C.POINTER(Constraints)]),
    "kb_pipeline_set_constraint_reporting": (i32, [vp, i32]),
    "kb_pipeline_last_constraints": (i32, [vp, C.POINTER(Constraints)]),
    "kb_pipeline_register_frames_constraints": (i32, [vp, vp, vp, vp, vp, sz, i32, vp, vp, vp]),
    "kb_debug_sym3_eig": (i32, [vp, vp, vp]),
    "kb_pipeline_set_degeneracy_ratio": (i32, [vp, dbl]),
    "kb_pipeline_degeneracy_ratio": (i32, [vp, C.POINTER(dbl)]),
    "kb_pipeline_last_degeneracy": (i32, [vp, C.POINTER(Degeneracy)]),
    "kb_pipeline_register_frames_degeneracy": (i32, [vp, vp, vp, vp, vp, sz, i32, vp, vp, vp, vp]),
    "kb_motion_check": (i32, [C.POINTER(Motion)]),
    "kb_pipeline_register_frames_motion": (i32, [vp, vp, vp, vp, vp, vp, sz, i32, vp, vp, vp, vp]),
    "kb_pipeline_motion_time": (i32, [vp, C.POINTER(dbl)]),
    "kb_pipeline_set_motion_time": (i32, [vp, dbl]),
    "kb_deskew_motion": (i32, [vp, sz, vp, sz, C.POINTER(Motion), vp]),
    "kb_rig_check": (i32, [vp, sz]),
    "kb_pipeline_register_rig_frames": (i32, [vp, vp, sz, vp, vp, vp, vp, vp, vp, sz, i32, vp, vp, vp, vp]),
    "kb_merge_rig": (i32, [vp, sz, vp, vp, vp, vp, vp, vp, vp, vp]),
    "kb_calibrate_rig": (i32, [vp, vp, sz, vp, sz, vp, vp, vp, i32, C.POINTER(RigCalibrationOptions), vp,
                               vp]),
    "kb_calibrate_rig_clocks": (i32, [vp, C.POINTER(Motion), vp, sz, vp, vp, vp, vp, vp, vp, vp, vp, sz, i32,
                                      C.POINTER(RigClockCalibrationOptions), vp, vp, vp]),
    "kb_place_params_default": (None, [C.POINTER(PlaceParams)]),
    "kb_place_db_create": (i32, [C.POINTER(PlaceParams), C.POINTER(vp)]),
    "kb_place_db_destroy": (i32, [vp]),
    "kb_place_db_size": (i32, [vp, C.POINTER(sz)]),
    "kb_place_descriptor": (i32, [vp, vp, sz, vp]),
    "kb_place_db_add": (i32, [vp, vp, sz, vp, C.POINTER(sz)]),
    "kb_place_db_dump": (i32, [vp, vp, vp, sz, C.POINTER(sz)]),
    "kb_place_db_load": (i32, [vp, vp, vp, sz]),
    "kb_place_query": (i32, [vp, vp, sz, i32, dbl, i32, vp, C.POINTER(sz), vp, vp]),
    "kb_place_relocalize": (i32, [vp, vp, vp, sz, vp, sz, vp, C.POINTER(PlaceSearch), C.POINTER(PlaceResult), vp]),
    "kb_debug_place_distance_ms": (i32, [vp, C.POINTER(C.c_float)]),
    "kb_place_db_match": (i32, [vp, vp, vp, dbl, i32, vp, vp, C.POINTER(PlaceMatchReport)]),
    "kb_debug_place_match_ms": (i32, [vp, vp]),
    "kb_debug_place_match_chunk": (i32, [sz]),
    "kb_debug_place_match_pairs": (i32, [vp, vp, vp, vp]),
    "kb_pose_graph_create": (i32, [C.POINTER(vp)]),
    "kb_pose_graph_destroy": (i32, [vp]),
    "kb_pose_graph_add_node": (i32, [vp, vp, i32, C.POINTER(sz)]),
    "kb_pose_graph_add_edge": (i32, [vp, sz, sz, vp, vp, dbl, C.POINTER(sz)]),
    "kb_pose_graph_add_pose_prior": (i32, [vp, sz, vp, vp, dbl, C.POINTER(sz)]),
    "kb_pose_graph_add_position_prior": (i32, [vp, sz, vp, vp, vp, dbl, C.POINTER(sz)]),
    "kb_pose_graph_num_priors": (i32, [vp, C.POINTER(sz)]),
    "kb_pose_graph_prior_chi2": (i32, [vp, vp, vp, sz, C.POINTER(sz)]),
    "kb_pose_graph_size": (i32, [vp, C.POINTER(sz), C.POINTER(sz)]),
    "kb_pose_graph_poses": (i32, [vp, vp, sz, C.POINTER(sz)]),
    "kb_pose_graph_options_default": (None, [C.POINTER(PoseGraphOptions)]),
    "kb_pose_graph_optimize": (i32, [vp, C.POINTER(PoseGraphOptions), C.POINTER(PoseGraphReport), vp, vp]),
    "kb_pose_graph_optimize_direct": (i32, [vp, C.POINTER(PoseGraphOptions), C.POINTER(PoseGraphReport), vp, vp]),
    "kb_debug_pose_graph_ms": (i32, [vp, C.POINTER(C.c_float)]),
    "kb_debug_se3_adjoint": (i32, [vp, vp]),
    "kb_debug_se3_right_jacobian_inverse": (i32, [vp, vp]),
    "kb_pose_graph_marginals": (i32, [vp, vp, sz, vp]),
    "kb_pose_graph_joint_marginals": (i32, [vp, vp, sz, vp]),
    "kb_pose_graph_factor_info": (i32, [vp, C.POINTER(PoseGraphFactorInfo)]),
    "kb_debug_pose_graph_symbolic": (i32, [vp, sz, C.POINTER(sz), vp, vp, vp]),
    "kb_debug_pose_graph_rows": (i32, [vp, sz, C.POINTER(sz), vp, vp]),
    "kb_debug_pose_graph_cov_ms": (i32, [vp, vp]),
    "kb_plane_adjust_params_default": (None, [C.POINTER(PlaneAdjustParams), dbl]),
    "kb_pose_graph_adjust_planes": (i32, [vp, vp, sz, vp, C.POINTER(PlaneAdjustParams), C.POINTER(PoseGraphOptions),
                                          C.POINTER(PlaneAdjustReport), vp, sz, vp, vp]),
    "kb_debug_pose_graph_plane_ms": (i32, [vp, vp]),
    "kb_debug_pose_graph_plane_terms": (i32, [vp, vp, sz, vp, C.POINTER(PlaneAdjustParams), vp, vp, vp, vp]),
    "kb_free_space_params_default": (None, [C.POINTER(FreeSpaceParams), dbl]),
    "kb_map_free_space": (i32, [vp, vp, sz, vp, sz, vp, C.POINTER(FreeSpaceParams), vp, vp, vp,
                                C.POINTER(FreeSpaceReport)]),
    "kb_debug_free_space_bin_size": (i32, [dbl]),
    "kb_debug_free_space_ms": (i32, [vp]),
}


def lib():
    """Load the CUDA library. Fails loudly if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). kiss_icp_b200 has no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
        atexit.register(_exit_without_teardown_if_stuck)
    return _lib


def _exit_without_teardown_if_stuck():
    """A launch that never ended (reported as an error by the call that waited for it) would block the CUDA context's
    teardown at interpreter exit forever: leave without it."""
    if _lib is not None and _lib.kb_any_device_stuck():
        import sys
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(1)


def check(status: int):
    if status == KB_OK:
        return
    msg = lib().kb_last_error().decode()
    if status == KB_ERR_NO_DEVICE:
        raise NoDeviceError(msg)
    if status == KB_ERR_OUT_OF_RANGE:
        raise IndexError(msg)  # pybind11 maps std::out_of_range to IndexError
    if status == KB_ERR_NOT_SE3:
        raise ValueError(msg)
    raise KissB200Error(f"kb_status {status}: {msg}")


def points_arg(points) -> np.ndarray:
    """ndarray (N,3) float64 C-contiguous, as py_array_to_vectors_double does
    (python/kiss_icp/pybind/stl_vector_eigen.h:67-80: c_style | forcecast, else cast_error)."""
    a = np.asarray(points)
    if a.ndim != 2 or a.shape[1] != 3:
        raise RuntimeError("Unable to cast Python instance to C++ type (expected an (N, 3) array)")
    return np.ascontiguousarray(a, dtype=np.float64)


def mat4_arg(T) -> np.ndarray:
    a = np.ascontiguousarray(T, dtype=np.float64)
    if a.shape != (4, 4):
        raise RuntimeError("Unable to cast Python instance to C++ type (expected a (4, 4) array)")
    return a


def ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)
