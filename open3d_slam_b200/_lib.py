"""ctypes binding of the C ABI in include/b2s.h (open3d_slam_b200/libb2s.so).

The CUDA library is the only implementation: if it is missing or no GPU is visible the calls fail loudly
(there is no CPU fallback and nothing here imports oracle/).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2S_LIB") or os.path.join(_HERE, "libb2s.so")   # B2S_LIB: an A/B build of the same library (tuning aid)

OK, E_INVALID, E_CUDA, E_EMPTY, E_NO_NORMALS, E_CAPACITY, E_UNSUPPORTED = 0, -1, -2, -3, -4, -5, -6
CROP_NONE, CROP_MAX_RADIUS, CROP_MIN_RADIUS, CROP_MINMAX_RADIUS, CROP_CYLINDER = 0, 1, 2, 3, 4
CROPPER_NAMES = {"None": 0, "MaxRadius": 1, "MinRadius": 2, "MinMaxRadius": 3, "Cylinder": 4}  # croppers.hpp cropperNames
REG_POINT_TO_PLANE, REG_POINT_TO_POINT, REG_GENERALIZED = 0, 1, 2


class Cropper(C.Structure):
    _fields_ = [("kind", C.c_int32), ("invert", C.c_int32), ("rmin", C.c_double), ("rmax", C.c_double),
                ("zmin", C.c_double), ("zmax", C.c_double), ("center", C.c_double * 3)]


class IcpParams(C.Structure):
    _fields_ = [("reg_type", C.c_int32), ("max_iter", C.c_int32), ("max_corr_dist", C.c_double), ("knn", C.c_int32),
                ("knn_radius", C.c_double), ("rel_fitness", C.c_double), ("rel_rmse", C.c_double)]


class ScanParams(C.Structure):
    _fields_ = [("voxel_size", C.c_double), ("downsampling_ratio", C.c_double), ("seed", C.c_uint32),
                ("map_builder_cropper", Cropper), ("scan_matcher_cropper", Cropper)]


class Config(C.Structure):
    _fields_ = [("icp", IcpParams), ("scan", ScanParams), ("map_voxel_size", C.c_double), ("dense_voxel_size", C.c_double),
                ("nn_cell_size", C.c_double), ("icp_cluster_ctas", C.c_int32), ("reserved_", C.c_int32)]


class Result(C.Structure):
    _fields_ = [("T", C.c_double * 16), ("fitness", C.c_double), ("inlier_rmse", C.c_double), ("n_corr", C.c_int32),
                ("iters", C.c_int32)]


class CarvingParams(C.Structure):
    _fields_ = [("voxel_size", C.c_double), ("max_raytracing_length", C.c_double), ("truncation_distance", C.c_double),
                ("min_dot_product_with_normal", C.c_double), ("neighborhood_radius_dense_map", C.c_double)]


class MapperOptions(C.Structure):
    _fields_ = [("min_movement_between_mapping_steps", C.c_double), ("carve_enabled", C.c_int32), ("carve_every_n_scans", C.c_int32),
                ("carving", CarvingParams), ("dense_enabled", C.c_int32), ("dense_carve_every_n_scans", C.c_int32),
                ("dense_carving", CarvingParams), ("dense_cropper", Cropper)]


class FeatureParams(C.Structure):
    _fields_ = [("feature_voxel_size", C.c_double), ("normal_estimation_radius", C.c_double), ("normal_knn", C.c_int32),
                ("feature_radius", C.c_double), ("feature_knn", C.c_int32)]


class RansacParams(C.Structure):
    _fields_ = [("mutual_filter", C.c_int32), ("ransac_n", C.c_int32), ("max_correspondence_distance", C.c_double),
                ("checker_distance", C.c_double), ("checker_edge_length", C.c_double), ("max_iteration", C.c_int64),
                ("confidence", C.c_double), ("seed", C.c_uint64)]


class RansacResult(C.Structure):
    _fields_ = [("result", Result), ("hypotheses", C.c_int64), ("validations", C.c_int64), ("best_hypothesis", C.c_int64), ("n_feature_corr", C.c_int32),
                ("used_mutual", C.c_int32)]


class OdometryParams(C.Structure):
    _fields_ = [("icp", IcpParams), ("voxel_size", C.c_double), ("downsampling_ratio", C.c_double), ("seed", C.c_uint32), ("cropper", Cropper),
                ("min_fitness", C.c_double), ("buffer_size", C.c_int32)]


class OdometryResult(C.Structure):
    _fields_ = [("registration", Result), ("odom_to_range_sensor", C.c_double * 16), ("outcome", C.c_int32), ("n_preprocessed", C.c_int32)]


class SlamResult(C.Structure):
    _fields_ = [("odometry", OdometryResult), ("mapper", Result), ("odom_used", C.c_int32), ("mapper_accepted", C.c_int32)]


class MotionCompensationParams(C.Structure):
    _fields_ = [("enabled", C.c_int32), ("spinning_clockwise", C.c_int32), ("scan_duration", C.c_double),
                ("num_poses_velocity_estimation", C.c_int32)]


class MotionCompensationResult(C.Structure):
    _fields_ = [("odometry_linear_velocity", C.c_double * 3), ("odometry_angular_velocity_rpy", C.c_double * 3),
                ("map_linear_velocity", C.c_double * 3), ("map_angular_velocity_rpy", C.c_double * 3),
                ("odometry_applied", C.c_int32), ("map_applied", C.c_int32)]


ODOM_INIT, ODOM_OK, ODOM_FAILED, ODOM_FAILED_KEPT_PREV = 0, 1, 2, 3


class OdometryConstraintParams(C.Structure):
    _fields_ = [("map_voxel_size", C.c_double), ("voxel_if_zero", C.c_double), ("overlap_factor", C.c_double), ("icp_factor", C.c_double),
                ("min_points_per_voxel", C.c_int32), ("refine", C.c_int32), ("max_iter", C.c_int32), ("rel_fitness", C.c_double),
                ("rel_rmse", C.c_double)]


class OdometryConstraint(C.Structure):
    _fields_ = [("T", C.c_double * 16), ("information", C.c_double * 36), ("n_source_overlap", C.c_int64), ("n_target_overlap", C.c_int64),
                ("refined", C.c_int32), ("icp", Result)]


class PoseGraphEdge(C.Structure):
    _fields_ = [("source", C.c_int32), ("target", C.c_int32), ("uncertain", C.c_int32), ("reserved_", C.c_int32), ("T", C.c_double * 16),
                ("information", C.c_double * 36)]


class GlobalOptimizationParams(C.Structure):
    _fields_ = [("max_correspondence_distance", C.c_double), ("edge_prune_threshold", C.c_double), ("preference_loop_closure", C.c_double),
                ("reference_node", C.c_int32), ("max_iteration", C.c_int32), ("min_relative_increment", C.c_double),
                ("min_relative_residual_increment", C.c_double), ("min_right_term", C.c_double), ("min_residual", C.c_double),
                ("max_iteration_lm", C.c_int32), ("reserved_", C.c_int32), ("upper_scale_factor", C.c_double), ("lower_scale_factor", C.c_double)]


class GlobalOptimizationStats(C.Structure):
    _fields_ = [("valid", C.c_int32), ("n_edges", C.c_int32), ("outer_iterations", C.c_int32), ("lm_tries", C.c_int32), ("accepted_steps", C.c_int32),
                ("stop_reason", C.c_int32), ("initial_residual", C.c_double), ("final_residual", C.c_double), ("final_lambda", C.c_double)]


# b2s_global_optimization_stats.stop_reason (B2S_LM_STOP_*)
LM_STOP_REASONS = ["none", "right_term", "relative_increment", "relative_residual_increment", "max_iteration_lm", "residual", "max_iteration"]


class MapperCounters(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("steps", "accepted", "inserted_map", "inserted_dense", "carve_runs", "carved_points_total",
                                         "dense_carve_runs", "carved_voxels_total")]


# every symbol include/b2s.h declares (checked by tests/test_abi.py without needing a GPU)
SYMBOLS = [
    "b2s_default_config", "b2s_create", "b2s_destroy", "b2s_set_config", "b2s_synchronize", "b2s_last_error", "b2s_version",
    "b2s_device_count", "b2s_launch_count", "b2s_graph_capture_count", "b2s_cloud_create", "b2s_cloud_destroy", "b2s_cloud_upload_f64", "b2s_cloud_upload_f32",
    "b2s_cloud_size", "b2s_cloud_download", "b2s_cloud_copy", "b2s_crop", "b2s_voxel_down_sample", "b2s_estimate_normals",
    "b2s_random_down_sample", "b2s_transform", "b2s_process_scan", "b2s_register", "b2s_register_batch", "b2s_register_host",
    "b2s_submap_create", "b2s_submap_destroy", "b2s_submap_insert", "b2s_submap_insert_dense", "b2s_submap_size", "b2s_submap_download",
    "b2s_submap_dense_download", "b2s_submap_set_cloud", "b2s_register_to_submap", "b2s_submap_set_pose", "b2s_submap_get_pose",
    "b2s_mapper_step_async", "b2s_scan_result_fetch", "b2s_profile_enable", "b2s_profile_read", "b2s_mapper_graph_enable", "b2s_debug_icp_clocks",
    "b2s_mapper_step_host", "b2s_mapper_step_host_async", "b2s_submap_carve", "b2s_overlap", "b2s_information_matrix", "b2s_undistort",
    "b2s_dense_query", "b2s_dense_remove", "b2s_dense_size", "b2s_dense_clear", "b2s_dense_carve", "b2s_submap_transform",
    "b2s_default_mapper_options", "b2s_submap_set_mapper_options", "b2s_submap_get_mapper_counters",
    "b2s_voxel_map_create", "b2s_voxel_map_destroy", "b2s_voxel_map_clear", "b2s_voxel_map_insert_cloud", "b2s_voxel_map_size",
    "b2s_voxel_map_has_voxel", "b2s_voxel_map_indices_in_voxel", "b2s_mapper_processed_scan",
    "b2s_cloud_export_device", "b2s_cloud_import_device", "b2s_submap_to_cloud", "b2s_nearest_neighbors",
    "b2s_feature_create", "b2s_feature_destroy", "b2s_feature_size", "b2s_feature_download", "b2s_feature_upload", "b2s_compute_fpfh",
    "b2s_default_feature_params", "b2s_submap_compute_features",
    "b2s_default_ransac_params", "b2s_ransac_feature_matching", "b2s_feature_correspondences",
    "b2s_default_odometry_params", "b2s_odometry_create", "b2s_odometry_destroy", "b2s_odometry_set_params", "b2s_odometry_set_initial_transform",
    "b2s_odometry_step_async", "b2s_odometry_result_fetch", "b2s_odometry_lookup", "b2s_odometry_preprocessed",
    "b2s_slam_step_async", "b2s_slam_result_fetch", "b2s_slam_step_host_async", "b2s_slam_graph_enable",
    "b2s_default_motion_compensation_params", "b2s_odometry_set_motion_compensation", "b2s_slam_map_pose_push", "b2s_slam_map_lookup",
    "b2s_slam_motion_fetch", "b2s_slam_undistorted",
    "b2s_default_odometry_constraint_params", "b2s_submap_odometry_constraints",
    "b2s_default_global_optimization_params", "b2s_global_optimization", "b2s_cloud_transform_inplace",
    "b2s_submap_set_initial_map", "b2s_submap_set_initial_transform", "b2s_submap_set_merge_scans", "b2s_debug_nn_index",
]
FEATURE_DIM, FEATURE_MAX_KNN = 33, 128   # B2S_FEATURE_DIM, B2S_FEATURE_MAX_KNN
PROFILE_KINDS = ["icp", "normals", "radix_sort", "nn_grid_build", "voxel", "fuse", "select", "crop"]

_lib = None


class B2SError(RuntimeError):
    """Mirrors the std::runtime_error the reference throws from assert_* / Open3D LogError."""

    def __init__(self, code, msg):
        super().__init__(f"b2s error {code}: {msg}")
        self.code = code


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: build it with __graft_entry__.build() (nvcc, sm_90a). "
                              "There is no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        L.b2s_last_error.restype = C.c_char_p
        L.b2s_version.restype = C.c_char_p
        L.b2s_launch_count.restype = C.c_int64
        L.b2s_launch_count.argtypes = [C.c_void_p]
        L.b2s_graph_capture_count.restype = C.c_int64
        L.b2s_graph_capture_count.argtypes = [C.c_void_p]
        L.b2s_destroy.restype = None
        L.b2s_cloud_destroy.restype = None
        L.b2s_submap_destroy.restype = None
        L.b2s_default_config.restype = None
        L.b2s_default_mapper_options.restype = None
        L.b2s_default_feature_params.restype = None
        L.b2s_default_ransac_params.restype = None
        L.b2s_destroy.argtypes = [C.c_void_p]
        L.b2s_cloud_destroy.argtypes = [C.c_void_p]
        L.b2s_submap_destroy.argtypes = [C.c_void_p]
        L.b2s_voxel_map_destroy.restype = None
        L.b2s_voxel_map_destroy.argtypes = [C.c_void_p]
        L.b2s_feature_destroy.restype = None
        L.b2s_feature_destroy.argtypes = [C.c_void_p]
        L.b2s_odometry_destroy.restype = None
        L.b2s_odometry_destroy.argtypes = [C.c_void_p]
        L.b2s_default_odometry_params.restype = None
        L.b2s_default_motion_compensation_params.restype = None
        L.b2s_default_odometry_constraint_params.restype = None
        L.b2s_default_global_optimization_params.restype = None
        _lib = L
    return _lib


def check(code):
    if code != OK:
        raise B2SError(code, lib().b2s_last_error().decode("utf-8", "replace"))
