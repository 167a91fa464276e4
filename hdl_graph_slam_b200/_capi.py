"""ctypes binding of libb200reg.so (include/b200reg.h).  Loading fails loudly: there is no Python/CPU fallback."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# B2R_LIB selects an A/B build variant of the same ABI (tools/build_variant.sh); the product library is the default
LIB_PATH = os.environ.get("B2R_LIB") or os.path.join(_HERE, "_lib", "libb200reg.so")

B2R_OK = 0
B2R_EINVAL, B2R_ENODEVICE, B2R_ECUDA, B2R_ESTATE, B2R_EUNSUPPORTED, B2R_ENCCL = -1, -2, -3, -4, -5, -6
B2R_METHOD_GICP, B2R_METHOD_NDT, B2R_METHOD_NDT_PCL, B2R_METHOD_VGICP, B2R_METHOD_GICP_PCL, B2R_METHOD_ICP_PCL, B2R_METHOD_VGICP_CUDA, B2R_METHOD_GICP_OMP, B2R_METHOD_NDT_KDTREE = 0, 1, 2, 3, 4, 5, 6, 8, 9  # 7 is unassigned
B2R_DOWNSAMPLE_NONE, B2R_DOWNSAMPLE_VOXELGRID, B2R_DOWNSAMPLE_APPROX_VOXELGRID = 0, 1, 2
FLOOR_REASONS = ("OK", "EMPTY_INPUT", "TOO_FEW_FILTERED", "NO_MODEL", "TOO_FEW_INLIERS", "NOT_VERTICAL")  # B2R_FLOOR_* codes 0..5


class Config(C.Structure):
    _fields_ = [
        ("method", C.c_int32), ("device_id", C.c_int32), ("max_iterations", C.c_int32), ("k_correspondences", C.c_int32),
        ("transformation_epsilon", C.c_double), ("rotation_epsilon", C.c_double), ("max_correspondence_distance", C.c_double),
        ("ndt_resolution", C.c_double), ("ndt_step_size", C.c_double), ("ndt_outlier_ratio", C.c_double),
        ("ndt_search_method", C.c_int32), ("ndt_mt_interval_flag", C.c_int32), ("ndt_fixed_iterations", C.c_int32),
        ("grid_cell_min", C.c_float), ("max_optimizer_iterations", C.c_int32), ("use_reciprocal_correspondences", C.c_int32),
    ]


class Result(C.Structure):
    _fields_ = [("T", C.c_float * 16), ("fitness", C.c_double), ("converged", C.c_int32), ("iterations", C.c_int32)]


class Pair(C.Structure):
    _fields_ = [("source", C.c_int32), ("target", C.c_int32), ("guess", C.c_float * 16)]


class InformationParams(C.Structure):
    _fields_ = [("use_const_inf_matrix", C.c_int32), ("reserved", C.c_int32), ("const_stddev_x", C.c_double), ("const_stddev_q", C.c_double),
                ("var_gain_a", C.c_double), ("min_stddev_x", C.c_double), ("max_stddev_x", C.c_double), ("min_stddev_q", C.c_double),
                ("max_stddev_q", C.c_double), ("fitness_score_thresh", C.c_double)]


class PrefilterParams(C.Structure):
    _fields_ = [("deskewing", C.c_int32), ("use_base_link_transform", C.c_int32), ("scan_period", C.c_double), ("angular_velocity", C.c_float * 3),
                ("base_link_transform", C.c_float * 16), ("use_distance_filter", C.c_int32), ("distance_near_thresh", C.c_double),
                ("distance_far_thresh", C.c_double), ("downsample_method", C.c_int32), ("downsample_resolution", C.c_float),
                ("outlier_removal_method", C.c_int32), ("statistical_mean_k", C.c_int32), ("statistical_stddev", C.c_double),
                ("radius_radius", C.c_double), ("radius_min_neighbors", C.c_int32), ("reserved", C.c_int32)]


class FloorParams(C.Structure):
    _fields_ = [("tilt_deg", C.c_double), ("sensor_height", C.c_double), ("height_clip_range", C.c_double), ("floor_pts_thresh", C.c_int32),
                ("use_normal_filtering", C.c_int32), ("floor_normal_thresh", C.c_double), ("normal_filter_thresh", C.c_double)]


class FloorResult(C.Structure):
    _fields_ = [("detected", C.c_int32), ("reason", C.c_int32), ("coeffs", C.c_float * 4), ("n_filtered", C.c_uint64), ("n_inliers", C.c_uint64),
                ("ransac_iterations", C.c_int32), ("model_indices", C.c_int32 * 3), ("ransac_batches", C.c_int32), ("ransac_hypotheses", C.c_int32),
                ("readbacks", C.c_int32), ("reserved", C.c_int32)]


class KeyframeSnapshot(C.Structure):
    _fields_ = [("points", C.c_void_p), ("n", C.c_size_t), ("pose", C.c_float * 16)]


class PointLayout(C.Structure):
    _fields_ = [("point_step", C.c_uint32), ("off_x", C.c_uint32), ("off_y", C.c_uint32), ("off_z", C.c_uint32), ("off_intensity", C.c_uint32),
                ("intensity_datatype", C.c_uint32), ("is_bigendian", C.c_uint32)]


class LoopParams(C.Structure):
    _fields_ = [("distance_thresh", C.c_double), ("accum_distance_thresh", C.c_double), ("min_edge_interval", C.c_double),
                ("fitness_score_max_range", C.c_double), ("fitness_score_thresh", C.c_double)]


class KeyframeState(C.Structure):
    _fields_ = [("accum_distance", C.c_double), ("estimate", C.c_double * 16)]


class OdometryParams(C.Structure):
    _fields_ = [
        ("keyframe_delta_trans", C.c_double), ("keyframe_delta_angle", C.c_double), ("keyframe_delta_time", C.c_double),
        ("transform_thresholding", C.c_int32), ("max_acceptable_trans", C.c_double), ("max_acceptable_angle", C.c_double),
        ("publish_status", C.c_int32), ("downsample_method", C.c_int32), ("downsample_resolution", C.c_float),
    ]


class OdometryStatus(C.Structure):
    _fields_ = [
        ("odom", C.c_float * 16), ("trans", C.c_float * 16), ("converged", C.c_int32), ("iterations", C.c_int32),
        ("keyframe_updated", C.c_int32), ("frame_rejected", C.c_int32), ("matching_error", C.c_double),
        ("inlier_fraction", C.c_float), ("reserved", C.c_int32),
    ]


class Stats(C.Structure):
    _fields_ = [("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("n_classes", C.c_int32), ("reserved", C.c_int32),
                ("launches", C.c_uint64 * 16), ("calls", C.c_uint64 * 16), ("ms", C.c_double * 16)]


# every symbol include/b200reg.h declares: (name, restype, argtypes)
_VP, _SZ, _I32P, _F32P, _F64P = C.c_void_p, C.c_size_t, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_double)
SYMBOLS = [
    ("b2r_last_error", C.c_char_p, []),
    ("b2r_version", C.c_char_p, []),
    ("b2r_config_default", C.c_int, [C.POINTER(Config), C.c_int]),
    ("b2r_select_registration_method", C.c_int, [C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.c_int, C.c_int, C.POINTER(_VP)]),
    ("b2r_create", C.c_int, [C.POINTER(Config), C.POINTER(_VP)]),
    ("b2r_destroy", None, [_VP]),
    ("b2r_get_config", C.c_int, [_VP, C.POINTER(Config)]),
    ("b2r_set_target", C.c_int, [_VP, _VP, _SZ, _SZ]),
    ("b2r_set_source", C.c_int, [_VP, _VP, _SZ, _SZ]),
    ("b2r_set_target_device", C.c_int, [_VP, _VP, _SZ, _SZ]),
    ("b2r_set_source_device", C.c_int, [_VP, _VP, _SZ, _SZ]),
    ("b2r_promote_source_to_target", C.c_int, [_VP]),
    ("b2r_prefetch_source", C.c_int, [_VP, _VP, _SZ, _SZ]),
    ("b2r_prefetch_source_device", C.c_int, [_VP, _VP, _SZ, _SZ]),
    ("b2r_odometry_prefetch", C.c_int, [_VP, _VP, _SZ, _SZ, C.c_int]),
    ("b2r_synchronize", C.c_int, [_VP]),
    ("b2r_set_profiling", C.c_int, [_VP, C.c_int]),
    ("b2r_get_stats", C.c_int, [_VP, C.POINTER(Stats), C.c_int]),
    ("b2r_kernel_class_name", C.c_char_p, [C.c_int]),
    ("b2r_get_stream", C.c_int, [_VP, C.POINTER(_VP)]),
    ("b2r_align", C.c_int, [_VP, _F32P, C.POINTER(Result)]),
    ("b2r_get_aligned", C.c_int, [_VP, _VP, _SZ, _SZ]),
    ("b2r_fitness", C.c_int, [_VP, _F32P, C.c_double, C.c_float, _F64P, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    ("b2r_target_nearest", C.c_int, [_VP, _VP, _SZ, _SZ, _I32P, _F32P]),
    ("b2r_get_correspondences", C.c_int, [_VP, _I32P, _SZ]),
    ("b2r_get_covariances", C.c_int, [_VP, C.c_int, _F64P, _SZ]),
    ("b2r_gicp_linearize_at", C.c_int, [_VP, _F64P, _F64P, _F64P, _F64P]),
    ("b2r_gicp_error_at", C.c_int, [_VP, _F64P, _F64P]),
    ("b2r_ndt_get_voxels", C.c_int, [_VP, _SZ, C.POINTER(_SZ), C.POINTER(C.c_int64), _I32P, _F64P, _F64P, _I32P, _I32P]),
    ("b2r_ndt_derivatives_at", C.c_int, [_VP, _F64P, _F64P, _F64P, _F64P, C.POINTER(C.c_uint64)]),
    ("b2r_ndt_hessian_at", C.c_int, [_VP, _F64P, _F64P]),
    ("b2r_ndt_get_centroids", C.c_int, [_VP, _SZ, C.POINTER(_SZ), C.POINTER(C.c_int64), _F32P]),
    ("b2r_ndt_neighbors_at", C.c_int, [_VP, _F64P, C.POINTER(C.c_uint32), _SZ, C.POINTER(C.c_int64), C.POINTER(_SZ)]),
    ("b2r_vgicp_get_voxels", C.c_int, [_VP, _SZ, C.POINTER(_SZ), C.POINTER(C.c_int32), C.POINTER(C.c_int32), _F64P, _F64P]),
    ("b2r_vgicp_linearize_at", C.c_int, [_VP, _F64P, _F64P, _F64P, _F64P, C.POINTER(C.c_uint64), C.POINTER(C.c_int32), _SZ]),
    ("b2r_gicp_pcl_correspondences_at", C.c_int, [_VP, _F32P, _F32P, C.POINTER(C.c_int32), _F64P, C.POINTER(C.c_uint64)]),
    ("b2r_gicp_pcl_cost_at", C.c_int, [_VP, _F32P, _F64P, _F64P, _F64P]),
    ("b2r_icp_pcl_correspondences_at", C.c_int, [_VP, _F32P, _I32P, _F32P, C.POINTER(C.c_uint64)]),
    ("b2r_icp_pcl_estimate_at", C.c_int, [_VP, _F32P, _F32P, _F64P]),
    ("b2r_voxelgrid", C.c_int, [_VP, _VP, _SZ, _SZ, C.c_float, _VP, C.POINTER(_SZ), _I32P, _I32P]),
    ("b2r_voxelgrid_device", C.c_int, [_VP, _VP, _SZ, _SZ, C.c_float, C.POINTER(_VP), C.POINTER(_SZ)]),
    ("b2r_approximate_voxelgrid", C.c_int, [_VP, _VP, _SZ, _SZ, C.c_float, _VP, C.POINTER(_SZ), _I32P]),
    ("b2r_approximate_voxelgrid_device", C.c_int, [_VP, _VP, _SZ, _SZ, C.c_float, C.POINTER(_VP), C.POINTER(_SZ)]),
    ("b2r_distance_filter", C.c_int, [_VP, _VP, _SZ, _SZ, C.c_double, C.c_double, _VP, C.POINTER(_SZ)]),
    ("b2r_radius_outlier_removal", C.c_int, [_VP, _VP, _SZ, _SZ, C.c_double, C.c_int, _VP, C.POINTER(_SZ)]),
    ("b2r_statistical_outlier_removal", C.c_int, [_VP, _VP, _SZ, _SZ, C.c_int, C.c_double, _VP, C.POINTER(_SZ)]),
    ("b2r_deskew", C.c_int, [_VP, _VP, _SZ, _SZ, C.c_double, _F32P, _VP]),
    ("b2r_prefilter_params_default", C.c_int, [C.POINTER(PrefilterParams)]),
    ("b2r_prefilter", C.c_int, [_VP, _VP, _SZ, _SZ, C.c_int, C.POINTER(PrefilterParams), _VP, C.POINTER(_VP), C.POINTER(_SZ)]),
    ("b2r_floor_params_default", C.c_int, [C.POINTER(FloorParams)]),
    ("b2r_floor_detect", C.c_int, [_VP, _VP, _SZ, _SZ, C.c_int, C.POINTER(FloorParams), C.POINTER(FloorResult), _VP, _VP, C.POINTER(_VP), C.POINTER(_VP)]),
    ("b2r_ingest_pointcloud2", C.c_int, [_VP, _VP, _SZ, C.POINTER(PointLayout), C.POINTER(_VP)]),
    ("b2r_ingest_pointcloud2_rows", C.c_int, [_VP, _VP, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(PointLayout), C.POINTER(_VP)]),
    ("b2r_pcd_read_header", C.c_int, [C.c_char_p, C.POINTER(PointLayout), C.POINTER(_SZ), C.POINTER(_SZ)]),
    ("b2r_ingest_pcd", C.c_int, [_VP, C.c_char_p, C.POINTER(_VP), C.POINTER(_SZ)]),
    ("b2r_map_cloud_generate", C.c_int, [_VP, C.POINTER(KeyframeSnapshot), _SZ, _SZ, C.c_double, _VP, _SZ, C.POINTER(_SZ)]),
    ("b2r_odometry_create", C.c_int, [_VP, C.POINTER(OdometryParams), C.POINTER(_VP)]),
    ("b2r_odometry_destroy", None, [_VP]),
    ("b2r_odometry_matching", C.c_int, [_VP, C.c_double, _VP, _SZ, _SZ, _F32P, C.POINTER(OdometryStatus)]),
    ("b2r_odometry_matching_device", C.c_int, [_VP, C.c_double, _VP, _SZ, _SZ, _F32P, C.POINTER(OdometryStatus)]),
    ("b2r_odometry_matching_ros", C.c_int, [_VP, C.c_uint32, C.c_uint32, _VP, _SZ, _SZ, C.c_int, _F32P, C.c_int, C.POINTER(OdometryStatus)]),
    ("b2r_odometry_aligned", C.c_int, [_VP, C.c_int, _VP, _SZ, _SZ]),
    ("b2r_loop_matching", C.c_int, [_VP, _VP, _SZ, _SZ, C.POINTER(_VP), C.POINTER(_SZ), _SZ, _F32P, C.c_double, C.c_double,
                                    C.POINTER(Result), _I32P]),
    ("b2r_batch_create", C.c_int, [C.POINTER(Config), C.POINTER(_VP)]),
    ("b2r_batch_destroy", None, [_VP]),
    ("b2r_batch_get_engine", C.c_int, [_VP, C.POINTER(_VP)]),
    ("b2r_batch_add_cloud", C.c_int, [_VP, _VP, _SZ, _SZ, _I32P]),
    ("b2r_batch_add_cloud_device", C.c_int, [_VP, _VP, _SZ, _SZ, _I32P]),
    ("b2r_batch_remove_cloud", C.c_int, [_VP, C.c_int32]),
    ("b2r_batch_cloud_count", C.c_int, [_VP]),
    ("b2r_batch_synchronize", C.c_int, [_VP]),
    ("b2r_batch_align", C.c_int, [_VP, C.POINTER(Pair), _SZ, C.c_int, C.c_double, C.POINTER(Result)]),
    ("b2r_batch_calc_fitness_score", C.c_int, [_VP, C.POINTER(Pair), _SZ, C.c_double, _F64P]),
    ("b2r_batch_map_cloud_generate", C.c_int, [_VP, _I32P, _F32P, _SZ, C.c_double, _SZ, _VP, _SZ, C.POINTER(_VP), C.POINTER(_SZ)]),
    ("b2r_information_params_default", C.c_int, [C.POINTER(InformationParams)]),
    ("b2r_information_from_fitness", C.c_int, [C.POINTER(InformationParams), C.c_double, _F64P]),
    ("b2r_batch_last_rounds", C.c_int, [_VP, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    ("b2r_loop_argmin", C.c_int, [C.POINTER(Result), _SZ, C.c_double, _I32P]),
    ("b2r_loop_params_default", C.c_int, [C.POINTER(LoopParams)]),
    ("b2r_loop_find_candidates", C.c_int, [C.POINTER(LoopParams), C.POINTER(KeyframeState), _SZ, C.POINTER(KeyframeState), C.c_double, _I32P, _SZ, C.POINTER(_SZ)]),
    ("b2r_loop_guess", C.c_int, [_F64P, _F64P, _F32P]),
    ("b2r_loop_detect_plan", C.c_int, [C.POINTER(LoopParams), C.POINTER(KeyframeState), _SZ, C.POINTER(KeyframeState), _SZ, C.c_double, _I32P, _F32P, _SZ,
                                       C.POINTER(C.c_int64), C.POINTER(_SZ)]),
    ("b2r_loop_detect_replay", C.c_int, [C.POINTER(LoopParams), C.POINTER(KeyframeState), _SZ, C.POINTER(C.c_int64), _I32P, C.c_double, _F64P, _I32P]),
    ("b2r_nccl_unique_id", C.c_int, [_VP, _SZ]),
    ("b2r_batch_comm_init", C.c_int, [_VP, _VP, C.c_int, C.c_int]),
    ("b2r_shard_range", C.c_int, [_SZ, C.c_int, C.c_int, C.POINTER(_SZ), C.POINTER(_SZ)]),
    ("b2r_batch_loop_detect", C.c_int, [_VP, C.POINTER(Pair), _SZ, C.POINTER(C.c_int64), _SZ, C.c_double, C.c_double, C.POINTER(Result), _I32P]),
]

_lib = None


def load():
    """Load libb200reg.so.  Raises (never falls back) if the library has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m hdl_graph_slam_b200.build` (or __graft_entry__.build()). "
            "hdl_graph_slam_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, res, args in SYMBOLS:
        fn = getattr(lib, name)  # AttributeError if the ABI is incomplete
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class B2RError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200reg error {code}: {msg}")
        self.code = code


def check(rc):
    if rc < 0:
        raise B2RError(rc, load().b2r_last_error().decode("utf-8", "replace"))
    return rc
