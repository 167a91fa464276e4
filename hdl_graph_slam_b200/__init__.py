"""hdl_graph_slam_b200 — GPU-native scan-matching engine (NDT + GICP + voxel grid) behind hdl_graph_slam's
pcl::Registration handle.  The product is `_lib/libb200reg.so` (hand-written sm_90a CUDA behind the C ABI of
include/b200reg.h); this package is the thin host-side mirror of the reference interface used by tests and bench.
"""
from ._capi import B2RError, B2R_METHOD_GICP, B2R_METHOD_NDT, B2R_METHOD_NDT_PCL, B2R_METHOD_VGICP, B2R_METHOD_GICP_PCL, B2R_METHOD_ICP_PCL, B2R_METHOD_VGICP_CUDA, B2R_METHOD_GICP_OMP, B2R_METHOD_NDT_KDTREE, Config, load as load_library  # noqa: F401
from ._capi import B2R_DOWNSAMPLE_NONE, B2R_DOWNSAMPLE_VOXELGRID, B2R_DOWNSAMPLE_APPROX_VOXELGRID  # noqa: F401
from .registration import (Registration, select_registration_method, ScanMatchingOdometry, LoopDetector,  # noqa: F401
                           default_config, RegistrationBatch, shard_range, loop_argmin, information_from_fitness, LoopClosureGate)
