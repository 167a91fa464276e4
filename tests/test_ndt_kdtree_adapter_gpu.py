"""GPU: the pcl::Registration adapter (adapter/b200_registration.hpp) driving a B2R_METHOD_NDT_KDTREE handle (NDT_OMP's KDTREE search) through
tests/adapter_harness.cpp, with every check of tests/test_adapter_gpu.py's walk: poses and flags bitwise b2r_align's, getFitnessScore and
the inlier sweep from one launch, the `output` cloud, and the nearest-neighbour cache under awkward consumers."""
import pytest

import hdl_graph_slam_b200 as pkg
import test_adapter_gpu as walk

pytestmark = pytest.mark.gpu
harness = walk.harness
frames = walk.frames


def test_adapter_walk_and_cache_ndt_kdtree(harness, frames, tmp_path):
    walk.test_adapter_walk_and_cache(harness, frames, tmp_path, pkg.B2R_METHOD_NDT_KDTREE)
