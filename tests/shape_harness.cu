// tests/shape_harness.cu — CPU-side print of the cluster launch shape the engine picks for a cloud size (csrc/bvh_build.cuh:
// build_shape_for, build_shape_index).  For every size on the command line it prints one line "n wide index cl per" for wide = 1
// (16-CTA clusters allowed) and wide = 0, so tests/test_launch_shapes_gpu.py can prove that its size list reaches every one of the
// nine instantiations of k_bvh_build_cluster / k_voxelgrid_cluster.
// Test infrastructure: built by tests/test_launch_shapes_gpu.py with nvcc (host code only), never shipped.
#include <cstdio>
#include <cstdlib>
#include "../hdl_graph_slam_b200/csrc/bvh_build.cuh"
using namespace b2r;

int main(int argc, char** argv) {
  for (int i = 1; i < argc; i++) {
    const size_t n = strtoull(argv[i], nullptr, 10);
    for (int wide = 1; wide >= 0; wide--) {
      const BuildShape s = build_shape_for(n, wide != 0);
      printf("%zu %d %d %d %d\n", n, wide, s.cl ? build_shape_index(s) : -1, s.cl, s.per);
    }
  }
  return 0;
}
