// tests/ransac_harness.cu — the device code of floor detection compiled for the host: pcl_eigen33 (csrc/linalg.cuh) and the RANSAC
// sample stream (Mt19937 + ransac_draw, csrc/floor.cuh) are __host__ __device__, so the same source runs here and is compared bit
// for bit with tests/floor_ref.cpp by tests/test_floor_harness.py.  Test infrastructure, built with nvcc (host code is what is called),
// never shipped.
#include <cstddef>
#include <string>
#include <vector>
#include "../hdl_graph_slam_b200/csrc/floor.cuh"
namespace b2r { thread_local std::string g_last_error; }
using namespace b2r;

extern "C" void h_eigen33(const float* A, size_t count, float* v) {
  for (size_t i = 0; i < count; i++) pcl_eigen33(A + 9 * i, v + 3 * i);
}

// the first `count` hypotheses of a fresh model, records as FloorHyp
extern "C" void h_ransac_hypotheses(const float* pts, size_t n, size_t sf, size_t count, FloorHyp* out) {
  Mt19937 g;
  g.seed(kRansacSeed);
  std::vector<int> shuffled(n);
  for (size_t i = 0; i < n; i++) shuffled[i] = (int)i;
  for (size_t t = 0; t < count; t++) {
    ransac_draw(g, shuffled.data(), (int)n, [&](int i) {
      const float* p = pts + (size_t)i * sf;
      return make_float3(p[0], p[1], p[2]);
    }, out[t]);
  }
}
