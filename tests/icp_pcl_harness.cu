// tests/icp_pcl_harness.cu — host build of the __host__ __device__ ICP step of csrc/linalg.cuh (icp_jacobi_svd3, icp_umeyama,
// icp_has_converged: the code the last block of k_icp_step runs), as a shared library that test_icp_pcl_oracle compares bit for bit
// with tests/icp_pcl_ref.cpp.
#include "../hdl_graph_slam_b200/csrc/linalg.cuh"

extern "C" {
void dev_icp_svd(const float* A, float* U, float* d, float* V) { b2r::icp_jacobi_svd3(A, U, d, V); }
void dev_icp_umeyama(const float* sigma, const float* sm, const float* dm, float* Rt) { b2r::icp_umeyama(sigma, sm, dm, Rt); }
int dev_icp_has_converged(const float* T, int iterations, int max_iterations, double rot_thr, double trans_thr, double mse, double* prev) {
  return b2r::icp_has_converged(T, iterations, max_iterations, rot_thr, trans_thr, mse, prev) ? 1 : 0;
}
}
