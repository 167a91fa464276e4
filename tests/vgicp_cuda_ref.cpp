/* tests/vgicp_cuda_ref.cpp — TEST INFRASTRUCTURE ONLY: the sequential CPU reference of fast_gicp::FastVGICPCuda that defines the parity
 * of B2R_METHOD_VGICP_CUDA (hdl_graph_slam_b200/csrc/vgicp_cuda.cuh).  Built by the tests with -O2 -ffp-contract=off: every float32
 * operation below is one IEEE rounding, in the order written, as the device's __fmul_rn / __fadd_rn / __fdiv_rn / __fsqrt_rn.
 *
 * fast_gicp is an unpinned dependency that is not part of the reference tree, so every choice below is UPSTREAM-RECALL (recalled from
 * fast_vgicp_cuda_impl.hpp and src/fast_gicp/cuda/{covariance_estimation, covariance_regularization, gaussian_voxelmap,
 * find_voxel_correspondences, compute_derivatives}.cu) or, where upstream is undefined or not reproduced, this engine's rule (ENGINE):
 *   factory (registrations.cpp:37-47): reg_resolution (1.0), reg_transformation_epsilon (0.01), reg_maximum_iterations (64),
 *     reg_correspondence_randomness (20); rotation_epsilon 2e-3 (LsqRegistration's default); reg_max_correspondence_distance and
 *     reg_num_threads are not read.  hdl never calls the neighbour-search, regularisation or kernel setters: k-NN exact, PLANE,
 *     voxel search DIRECT1.                                                                                         UPSTREAM-RECALL
 *   k-NN: k = reg_correspondence_randomness neighbours in the same cloud, the point itself included, ascending (d2, index); d2 in
 *     float32 ((dx dx + dy dy) + dz dz).  Upstream's default kd-tree and its brute force are both exact; only the tie order is
 *     unspecified upstream.                                                                                 UPSTREAM-RECALL (ties: ENGINE)
 *   covariance: float32 throughout; mean += p and cov(a, b) += p_a p_b over the list in order; mean /= k; cov = cov / k - mean mean^T.
 *     Far from the origin the raw moments cancel catastrophically (that is upstream's arithmetic, kept on purpose).  UPSTREAM-RECALL
 *   PLANE: upstream runs a branch-free float32 3x3 SVD (McAdams-style svd3) and forms U diag(1, 1, 1e-3) V^T.  Restated here as
 *     C = sum_i v_i u_i u_i^T over a float32 symmetric eigen-decomposition (cyclic Jacobi, the rules of eigen3f below), eigenvalues
 *     ascending, v = (1e-3, 1, 1), each entry (a <= b, mirrored) ((1e-3 u0_a) u0_b + u1_a u1_b) + u2_a u2_b.  svd3's iterations are not
 *     reproduced: its U and V agree with these eigenvectors only to float32 rounding, and for an indefinite matrix (cancellation far
 *     from the origin) svd3 orders by |eigenvalue| where this keeps the smallest eigenvalue.                         ENGINE
 *     An exactly diagonal matrix (an axis-aligned line) has tied eigenvalues: the normal is whichever column this Jacobi's selection
 *     sort leaves first, not the JacobiSVD rule of the float64 engines (svd3 is not JacobiSVD).                          ENGINE
 *   a cloud with fewer than k finite points: the moments run over the neighbours found and divide by their count.    ENGINE
 *   non-finite points are nobody's neighbour, have no covariance, belong to no voxel and have no correspondence.      ENGINE
 *   voxel map of the target: cell = floorf(x / res - 0.5f) per axis in float32, the division and the subtraction rounded separately
 *     (calc_voxel_coord; recalled with more confidence than the CPU FastVGICP's cell, whose floor(p / res) contract is unchanged);
 *     each voxel holds num_points and float32 sums of the points and of their covariances; finalize: / num_points in float32; no
 *     minimum count.                                                                                                 UPSTREAM-RECALL
 *     The sums run in ascending point index (upstream's atomicAdd order is undefined).                              ENGINE
 *     Cells are limited to [-2^20, 2^20) per axis (21-bit keys): a finite target point beyond fails the build (status 1); a source
 *     point that transforms beyond has no correspondence.                                                            ENGINE
 *   correspondence (DIRECT1): the LM's Isometry3d rounded to float32 (R_f, t_f); x' = R_f mu_A + t_f per row ((r0 x + r1 y) + r2 z) + t;
 *     the voxel of x''s cell, or none.                                                                               UPSTREAM-RECALL
 *   terms, float32: RC = R C_A ((r0 c0j + r1 c1j) + r2 c2j), RCR(i, j) = C_B(i, j) + ((RC_i0 r_j0 + RC_i1 r_j1) + RC_i2 r_j2) for i <= j,
 *     mirrored; M = Eigen's cofactor inverse: cof(i, j) = m(i1, j1) m(i2, j2) - m(i1, j2) m(i2, j1), det = (c00 m00 + c10 m10) + c20 m20,
 *     M(i, j) = cof(j, i) * (1 / det); w = sqrtf((float)n); e = mu_B - x'; J = [skew(x') | -I] with S = skew(x') and (S^T X)_a as
 *     skew_t below; Me_r = (M_r0 e0 + M_r1 e1) + M_r2 e2; H rotation block w (S^T (M S)) (M S)(r, c) = (S^T m_r)_c, cross block
 *     -(w (S^T M)), translation block w M; b = (w S^T Me, -(w Me)); cost = w ((e0 Me0 + e1 Me1) + e2 Me2).  Upstream evaluates the same
 *     products through Eigen's expression templates; their order (and upstream's nvcc contractions) are not reproduced.  UPSTREAM-RECALL
 *     compute_error at a trial pose reuses the linearisation's voxels and M (upstream recomputes M from the linearisation pose, which
 *     gives the same value).                                                                                         UPSTREAM-RECALL
 *   sums: the float32 terms are added in float64 in ascending source index (the device: k_pair_accumulate's fixed tree; upstream's
 *     float32 thrust::transform_reduce has no defined order, so no choice matches it).  A deliberate deviation.      ENGINE
 *   optimiser: LsqRegistration::step_lm with FastGICP's convergence test, exactly vgicp_ref.cpp's (a singular / non-finite step ends the
 *     registration as "lm not converged", pose kept).
 */
#include "vgicp_ref.cpp"  // the step_lm of the FastVGICP reference (se3_exp, is_converged, mul4_iso): the optimiser is the same
#include "../oracle/kdtree.hpp"

namespace {

bool vc_finite(const float* p) { return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]); }

// cyclic Jacobi of a symmetric 3x3 (row-major) in float32; w ascending, V columns = eigenvectors (the device's vcuda_eigen3)
void eigen3f(const float* Ain, float* w, float* V) {
  float A[9];
  for (int i = 0; i < 9; i++) A[i] = Ain[i];
  for (int i = 0; i < 9; i++) V[i] = (i % 4 == 0) ? 1.f : 0.f;
  for (int sweep = 0; sweep < 32; sweep++) {
    if ((std::fabs(A[1]) + std::fabs(A[2])) + std::fabs(A[5]) == 0.f) break;
    for (int pq = 0; pq < 3; pq++) {
      const int p = (pq == 2) ? 1 : 0;
      const int q = (pq == 0) ? 1 : 2;
      const float apq = A[p * 3 + q];
      if (apq == 0.f) continue;
      const float app = A[p * 3 + p], aqq = A[q * 3 + q];
      const float g = 100.f * std::fabs(apq);
      if (std::fabs(app) + g == std::fabs(app) && std::fabs(aqq) + g == std::fabs(aqq)) {
        A[p * 3 + q] = 0.f; A[q * 3 + p] = 0.f;
        continue;
      }
      const float h = aqq - app;
      float t;
      if (std::fabs(h) + g == std::fabs(h)) {
        t = apq / h;
      } else {
        const float theta = (0.5f * h) / apq;
        t = 1.f / (std::fabs(theta) + std::sqrt(1.f + theta * theta));
        if (theta < 0.f) t = -t;
      }
      const float c = 1.f / std::sqrt(1.f + t * t), s = t * c;
      for (int k = 0; k < 3; k++) {
        const float akp = A[k * 3 + p], akq = A[k * 3 + q];
        A[k * 3 + p] = c * akp - s * akq;
        A[k * 3 + q] = s * akp + c * akq;
      }
      for (int k = 0; k < 3; k++) {
        const float apk = A[p * 3 + k], aqk = A[q * 3 + k];
        A[p * 3 + k] = c * apk - s * aqk;
        A[q * 3 + k] = s * apk + c * aqk;
      }
      for (int k = 0; k < 3; k++) {
        const float vkp = V[k * 3 + p], vkq = V[k * 3 + q];
        V[k * 3 + p] = c * vkp - s * vkq;
        V[k * 3 + q] = s * vkp + c * vkq;
      }
      A[p * 3 + q] = 0.f; A[q * 3 + p] = 0.f;
    }
  }
  w[0] = A[0]; w[1] = A[4]; w[2] = A[8];
  auto swapcol = [&](int a, int b) {
    std::swap(w[a], w[b]);
    for (int k = 0; k < 3; k++) std::swap(V[k * 3 + a], V[k * 3 + b]);
  };
  if (w[1] < w[0]) {
    if (w[2] < w[1]) swapcol(0, 2); else swapcol(0, 1);
  } else if (w[2] < w[0]) {
    swapcol(0, 2);
  }
  if (w[2] < w[1]) swapcol(1, 2);
}

void covariances_f(const float* pts, size_t n, size_t stride, int k, double* out) {
  orc::KdTree tree;
  tree.build(pts, n, stride);
  std::vector<int> idx(k);
  std::vector<float> d2(k);
  for (size_t i = 0; i < n; i++) {
    double* o = out + i * 9;
    const float* q = pts + i * stride;
    if (!vc_finite(q)) { for (int a = 0; a < 9; a++) o[a] = NAN; continue; }
    const int kk = tree.knn(q, k, idx.data(), d2.data());
    float m[3] = {0.f, 0.f, 0.f}, s[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < kk; j++) {
      const float* p = pts + (size_t)idx[j] * stride;
      for (int a = 0; a < 3; a++) m[a] = m[a] + p[a];
      for (int a = 0; a < 3; a++)
        for (int b = a; b < 3; b++) s[a * 3 + b] = s[a * 3 + b] + p[a] * p[b];
    }
    const float kf = (float)kk;
    for (int a = 0; a < 3; a++) m[a] = m[a] / kf;
    float C[9];
    for (int a = 0; a < 3; a++)
      for (int b = a; b < 3; b++) C[a * 3 + b] = C[b * 3 + a] = s[a * 3 + b] / kf - m[a] * m[b];
    float w[3], V[9];
    eigen3f(C, w, V);
    for (int a = 0; a < 3; a++)
      for (int b = a; b < 3; b++) {
        const float x = ((1e-3f * V[a * 3 + 0]) * V[b * 3 + 0] + V[a * 3 + 1] * V[b * 3 + 1]) + V[a * 3 + 2] * V[b * 3 + 2];
        o[a * 3 + b] = o[b * 3 + a] = (double)x;
      }
  }
}

struct FVoxel {
  int n = 0;
  float mean[3] = {0, 0, 0};
  float cov[6] = {0, 0, 0, 0, 0, 0};  // xx xy xz yy yz zz
};

struct FMap {
  float res;
  std::map<std::array<int, 3>, int> index;
  std::vector<std::array<int, 3>> cells;
  std::vector<FVoxel> vox;
};

bool cell_f(const float* x, float res, std::array<int, 3>& c) {
  for (int a = 0; a < 3; a++) {
    const float q = x[a] / res;
    const float f = std::floor(q - 0.5f);
    if (!(f >= -(float)kBias && f < (float)kBias)) return false;
    c[a] = (int)f;
  }
  return true;
}

// (S^T X)_a for S = skew(x)
float skew_t(int a, const float* x, float X0, float X1, float X2) {
  if (a == 0) return x[2] * X1 - x[1] * X2;
  if (a == 1) return x[0] * X2 - x[2] * X0;
  return x[1] * X0 - x[0] * X1;
}

void pose_f(const double* T, float* Tf) {
  for (int i = 0; i < 12; i++) Tf[i] = (float)T[i];
}

void xform_f(const float* Tf, const float* p, float* x) {
  for (int r = 0; r < 3; r++) x[r] = ((Tf[r * 4] * p[0] + Tf[r * 4 + 1] * p[1]) + Tf[r * 4 + 2] * p[2]) + Tf[r * 4 + 3];
}

float quad_f(const float* M, const float* e, float* Me) {
  for (int r = 0; r < 3; r++) Me[r] = (M[r * 3] * e[0] + M[r * 3 + 1] * e[1]) + M[r * 3 + 2] * e[2];
  return (e[0] * Me[0] + e[1] * Me[1]) + e[2] * Me[2];
}

// update_correspondences + linearize at T (row-major double 4x4); M per point (9 floats) kept for compute_error
double linearize_f(const FMap& Mp, const float* src, size_t n, size_t stride, const double* scov, const double* T, int32_t* vox_of, float* Ms,
                   double* H, double* b) {
  float Tf[12];
  pose_f(T, Tf);
  const float R[9] = {Tf[0], Tf[1], Tf[2], Tf[4], Tf[5], Tf[6], Tf[8], Tf[9], Tf[10]};
  double cost = 0.0;
  std::memset(H, 0, 36 * sizeof(double));
  std::memset(b, 0, 6 * sizeof(double));
  for (size_t i = 0; i < n; i++) {
    const float* p = src + i * stride;
    vox_of[i] = -1;
    if (!vc_finite(p)) continue;
    float x[3];
    xform_f(Tf, p, x);
    std::array<int, 3> c;
    if (!cell_f(x, Mp.res, c)) continue;
    auto it = Mp.index.find(c);
    if (it == Mp.index.end()) continue;
    const int v = it->second;
    vox_of[i] = v;
    const FVoxel& V = Mp.vox[v];
    float CA[9];
    for (int a = 0; a < 9; a++) CA[a] = (float)scov[i * 9 + a];
    float RC[9], m[9];
    for (int r = 0; r < 3; r++)
      for (int j = 0; j < 3; j++) RC[r * 3 + j] = (R[r * 3] * CA[j] + R[r * 3 + 1] * CA[3 + j]) + R[r * 3 + 2] * CA[6 + j];
    int k = 0;
    for (int r = 0; r < 3; r++)
      for (int j = r; j < 3; j++, k++) {
        const float u = (RC[r * 3] * R[j * 3] + RC[r * 3 + 1] * R[j * 3 + 1]) + RC[r * 3 + 2] * R[j * 3 + 2];
        m[r * 3 + j] = m[j * 3 + r] = V.cov[k] + u;
      }
    float cof[9];
    for (int r = 0; r < 3; r++)
      for (int j = 0; j < 3; j++) {
        const int r1 = (r + 1) % 3, r2 = (r + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        cof[r * 3 + j] = m[r1 * 3 + j1] * m[r2 * 3 + j2] - m[r1 * 3 + j2] * m[r2 * 3 + j1];
      }
    const float det = (cof[0] * m[0] + cof[3] * m[3]) + cof[6] * m[6];
    const float inv = 1.f / det;
    float* M = Ms + i * 9;
    for (int r = 0; r < 3; r++)
      for (int j = 0; j < 3; j++) M[r * 3 + j] = cof[j * 3 + r] * inv;
    const float w = std::sqrt((float)V.n);
    const float e[3] = {V.mean[0] - x[0], V.mean[1] - x[1], V.mean[2] - x[2]};
    float Me[3];
    const float q = quad_f(M, e, Me);
    float MS[9];
    for (int r = 0; r < 3; r++)
      for (int cc = 0; cc < 3; cc++) MS[r * 3 + cc] = skew_t(cc, x, M[r * 3], M[r * 3 + 1], M[r * 3 + 2]);
    for (int a = 0; a < 6; a++)
      for (int bb = a; bb < 6; bb++) {
        float h;
        if (a < 3 && bb < 3) h = w * skew_t(a, x, MS[bb], MS[3 + bb], MS[6 + bb]);
        else if (a < 3) h = -(w * skew_t(a, x, M[bb - 3], M[3 + bb - 3], M[6 + bb - 3]));
        else h = w * M[(a - 3) * 3 + (bb - 3)];
        H[a * 6 + bb] += (double)h;
      }
    for (int a = 0; a < 3; a++) b[a] += (double)(w * skew_t(a, x, Me[0], Me[1], Me[2]));
    for (int a = 0; a < 3; a++) b[3 + a] += (double)(-(w * Me[a]));
    cost += (double)(w * q);
  }
  for (int a = 0; a < 6; a++)
    for (int bb = 0; bb < a; bb++) H[a * 6 + bb] = H[bb * 6 + a];
  return cost;
}

double error_f(const FMap& Mp, const float* src, size_t n, size_t stride, const int32_t* vox_of, const float* Ms, const double* T) {
  float Tf[12];
  pose_f(T, Tf);
  double cost = 0.0;
  for (size_t i = 0; i < n; i++) {
    const int v = vox_of[i];
    if (v < 0) continue;
    const FVoxel& V = Mp.vox[v];
    float x[3], Me[3];
    xform_f(Tf, src + i * stride, x);
    const float e[3] = {V.mean[0] - x[0], V.mean[1] - x[1], V.mean[2] - x[2]};
    const float q = quad_f(Ms + i * 9, e, Me);
    cost += (double)(std::sqrt((float)V.n) * q);
  }
  return cost;
}

}  // namespace

extern "C" {

/* covariances of every point (n x 9, row-major 3x3 of float32 values widened; NaN rows for non-finite points) */
void ref_vcuda_covariances(const float* pts, size_t n, size_t stride, int k, double* out) { covariances_f(pts, n, stride, k, out); }

/* voxel map of the target; cov: m x 9 (the covariances above).  *status = 1: a finite point lies beyond the 21-bit cell range */
void* ref_vcuda_map(const float* tgt, size_t m, size_t stride, const double* cov, double res, int* status) {
  FMap* M = new FMap();
  M->res = (float)res;
  *status = 0;
  std::map<std::array<int, 3>, FVoxel> acc;
  for (size_t i = 0; i < m; i++) {
    const float* p = tgt + i * stride;
    if (!vc_finite(p)) continue;
    std::array<int, 3> c;
    if (!cell_f(p, M->res, c)) { *status = 1; continue; }
    FVoxel& V = acc[c];
    V.n++;
    for (int a = 0; a < 3; a++) V.mean[a] = V.mean[a] + p[a];
    const double* ci = cov + i * 9;
    const float cu[6] = {(float)ci[0], (float)ci[1], (float)ci[2], (float)ci[4], (float)ci[5], (float)ci[8]};
    for (int a = 0; a < 6; a++) V.cov[a] = V.cov[a] + cu[a];
  }
  if (*status) return M;
  for (auto& kv : acc) {
    FVoxel V = kv.second;
    const float nf = (float)V.n;
    for (int a = 0; a < 3; a++) V.mean[a] = V.mean[a] / nf;
    for (int a = 0; a < 6; a++) V.cov[a] = V.cov[a] / nf;
    M->index[kv.first] = (int)M->vox.size();
    M->cells.push_back(kv.first);
    M->vox.push_back(V);
  }
  return M;
}

void ref_vcuda_free(void* m) { delete static_cast<FMap*>(m); }

/* returns V; arrays (cells 3V, counts V, mean 3V, cov 9V, float32 values widened) may be NULL */
size_t ref_vcuda_voxels(const void* m, int32_t* cells, int32_t* counts, double* mean, double* cov) {
  const FMap& M = *static_cast<const FMap*>(m);
  static const int full[9] = {0, 1, 2, 1, 3, 4, 2, 4, 5};
  for (size_t v = 0; v < M.vox.size(); v++) {
    if (cells) for (int a = 0; a < 3; a++) cells[v * 3 + a] = M.cells[v][a];
    if (counts) counts[v] = M.vox[v].n;
    if (mean) for (int a = 0; a < 3; a++) mean[v * 3 + a] = M.vox[v].mean[a];
    if (cov) for (int a = 0; a < 9; a++) cov[v * 9 + a] = M.vox[v].cov[full[a]];
  }
  return M.vox.size();
}

/* update_correspondences + linearize at T (row-major 4x4 double): H[36], b[6], vox_of[n]; returns the cost */
double ref_vcuda_linearize(const void* m, const float* src, size_t n, size_t stride, const double* scov, const double* T, double* H, double* b,
                           int32_t* vox_of) {
  std::vector<float> Ms(n * 9 + 9);
  return linearize_f(*static_cast<const FMap*>(m), src, n, stride, scov, T, vox_of, Ms.data(), H, b);
}

/* compute_error at T2 with the voxels and M of the linearisation at T1 */
double ref_vcuda_error(const void* m, const float* src, size_t n, size_t stride, const double* scov, const double* T1, const double* T2) {
  std::vector<float> Ms(n * 9 + 9);
  std::vector<int32_t> vox(n + 1);
  double H[36], b[6];
  const FMap& M = *static_cast<const FMap*>(m);
  linearize_f(M, src, n, stride, scov, T1, vox.data(), Ms.data(), H, b);
  return error_f(M, src, n, stride, vox.data(), Ms.data(), T2);
}

/* align(): cfg_d = {transformation_epsilon, rotation_epsilon}, cfg_i = {max_iterations}; guess / T_out row-major float;
 * out = {converged, iterations, lm_failed}; T64 (16, may be NULL) = the pose before the float cast.  step_lm as ref_vgicp_align */
void ref_vcuda_align(const void* m, const float* src, size_t n, size_t stride, const double* scov, const double* cfg_d, const int* cfg_i,
                     const float* guess, float* T_out, int* out, double* T64) {
  const FMap& M = *static_cast<const FMap*>(m);
  double x0[16];
  for (int i = 0; i < 16; i++) x0[i] = (double)guess[i];
  x0[12] = x0[13] = x0[14] = 0; x0[15] = 1;
  out[0] = out[1] = out[2] = 0;
  std::vector<int32_t> vox(n + 1);
  std::vector<float> Ms(n * 9 + 9);
  double lambda = -1.0;
  bool converged = false, lm_failed = false;
  int it = 0;
  for (it = 0; it < cfg_i[0] && !converged; it++) {
    double H[36], b[6], delta[16];
    const double y0 = linearize_f(M, src, n, stride, scov, x0, vox.data(), Ms.data(), H, b);
    if (lambda < 0.0) {
      double mx = 0;
      for (int i = 0; i < 6; i++) mx = std::max(mx, std::fabs(H[i * 6 + i]));
      lambda = 1e-9 * mx;
    }
    double nu = 2.0;
    bool ok = false;
    for (int li = 0; li < 10; li++) {
      double A[36], nb[6], d[6];
      for (int i = 0; i < 36; i++) A[i] = H[i] + ((i % 7 == 0) ? lambda : 0.0);
      for (int i = 0; i < 6; i++) nb[i] = -b[i];
      bool solved = ldlt6_solve(A, nb, d);
      for (int i = 0; i < 6; i++) solved &= std::isfinite(d[i]);
      if (!solved) break;
      se3_exp(d, delta);
      double xi[16];
      mul4_iso(delta, x0, xi);
      const double yi = error_f(M, src, n, stride, vox.data(), Ms.data(), xi);
      double den = 0;
      for (int i = 0; i < 6; i++) den += d[i] * (lambda * d[i] - b[i]);
      const double rho = (y0 - yi) / den;
      if (rho < 0) {
        if (is_converged(delta, cfg_d[1], cfg_d[0])) { ok = true; break; }
        lambda = nu * lambda;
        nu = 2 * nu;
        continue;
      }
      const double t = 2 * rho - 1;
      lambda = lambda * std::max(1.0 / 3.0, 1 - t * t * t);
      std::memcpy(x0, xi, sizeof(xi));
      ok = true;
      break;
    }
    if (!ok) { lm_failed = true; it++; break; }
    converged = is_converged(delta, cfg_d[1], cfg_d[0]);
  }
  for (int i = 0; i < 16; i++) T_out[i] = (float)x0[i];
  if (T64) std::memcpy(T64, x0, sizeof(x0));
  out[0] = converged ? 1 : 0;
  out[1] = it;
  out[2] = lm_failed ? 1 : 0;
}

}  // extern "C"
