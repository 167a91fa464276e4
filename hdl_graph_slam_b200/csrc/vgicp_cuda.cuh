// vgicp_cuda.cuh — fast_gicp::FastVGICPCuda on the device (B2R_METHOD_VGICP_CUDA): float32 raw-moment covariances, a float32
// Gaussian voxel map with a half-cell offset, and a float32 VGICP round.
//
// Semantics (tests/vgicp_cuda_ref.cpp is the sequential statement the tests hold this file to; every float32 operation below is
// correctly rounded and unfused, __fmul_rn / __fadd_rn / __fdiv_rn / __fsqrt_rn, in the order written there):
//   * covariances (VcudaCov, on the raw-moment k-NN kernels of gicp_pcl.cuh): mean += p and cov(a, b) += p_a p_b in float32 over the
//     k-NN list in order; mean /= k; cov = cov / k - mean mean^T; PLANE: the float32 Jacobi eigen-decomposition vcuda_eigen3 below,
//     C = sum_i v_i u_i u_i^T over the eigenvectors in ascending eigenvalue order with v = (1e-3, 1, 1).  Stored widened to double in
//     the cloud's covariance slot (exact), so prefetch, promotion and the batch's cloud cache carry them unchanged.
//   * voxel map (VcudaMapRule on vgicp.cuh's build): cell = floorf(x / res - 0.5f) per axis in float32; float32 sums of the points
//     and covariances in ascending point index; finalize / num_points in float32.
//   * correspondence (DIRECT1): x' = R_f mu_A + t_f with the LM pose rounded to float32, ((r0 x + r1 y) + r2 z) + t; the voxel of
//     x''s cell, or none.
//   * terms: RCR = C_B + (R C_A) R^T (upper triangle, mirrored), M = Eigen's cofactor inverse, w = sqrtf(n), e = mu_B - x',
//     J = [skew(x') | -I]; H = w J^T M J, b = w J^T M e, cost = w e^T M e in float32; summed in float64 by k_pair_accumulate's tree.
//     compute_error at a trial pose reuses the linearisation's voxel and M.
#pragma once
#include "vgicp.cuh"
#include "gicp_pcl.cuh"

namespace b2r {

// Cyclic Jacobi eigen-decomposition of a symmetric 3x3 (row-major) in float32: w ascending, V columns = eigenvectors.  Only
// correctly rounded operations, so the host reference reproduces it bit for bit: a rotation whose pivot is negligible against both
// diagonal entries (|a| + 100 |apq| == |a|) zeroes the pivot instead, and every rotation sets its pivot to an exact zero.  Ties keep
// the column order (selection sort, the first minimum wins).
__device__ __forceinline__ void vcuda_eigen3(const float* Ain, float* w, float* V) {
  float A[9];
#pragma unroll
  for (int i = 0; i < 9; i++) A[i] = Ain[i];
  V[0] = 1.f; V[1] = 0.f; V[2] = 0.f; V[3] = 0.f; V[4] = 1.f; V[5] = 0.f; V[6] = 0.f; V[7] = 0.f; V[8] = 1.f;
  for (int sweep = 0; sweep < 32; sweep++) {
    if (__fadd_rn(__fadd_rn(fabsf(A[1]), fabsf(A[2])), fabsf(A[5])) == 0.f) break;
#pragma unroll
    for (int pq = 0; pq < 3; pq++) {
      const int p = (pq == 2) ? 1 : 0;
      const int q = (pq == 0) ? 1 : 2;
      const float apq = A[p * 3 + q];
      if (apq == 0.f) continue;
      const float app = A[p * 3 + p], aqq = A[q * 3 + q];
      const float g = __fmul_rn(100.f, fabsf(apq));
      if (__fadd_rn(fabsf(app), g) == fabsf(app) && __fadd_rn(fabsf(aqq), g) == fabsf(aqq)) {
        A[p * 3 + q] = 0.f; A[q * 3 + p] = 0.f;
        continue;
      }
      const float h = __fsub_rn(aqq, app);
      float t;
      if (__fadd_rn(fabsf(h), g) == fabsf(h)) {
        t = __fdiv_rn(apq, h);
      } else {
        const float theta = __fdiv_rn(__fmul_rn(0.5f, h), apq);
        t = __fdiv_rn(1.f, __fadd_rn(fabsf(theta), __fsqrt_rn(__fadd_rn(1.f, __fmul_rn(theta, theta)))));
        if (theta < 0.f) t = -t;
      }
      const float c = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(1.f, __fmul_rn(t, t)))), s = __fmul_rn(t, c);
#pragma unroll
      for (int k = 0; k < 3; k++) {
        const float akp = A[k * 3 + p], akq = A[k * 3 + q];
        A[k * 3 + p] = __fsub_rn(__fmul_rn(c, akp), __fmul_rn(s, akq));
        A[k * 3 + q] = __fadd_rn(__fmul_rn(s, akp), __fmul_rn(c, akq));
      }
#pragma unroll
      for (int k = 0; k < 3; k++) {
        const float apk = A[p * 3 + k], aqk = A[q * 3 + k];
        A[p * 3 + k] = __fsub_rn(__fmul_rn(c, apk), __fmul_rn(s, aqk));
        A[q * 3 + k] = __fadd_rn(__fmul_rn(s, apk), __fmul_rn(c, aqk));
      }
#pragma unroll
      for (int k = 0; k < 3; k++) {
        const float vkp = V[k * 3 + p], vkq = V[k * 3 + q];
        V[k * 3 + p] = __fsub_rn(__fmul_rn(c, vkp), __fmul_rn(s, vkq));
        V[k * 3 + q] = __fadd_rn(__fmul_rn(s, vkp), __fmul_rn(c, vkq));
      }
      A[p * 3 + q] = 0.f; A[q * 3 + p] = 0.f;
    }
  }
  w[0] = A[0]; w[1] = A[4]; w[2] = A[8];
#define B2R_SWAPCOL(a, b)                                  \
  {                                                        \
    float tw = w[a]; w[a] = w[b]; w[b] = tw;               \
    for (int k = 0; k < 3; k++) { float tv = V[k * 3 + a]; V[k * 3 + a] = V[k * 3 + b]; V[k * 3 + b] = tv; } \
  }
  if (w[1] < w[0]) {
    if (w[2] < w[1]) B2R_SWAPCOL(0, 2) else B2R_SWAPCOL(0, 1)
  } else if (w[2] < w[0]) {
    B2R_SWAPCOL(0, 2)
  }
  if (w[2] < w[1]) B2R_SWAPCOL(1, 2)
#undef B2R_SWAPCOL
}

// The float32 raw-moment covariance of kk neighbours in list order, row-major into C: sums of p and of p_a p_b, / kk, then
// cov = E[ab] - E[a]E[b].  Statement for statement this is also pcl::computeMeanAndCovarianceMatrix's dense path (PCL 1.10), the
// moments of NormalEstimation in floor.cuh.
template <class PtAt>
__device__ __forceinline__ void raw_moment_cov_f32(int kk, PtAt pt_at, float* C) {
  float m[3] = {0.f, 0.f, 0.f}, s[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // s: xx xy xz yy yz zz
  for (int j = 0; j < kk; j++) {
    const float3 p = pt_at(j);
    m[0] = __fadd_rn(m[0], p.x); m[1] = __fadd_rn(m[1], p.y); m[2] = __fadd_rn(m[2], p.z);
    s[0] = __fadd_rn(s[0], __fmul_rn(p.x, p.x)); s[1] = __fadd_rn(s[1], __fmul_rn(p.x, p.y)); s[2] = __fadd_rn(s[2], __fmul_rn(p.x, p.z));
    s[3] = __fadd_rn(s[3], __fmul_rn(p.y, p.y)); s[4] = __fadd_rn(s[4], __fmul_rn(p.y, p.z)); s[5] = __fadd_rn(s[5], __fmul_rn(p.z, p.z));
  }
  const float kf = (float)kk;
#pragma unroll
  for (int a = 0; a < 3; a++) m[a] = __fdiv_rn(m[a], kf);
  const float c00 = __fsub_rn(__fdiv_rn(s[0], kf), __fmul_rn(m[0], m[0])), c01 = __fsub_rn(__fdiv_rn(s[1], kf), __fmul_rn(m[0], m[1]));
  const float c02 = __fsub_rn(__fdiv_rn(s[2], kf), __fmul_rn(m[0], m[2])), c11 = __fsub_rn(__fdiv_rn(s[3], kf), __fmul_rn(m[1], m[1]));
  const float c12 = __fsub_rn(__fdiv_rn(s[4], kf), __fmul_rn(m[1], m[2])), c22 = __fsub_rn(__fdiv_rn(s[5], kf), __fmul_rn(m[2], m[2]));
  C[0] = c00; C[1] = c01; C[2] = c02; C[3] = c01; C[4] = c11; C[5] = c12; C[6] = c02; C[7] = c12; C[8] = c22;
}

// FastVGICPCuda's covariance of one point over its kk neighbours (covariance_estimation + covariance_regularization PLANE).  Stores
// xx, xy, xz, yy, yz, zz, each a float32 value widened.
struct VcudaCov {
  template <class PtAt>
  __device__ __forceinline__ static void store(int kk, PtAt pt_at, double* __restrict__ o) {
    float C[9];
    raw_moment_cov_f32(kk, pt_at, C);
    float w[3], V[9];
    vcuda_eigen3(C, w, V);
    // (1e-3 u0_a u0_b + u1_a u1_b) + u2_a u2_b for a <= b
    int k = 0;
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
      for (int b = a; b < 3; b++)
        o[k++] = (double)__fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn(1e-3f, V[a * 3 + 0]), V[b * 3 + 0]), __fmul_rn(V[a * 3 + 1], V[b * 3 + 1])),
                                   __fmul_rn(V[a * 3 + 2], V[b * 3 + 2]));
  }
};

// FastVGICPCuda's voxel rule: cell floorf(x / res - 0.5f) in float32 (division and subtraction rounded separately), float32 sums
struct VcudaMapRule {
  using Acc = float;
  __device__ __forceinline__ static bool cell(float x, float y, float z, double res, unsigned long long* key) {
    const float r = (float)res;
    return vgicp_key((double)floorf(__fsub_rn(__fdiv_rn(x, r), 0.5f)), (double)floorf(__fsub_rn(__fdiv_rn(y, r), 0.5f)),
                     (double)floorf(__fsub_rn(__fdiv_rn(z, r), 0.5f)), key);
  }
  __device__ __forceinline__ static float add(float a, float b) { return __fadd_rn(a, b); }
  __device__ __forceinline__ static float div(float a, int n) { return __fdiv_rn(a, (float)n); }
};

#ifdef __CUDACC__
// (S^T X)_a for S = skew(x), X a 3-vector: S's column a is (0, z, -y), (-z, 0, x), (y, -x, 0)
__device__ __forceinline__ float vcuda_skew_t(int a, float x, float y, float z, float X0, float X1, float X2) {
  return a == 0 ? __fsub_rn(__fmul_rn(z, X1), __fmul_rn(y, X2)) : a == 1 ? __fsub_rn(__fmul_rn(x, X2), __fmul_rn(z, X0))
                                                                        : __fsub_rn(__fmul_rn(y, X0), __fmul_rn(x, X1));
}

// The FastVGICPCuda round of every active pair, as k_vgicp_round: probe at xe (PM_FIRST / PM_FUSED) into the write set, M and the
// weighted float32 linearisation, and compute_error at xe with the previous set (PM_FUSED / PM_ERR).  The stored matrix is M itself
// (widened); the trial cost recomputes w from the voxel.  Block partials as k_pair_accumulate leaves them, for k_pair_lm.
__global__ void __launch_bounds__(kAccThreads, B2R_ACC_MINBLOCKS) k_vgicp_cuda_round(PairDev* pairs, const int* __restrict__ active,
                                                                                     const VgicpMapDev* __restrict__ maps) {
  __shared__ double red[kAcc * 8];
  __shared__ double tiles[(kAccThreads / 32) * 8 * kRedRow];
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (!active) asm volatile("griddepcontrol.launch_dependents;");
  if (active && (int)blockIdx.y >= active[0]) return;
  const int pi = active ? active[1 + blockIdx.y] : blockIdx.y;
  PairDev& p = pairs[pi];
  const int mode = p.mode;
  if (mode < PM_FIRST || mode > PM_ERR) return;
  const int nblk = p.nblk_acc;
  if ((int)blockIdx.x >= nblk) return;
  const VgicpMapDev Mp = maps[pi];
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* tile = tiles + warp * 8 * kRedRow;
  const int cur = p.cur;
  const int wset = (mode == PM_FIRST) ? cur : (cur ^ 1);
  float4 pt = make_float4(0.f, 0.f, 0.f, bits_idx(kPadIdx));
  if (s < p.src.nleaf * kLeaf) pt = p.src.sp[s];
  const bool is_point = idx_bits(pt.w) != kPadIdx;
  const bool do_trial = (mode == PM_FUSED || mode == PM_ERR) && is_point;
  const bool do_lin = (mode == PM_FIRST || mode == PM_FUSED) && is_point;
  float T[12];
#pragma unroll
  for (int i = 0; i < 12; i++) T[i] = __double2float_rn(p.xe[i]);
  const float tx = xform_row(T[0], T[1], T[2], T[3], pt.x, pt.y, pt.z);
  const float ty = xform_row(T[4], T[5], T[6], T[7], pt.x, pt.y, pt.z);
  const float tz = xform_row(T[8], T[9], T[10], T[11], pt.x, pt.y, pt.z);
  // ---- compute_error at xe with the previous correspondences and M
  float trial = 0.f;
  if (do_trial) {
    const int v = p.cpos[cur][s];
    if (v >= 0) {
      const double* md = p.mahal[cur] + (size_t)s * 6;
      const float M[9] = {(float)md[0], (float)md[1], (float)md[2], (float)md[1], (float)md[3], (float)md[4], (float)md[2], (float)md[4], (float)md[5]};
      const double* mb = Mp.mean + (size_t)v * 3;
      const float e[3] = {__fsub_rn((float)mb[0], tx), __fsub_rn((float)mb[1], ty), __fsub_rn((float)mb[2], tz)};
      float Me[3];
#pragma unroll
      for (int r = 0; r < 3; r++) Me[r] = __fadd_rn(__fadd_rn(__fmul_rn(M[r * 3], e[0]), __fmul_rn(M[r * 3 + 1], e[1])), __fmul_rn(M[r * 3 + 2], e[2]));
      const float w = __fsqrt_rn((float)Mp.count[v]);
      trial = __fmul_rn(w, __fadd_rn(__fadd_rn(__fmul_rn(e[0], Me[0]), __fmul_rn(e[1], Me[1])), __fmul_rn(e[2], Me[2])));
    }
  }
  // ---- update_correspondences (DIRECT1) + linearize
  float h[21], bv[6], cost = 0.f;
#pragma unroll
  for (int i = 0; i < 21; i++) h[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 6; i++) bv[i] = 0.f;
  if (do_lin) {
    unsigned long long key;
    const int v = VcudaMapRule::cell(tx, ty, tz, Mp.res, &key) ? vgicp_probe(Mp, key) : -1;
    p.cpos[wset][s] = v;
    p.corr[wset][idx_bits(pt.w)] = v;
    if (v >= 0) {
      const double* ca = p.scov + (size_t)s * 6;
      const double* cb = Mp.cov + (size_t)v * 6;
      const double* mb = Mp.mean + (size_t)v * 3;
      const float CA[9] = {(float)ca[0], (float)ca[1], (float)ca[2], (float)ca[1], (float)ca[3], (float)ca[4], (float)ca[2], (float)ca[4], (float)ca[5]};
      const float R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
      float RC[9], m[9];
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++)
          RC[i * 3 + j] = __fadd_rn(__fadd_rn(__fmul_rn(R[i * 3], CA[j]), __fmul_rn(R[i * 3 + 1], CA[3 + j])), __fmul_rn(R[i * 3 + 2], CA[6 + j]));
      {
        int k = 0;
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
          for (int j = i; j < 3; j++, k++) {
            const float u = __fadd_rn(__fadd_rn(__fmul_rn(RC[i * 3], R[j * 3]), __fmul_rn(RC[i * 3 + 1], R[j * 3 + 1])), __fmul_rn(RC[i * 3 + 2], R[j * 3 + 2]));
            m[i * 3 + j] = m[j * 3 + i] = __fadd_rn((float)cb[k], u);
          }
      }
      // Eigen's 3x3 inverse: cofactor(i, j) = m(i1, j1) m(i2, j2) - m(i1, j2) m(i2, j1); det = (c00 m00 + c10 m10) + c20 m20;
      // inverse(i, j) = cofactor(j, i) * (1 / det).  m is symmetric, so the inverse is too, bit for bit
      float cof[9];
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) {
          const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
          cof[i * 3 + j] = __fsub_rn(__fmul_rn(m[i1 * 3 + j1], m[i2 * 3 + j2]), __fmul_rn(m[i1 * 3 + j2], m[i2 * 3 + j1]));
        }
      const float det = __fadd_rn(__fadd_rn(__fmul_rn(cof[0], m[0]), __fmul_rn(cof[3], m[3])), __fmul_rn(cof[6], m[6]));
      const float inv = __fdiv_rn(1.f, det);
      float M[9];
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) M[i * 3 + j] = __fmul_rn(cof[j * 3 + i], inv);
      double* mo = p.mahal[wset] + (size_t)s * 6;
      mo[0] = M[0]; mo[1] = M[1]; mo[2] = M[2]; mo[3] = M[4]; mo[4] = M[5]; mo[5] = M[8];
      const float w = __fsqrt_rn((float)Mp.count[v]);
      const float e[3] = {__fsub_rn((float)mb[0], tx), __fsub_rn((float)mb[1], ty), __fsub_rn((float)mb[2], tz)};
      float Me[3], MS[9];
#pragma unroll
      for (int r = 0; r < 3; r++) {
        Me[r] = __fadd_rn(__fadd_rn(__fmul_rn(M[r * 3], e[0]), __fmul_rn(M[r * 3 + 1], e[1])), __fmul_rn(M[r * 3 + 2], e[2]));
        // (M S)(r, c) = sum_k M(r, k) S(k, c) = (S^T m_r)_c with m_r = row r of M
#pragma unroll
        for (int c = 0; c < 3; c++) MS[r * 3 + c] = vcuda_skew_t(c, tx, ty, tz, M[r * 3], M[r * 3 + 1], M[r * 3 + 2]);
      }
      // H rotation block (a <= b): w (S^T (M S))(a, b); cross block: -(w (S^T M)(a, j)); translation block: w M
      int k = 0;
#pragma unroll
      for (int a = 0; a < 6; a++)
#pragma unroll
        for (int b = a; b < 6; b++, k++) {
          float x;
          if (a < 3 && b < 3) x = __fmul_rn(w, vcuda_skew_t(a, tx, ty, tz, MS[b], MS[3 + b], MS[6 + b]));
          else if (a < 3) x = -__fmul_rn(w, vcuda_skew_t(a, tx, ty, tz, M[b - 3], M[3 + b - 3], M[6 + b - 3]));
          else x = __fmul_rn(w, M[(a - 3) * 3 + (b - 3)]);
          h[k] = x;
        }
#pragma unroll
      for (int a = 0; a < 3; a++) bv[a] = __fmul_rn(w, vcuda_skew_t(a, tx, ty, tz, Me[0], Me[1], Me[2]));
#pragma unroll
      for (int a = 0; a < 3; a++) bv[3 + a] = -__fmul_rn(w, Me[a]);
      cost = __fmul_rn(w, __fadd_rn(__fadd_rn(__fmul_rn(e[0], Me[0]), __fmul_rn(e[1], Me[1])), __fmul_rn(e[2], Me[2])));
    }
  }
#define B2R_EMIT(i, v) red_emit<i, 28>((double)(v), tile, red, lane, warp)
  B2R_EMIT(0, h[0]); B2R_EMIT(1, h[1]); B2R_EMIT(2, h[2]); B2R_EMIT(3, h[3]); B2R_EMIT(4, h[4]); B2R_EMIT(5, h[5]); B2R_EMIT(6, h[6]);
  B2R_EMIT(7, h[7]); B2R_EMIT(8, h[8]); B2R_EMIT(9, h[9]); B2R_EMIT(10, h[10]); B2R_EMIT(11, h[11]); B2R_EMIT(12, h[12]); B2R_EMIT(13, h[13]);
  B2R_EMIT(14, h[14]); B2R_EMIT(15, h[15]); B2R_EMIT(16, h[16]); B2R_EMIT(17, h[17]); B2R_EMIT(18, h[18]); B2R_EMIT(19, h[19]);
  B2R_EMIT(20, h[20]); B2R_EMIT(21, bv[0]); B2R_EMIT(22, bv[1]); B2R_EMIT(23, bv[2]); B2R_EMIT(24, bv[3]); B2R_EMIT(25, bv[4]);
  B2R_EMIT(26, bv[5]); B2R_EMIT(27, cost); B2R_EMIT(28, trial);
#undef B2R_EMIT
  __syncthreads();
  if (threadIdx.x < kAcc) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < kAccThreads / 32; w++) v += red[threadIdx.x * 8 + w];
    p.partials[(size_t)threadIdx.x * (((unsigned)nblk + 31u) & ~31u) + blockIdx.x] = v;
  }
}
#endif  // __CUDACC__

}  // namespace b2r
