// gicp_pcl.cuh — the factory's `GICP` branch: pcl::GeneralizedIterativeClosestPoint (PCL 1.10) on the device (B2R_METHOD_GICP_PCL).
//
// Re-creates, GPU-first, what registrations.cpp:66-76 selects (semantics pinned by tests/gicp_pcl_ref.cpp, see its header):
//   k_pcl_cov_reg<20, PclCov> / k_pcl_cov<PclCov>  <- computeCovariances: k-NN (the point itself included) in ascending (d2, index) order, raw
//                                     moments in float64 with float32 products, cov -= mean mean^T, singular values (1, 1, gicp_epsilon)
//   k_gicp_pcl_corr                <- the correspondence loop of computeTransformation: q = transformation_ (guess p), exact 1-NN,
//                                     d2 < corr_dist^2 in float64, M = (R C1 R^T + C2)^-1 with Eigen's 3x3 inverse
//   k_gicp_pcl_cost                <- OptimizationFunctorWithIndices: the 13 sums behind f, df and fdf at one float32 pose
//   k_gicp_omp_cost                <- the same for pclomp::GeneralizedIterativeClosestPoint (B2R_METHOD_GICP_OMP, the factory's
//                                     GICP_OMP branch): the pose applyState(guess, x) moves the raw source point (OmpPose)
// The k-NN traversal and lists (bvh_group_search, KnnRegs, KnnList) and the fixed reduction tree (block_reduce / finish_partials) are
// shared with FastGICP's kernels; the BFGS driver (gicp_pcl_compute) runs on the host, one device pass per functor evaluation.
#pragma once
#include <array>
#include <cmath>
#include <cstring>
#include <limits>
#include "engine.cuh"
#include "gicp.cuh"

namespace b2r {

constexpr double kGicpPclEpsilon = 1e-3;  // gicp_epsilon_: the smallest singular value of every covariance
constexpr int kGicpPclThreads = 128;
constexpr int kGicpPclSums = 13;          // f, sum temp (3), sum p temp^T (9)

// computeCovariances for one point over its kk neighbours in ascending (d2, index) order: mean += p and cov(k, l) += p_k * p_l in
// float64, each product rounded to float32 (__fmul_rn: never contracted); / kk; cov -= mean mean^T; the normal n (eigenvector of the
// smallest eigenvalue) rebuilds the matrix as I - (1 - eps) n n^T.  Stores xx, xy, xz, yy, yz, zz.
template <class PtAt>
__device__ __forceinline__ void pcl_cov_store(int kk, PtAt pt_at, double* __restrict__ o) {
  double mx = 0, my = 0, mz = 0, c00 = 0, c10 = 0, c11 = 0, c20 = 0, c21 = 0, c22 = 0;
  for (int j = 0; j < kk; j++) {
    const float3 p = pt_at(j);
    mx = dadd(mx, (double)p.x); my = dadd(my, (double)p.y); mz = dadd(mz, (double)p.z);
    c00 = dadd(c00, (double)__fmul_rn(p.x, p.x));
    c10 = dadd(c10, (double)__fmul_rn(p.y, p.x));
    c11 = dadd(c11, (double)__fmul_rn(p.y, p.y));
    c20 = dadd(c20, (double)__fmul_rn(p.z, p.x));
    c21 = dadd(c21, (double)__fmul_rn(p.z, p.y));
    c22 = dadd(c22, (double)__fmul_rn(p.z, p.z));
  }
  const double kd = (double)kk;
  mx = __ddiv_rn(mx, kd); my = __ddiv_rn(my, kd); mz = __ddiv_rn(mz, kd);
  c00 = dsub(__ddiv_rn(c00, kd), dmul(mx, mx));
  c10 = dsub(__ddiv_rn(c10, kd), dmul(my, mx));
  c11 = dsub(__ddiv_rn(c11, kd), dmul(my, my));
  c20 = dsub(__ddiv_rn(c20, kd), dmul(mz, mx));
  c21 = dsub(__ddiv_rn(c21, kd), dmul(mz, my));
  c22 = dsub(__ddiv_rn(c22, kd), dmul(mz, mz));
  const double c[9] = {c00, c10, c20, c10, c11, c21, c20, c21, c22};
  double n[3];
  sym_min_eigvec3(c, n);
  const double w = 1.0 - kGicpPclEpsilon;
  o[0] = dsub(1.0, dmul(dmul(w, n[0]), n[0]));
  o[1] = -dmul(dmul(w, n[0]), n[1]);
  o[2] = -dmul(dmul(w, n[0]), n[2]);
  o[3] = dsub(1.0, dmul(dmul(w, n[1]), n[1]));
  o[4] = -dmul(dmul(w, n[1]), n[2]);
  o[5] = dsub(1.0, dmul(dmul(w, n[2]), n[2]));
}

// the moment rule of the kernels below: pcl GICP's (this file); FastVGICPCuda's float32 one is VcudaCov (vgicp_cuda.cuh)
struct PclCov {
  template <class PtAt>
  __device__ __forceinline__ static void store(int kk, PtAt pt_at, double* __restrict__ o) { pcl_cov_store(kk, pt_at, o); }
};

// k = 20 (reg_correspondence_randomness' default): register lists, one warp per leaf, as k_knn_cov_reg
template <int K, class Rule>
__device__ __forceinline__ void pcl_cov_reg_body(const Bvh& b, const float* __restrict__ raw, int stride_f, double* __restrict__ cov, int block_x) {
  __shared__ int nbr[K][kKnnThreads];
  const int s = block_x * blockDim.x + threadIdx.x;
  const int leaf = s >> 5;
  if (leaf >= b.nleaf) return;  // whole warps only
  const float4 q = b.sp[s];
  const bool active = idx_bits(q.w) != kPadIdx;
  KnnRegs<K> L;
  L.reset();
  bvh_group_search(b, q.x, q.y, q.z, active, L, leaf);
  if (!active) return;
#pragma unroll
  for (int j = 0; j < K; j++) nbr[j][threadIdx.x] = (int)(unsigned int)(L.key[j] & 0xffffffffull);
  const int tx = threadIdx.x;
  Rule::store(L.count(), [&](int j) {
    const float* p = raw + (size_t)nbr[j][tx] * stride_f;
    return make_float3(p[0], p[1], p[2]);
  }, cov + (size_t)s * 6);
}

template <int K, class Rule>
__global__ void __launch_bounds__(kKnnThreads, B2R_KNN_MINBLOCKS) k_pcl_cov_reg(Bvh b, const float* __restrict__ raw, int stride_f, double* __restrict__ cov) {
  pcl_cov_reg_body<K, Rule>(b, raw, stride_f, cov, blockIdx.x);
}

// the same for MANY clouds in one launch (blockIdx.y = cloud), as k_knn_cov_reg_batch
template <int K, class Rule>
__global__ void __launch_bounds__(kKnnThreads, B2R_KNN_BATCH_MINBLOCKS) k_pcl_cov_reg_batch(const KnnBatchItem* __restrict__ items) {
  const KnnBatchItem it = items[blockIdx.y];
  pcl_cov_reg_body<K, Rule>(it.b, it.raw, it.stride_f, it.cov, blockIdx.x);
}

// any k: per-lane lists in shared memory, as k_knn_cov
template <class Rule>
__global__ void __launch_bounds__(kKnnThreads, 4) k_pcl_cov(Bvh b, int k, const float* __restrict__ raw, int stride_f, double* __restrict__ cov) {
  extern __shared__ unsigned long long pcl_knn_keys[];  // [k][blockDim]
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int leaf = s >> 5;
  if (leaf >= b.nleaf) return;
  const float4 q = b.sp[s];
  const bool active = idx_bits(q.w) != kPadIdx;
  KnnList L;
  L.key = pcl_knn_keys + threadIdx.x;
  L.k = k;
  L.cnt = 0;
  L.stride = blockDim.x;
  L.wkey = kKeyInf;
  bvh_group_search(b, q.x, q.y, q.z, active, L, leaf);
  if (!active) return;
  const int stride = L.stride;
  const unsigned long long* keyp = L.key;
  Rule::store(L.cnt, [=](int j) {
    const int idx = (int)(unsigned int)(keyp[j * stride] & 0xffffffffull);
    const float* p = raw + (size_t)idx * stride_f;
    return make_float3(p[0], p[1], p[2]);
  }, cov + (size_t)s * 6);
}

struct GicpPclArgs {
  Bvh src, tgt;
  const double* scov;     // source covariances, sorted order, 6 per point
  const double* tcov;     // target covariances, sorted order
  float G[12];            // guess, rows of the 3x4 (applied to the source first: transformPointCloud(output, output, guess))
  float T[12];            // transformation_ (correspondence pass) or applyState(x) (cost pass)
  double R[9];            // top-left 3x3 of double(transformation_) * double(guess), row-major
  double thr2;            // corr_dist_threshold_^2
  int* corr;              // per source sorted position: the correspondent's TARGET SORTED position, -1 = none (the cost pass reads the
                          // target's BVH points, never its raw records: a promoted keyframe's records may be gone)
  double* M;              // per source sorted position: 9 doubles, row-major
  double* partials;
  double* out;            // host-mapped message
  unsigned int* counter;
  unsigned long long* flag;
  unsigned long long seq;
  unsigned int* round;    // batch: the round's message counter (the last message publishes the flag); nullptr alone
  unsigned int round_n;   // messages of the round
  unsigned int nrow;      // blocks of this pair (a batched launch's grid covers the largest pair); 0 = gridDim.x
};

// output_i = guess p (float32, transformPointCloud), as both passes compute it
__device__ __forceinline__ float3 gicp_pcl_output(const float* G, float x, float y, float z) {
  return make_float3(xform_row(G[0], G[1], G[2], G[3], x, y, z), xform_row(G[4], G[5], G[6], G[7], x, y, z),
                     xform_row(G[8], G[9], G[10], G[11], x, y, z));
}

// one thread per source sorted position (a warp = a leaf: spatial neighbours share the target leaves they visit)
__device__ __forceinline__ void gicp_pcl_corr_body(const GicpPclArgs& A) {
  __shared__ double red[32];
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const bool real = s < A.src.nleaf * kLeaf;
  float4 p = make_float4(0.f, 0.f, 0.f, bits_idx(kPadIdx));
  if (real) p = A.src.sp[s];
  float qx = 0.f, qy = 0.f, qz = 0.f;
  bool active = false;
  if (idx_bits(p.w) != kPadIdx) {
    const float3 o = gicp_pcl_output(A.G, p.x, p.y, p.z);
    qx = xform_row(A.T[0], A.T[1], A.T[2], A.T[3], o.x, o.y, o.z);
    qy = xform_row(A.T[4], A.T[5], A.T[6], A.T[7], o.x, o.y, o.z);
    qz = xform_row(A.T[8], A.T[9], A.T[10], A.T[11], o.x, o.y, o.z);
    active = finite3(qx, qy, qz);  // a non-finite query has no correspondence (engine rule, as k_fitness)
  }
  Nn1 v;
  v.reset(INFINITY);
  bvh_group_search(A.tgt, qx, qy, qz, active, v, -1);
  double cnt = 0.0;
  if (real) {
    int ci = -1;
    if (active && v.best_pos >= 0 && (double)v.best_d2() < A.thr2) {
      ci = v.best_pos;
      const double* a = A.scov + (size_t)s * 6;
      const double* b = A.tcov + (size_t)v.best_pos * 6;
      const double C1[9] = {a[0], a[1], a[2], a[1], a[3], a[4], a[2], a[4], a[5]};
      const double C2[9] = {b[0], b[1], b[2], b[1], b[3], b[4], b[2], b[4], b[5]};
      double RC[9], Tm[9];
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) RC[i * 3 + j] = dadd(dadd(dmul(A.R[i * 3], C1[j]), dmul(A.R[i * 3 + 1], C1[3 + j])), dmul(A.R[i * 3 + 2], C1[6 + j]));
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++)
          Tm[i * 3 + j] = dadd(dadd(dadd(dmul(RC[i * 3], A.R[j * 3]), dmul(RC[i * 3 + 1], A.R[j * 3 + 1])), dmul(RC[i * 3 + 2], A.R[j * 3 + 2])), C2[i * 3 + j]);
      // Eigen's 3x3 inverse: cofactor(i, j) = m(i1, j1) m(i2, j2) - m(i1, j2) m(i2, j1) (i1 = i+1, i2 = i+2 mod 3); det = the first
      // column's cofactors dotted with column 0; inverse(i, j) = cofactor(j, i) * (1 / det)
      double cof[9];
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) {
          const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
          cof[i * 3 + j] = dsub(dmul(Tm[i1 * 3 + j1], Tm[i2 * 3 + j2]), dmul(Tm[i1 * 3 + j2], Tm[i2 * 3 + j1]));
        }
      const double det = dadd(dadd(dmul(cof[0], Tm[0]), dmul(cof[3], Tm[3])), dmul(cof[6], Tm[6]));
      const double inv = __ddiv_rn(1.0, det);
      double* Mo = A.M + (size_t)s * 9;
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) Mo[i * 3 + j] = dmul(cof[j * 3 + i], inv);
      cnt = 1.0;
    }
    A.corr[s] = ci;
  }
  block_reduce<1>(&cnt, red);
  finish_partials<1>(&cnt, A.partials, A.out, A.counter, A.flag, A.seq, nullptr, A.nrow, A.round, A.round_n);
}

__global__ void __launch_bounds__(kGicpPclThreads) k_gicp_pcl_corr(const __grid_constant__ GicpPclArgs A) { gicp_pcl_corr_body(A); }

// many pairs: blockIdx.y = the pair's record; blocks beyond the pair's own count leave at once
__global__ void __launch_bounds__(kGicpPclThreads) k_gicp_pcl_corr_batch(const GicpPclArgs* __restrict__ recs) {
  const GicpPclArgs& A = recs[blockIdx.y];
  if (blockIdx.x >= A.nrow) return;
  gicp_pcl_corr_body(A);
}

// the pose rule of the cost pass: which point the functor's pose T moves.  pcl GICP (PCL 1.10) transforms the source by the guess
// first, so T = applyState(I, x) moves output_i = guess p; pclomp's GICP (B2R_METHOD_GICP_OMP) keeps base_transformation_ = guess, so
// T = applyState(guess, x) moves the raw source point (UPSTREAM-RECALL (DOUBT), tests/gicp_omp_ref.cpp; the host side is
// gicp_pcl::functor_pose)
struct PclPose {
  __device__ __forceinline__ static float3 point(float3 o, float4) { return o; }
};
struct OmpPose {
  __device__ __forceinline__ static float3 point(float3, float4 p) { return make_float3(p.x, p.y, p.z); }
};

// the fixed-tree reduction of a cost pass's 13 sums (outside the templated body below, so that pcl GICP's kernels keep their shared
// memory layout)
__device__ __forceinline__ void gicp_pcl_cost_reduce(double* acc, const GicpPclArgs& A) {
  __shared__ double red[kGicpPclSums * 32];
  block_reduce<kGicpPclSums>(acc, red);
  finish_partials<kGicpPclSums>(acc, A.partials, A.out, A.counter, A.flag, A.seq, nullptr, A.nrow, A.round, A.round_n);
}

// OptimizationFunctorWithIndices' loop body at the pose T over the accepted correspondences: res = (double)(T v - tgt) (float32
// difference, v = Pose::point), temp = M res, sums f += res^T temp, g += temp, dR += p_src temp^T (p_src = output_i, promoted)
template <class Pose>
__device__ __forceinline__ void gicp_pcl_cost_body(const GicpPclArgs& A) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  double acc[kGicpPclSums];
#pragma unroll
  for (int i = 0; i < kGicpPclSums; i++) acc[i] = 0.0;
  const int ci = s < A.src.nleaf * kLeaf ? A.corr[s] : -1;
  if (ci >= 0) {
    const float4 p = A.src.sp[s];
    const float3 o = gicp_pcl_output(A.G, p.x, p.y, p.z);
    const float3 v = Pose::point(o, p);
    const float4 q4 = A.tgt.sp[ci];
    const float q[3] = {q4.x, q4.y, q4.z};
    const double r[3] = {(double)fsub(xform_row(A.T[0], A.T[1], A.T[2], A.T[3], v.x, v.y, v.z), q[0]),
                         (double)fsub(xform_row(A.T[4], A.T[5], A.T[6], A.T[7], v.x, v.y, v.z), q[1]),
                         (double)fsub(xform_row(A.T[8], A.T[9], A.T[10], A.T[11], v.x, v.y, v.z), q[2])};
    const double* M = A.M + (size_t)s * 9;
    double t[3];
#pragma unroll
    for (int a = 0; a < 3; a++) t[a] = dadd(dadd(dmul(M[a * 3], r[0]), dmul(M[a * 3 + 1], r[1])), dmul(M[a * 3 + 2], r[2]));
    acc[0] = dadd(dadd(dmul(r[0], t[0]), dmul(r[1], t[1])), dmul(r[2], t[2]));
    acc[1] = t[0]; acc[2] = t[1]; acc[3] = t[2];
    const double pd[3] = {(double)o.x, (double)o.y, (double)o.z};
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
      for (int b = 0; b < 3; b++) acc[4 + a * 3 + b] = dmul(pd[a], t[b]);
  }
  gicp_pcl_cost_reduce(acc, A);
}

__global__ void __launch_bounds__(kGicpPclThreads) k_gicp_pcl_cost(const __grid_constant__ GicpPclArgs A) { gicp_pcl_cost_body<PclPose>(A); }

__global__ void __launch_bounds__(kGicpPclThreads) k_gicp_pcl_cost_batch(const GicpPclArgs* __restrict__ recs) {
  const GicpPclArgs& A = recs[blockIdx.y];
  if (blockIdx.x >= A.nrow) return;
  gicp_pcl_cost_body<PclPose>(A);
}

// the same two for pclomp's GICP (OmpPose)
__global__ void __launch_bounds__(kGicpPclThreads) k_gicp_omp_cost(const __grid_constant__ GicpPclArgs A) { gicp_pcl_cost_body<OmpPose>(A); }

__global__ void __launch_bounds__(kGicpPclThreads) k_gicp_omp_cost_batch(const GicpPclArgs* __restrict__ recs) {
  const GicpPclArgs& A = recs[blockIdx.y];
  if (blockIdx.x >= A.nrow) return;
  gicp_pcl_cost_body<OmpPose>(A);
}

// does this method's functor evaluate at applyState(guess, x) on the raw source (pclomp's GICP) rather than applyState(I, x) on
// guess p (pcl GICP)?
inline bool gicp_pcl_base_pose(int method) { return method == B2R_METHOD_GICP_OMP; }

// ------------------------------------------------------------------------------------------------ host side
// per-handle workspaces of the two passes
struct GicpPclWork {
  DevBuf<int> corr;
  DevBuf<double> M, partials;
  DevBuf<unsigned int> counter;  // 1 word, re-armed by finish_stored
  MappedBuf<double> msg;         // [0, 16) result message, [16] flag
  unsigned long long seq = 0;
  uint64_t m = 0;                // accepted correspondences of the last correspondence pass
  bool corr_valid = false;
  GicpPclArgs A;                 // inputs of the last correspondence pass (the cost pass reuses its clouds, guess and buffers)
};

inline int gicp_pcl_ensure_ws(GicpPclWork& W, size_t n_sorted, cudaStream_t st) {
  B2R_CUDA(W.corr.reserve(n_sorted + 1));
  B2R_CUDA(W.M.reserve(n_sorted * 9 + 9));
  B2R_CUDA(W.partials.reserve((n_sorted / kGicpPclThreads + 1) * kGicpPclSums));
  if (!W.counter.p) {
    B2R_CUDA(W.counter.alloc(1));
    B2R_CUDA(cudaMemsetAsync(W.counter.p, 0, sizeof(unsigned int), st));
  }
  if (!W.msg.p) {
    B2R_CUDA(W.msg.alloc(17));
    std::memset(W.msg.p, 0, 17 * sizeof(double));
  }
  return B2R_OK;
}

// the inputs of a correspondence pass of the pair (s, t) at (guess G, transformation_ T) with R = rel_rotation (row-major float 4x4s;
// the cost passes reuse the record with T replaced); corr / M: the pair's per-point buffers
inline void gicp_pcl_fill_args(const b2r_config& cfg, const Cloud& s, const Cloud& t, const float* G, const float* T, const double* R, int* corr,
                               double* M, GicpPclArgs& A) {
  std::memset(&A, 0, sizeof(A));
  A.src = s.bvh(); A.tgt = t.bvh(); A.scov = s.cov.p; A.tcov = t.cov.p;
  for (int i = 0; i < 12; i++) { A.G[i] = G[i]; A.T[i] = T[i]; }
  for (int i = 0; i < 9; i++) A.R[i] = R[i];
  A.thr2 = cfg.max_correspondence_distance * cfg.max_correspondence_distance;
  A.corr = corr; A.M = M;
}

// one pass of either kernel (the cost kernel of the method's pose rule); waits for its message and copies the NV result words to res
template <int NV>
inline int gicp_pcl_run(GicpPclWork& W, bool corr_pass, int method, Telemetry* tel, cudaStream_t st, double* res) {
  GicpPclArgs& A = W.A;
  A.partials = W.partials.p; A.counter = W.counter.p; A.out = W.msg.d;
  A.flag = reinterpret_cast<unsigned long long*>(W.msg.d + 16);
  A.seq = ++W.seq;
  const unsigned nb = (unsigned)((size_t)A.src.nsup * 1024 / kGicpPclThreads);
  TEL_BEGIN(tel, st);
  if (corr_pass) k_gicp_pcl_corr<<<nb, kGicpPclThreads, 0, st>>>(A);
  else if (gicp_pcl_base_pose(method)) k_gicp_omp_cost<<<nb, kGicpPclThreads, 0, st>>>(A);
  else k_gicp_pcl_cost<<<nb, kGicpPclThreads, 0, st>>>(A);
  TEL_END(tel, corr_pass ? KC_GICP_PCL_CORR : KC_GICP_PCL_COST, 1, st);
  B2R_CUDA(cudaGetLastError());
  int rc = wait_host_result(reinterpret_cast<unsigned long long*>(W.msg.p + 16), A.seq, W.msg.p, NV, false, st);
  if (rc) return rc;
  for (int i = 0; i < NV; i++) res[i] = W.msg.p[i];
  if (tel) tel->d2h += (NV + 2) * sizeof(double);
  return B2R_OK;
}

// row-major float 4x4 product ((a0 b0 + a1 b1) + a2 b2) + a3 b3, unfused (Eigen's Matrix4f product)
B2R_HD void gicp_pcl_mul4f(const float* A, const float* B, float* O) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) O[i * 4 + j] = fadd(fadd(fadd(fmul(A[i * 4], B[j]), fmul(A[i * 4 + 1], B[4 + j])), fmul(A[i * 4 + 2], B[8 + j])), fmul(A[i * 4 + 3], B[12 + j]));
}

// top-left 3x3 of PCL's float64 triple-loop product double(T_rel) * double(guess) (row-major float 4x4 in, row-major 3x3 out)
inline void gicp_pcl_rel_rotation(const float* Trel, const float* guess, double* R) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      double s = 0.0;
      for (int k = 0; k < 4; k++) s += double(Trel[i * 4 + k]) * double(guess[k * 4 + j]);
      R[i * 3 + j] = s;
    }
}

namespace gicp_pcl {

using V6 = std::array<double, 6>;
using Sums = std::array<double, kGicpPclSums>;
// the cost passes answered since the last checkpoint of a GicpPclPairState, replayed in order; a functor evaluation beyond them
// records its pose and unwinds (NeedPass)
struct Replay {
  std::vector<Sums> log;
  size_t idx = 0;
  float need_T[16];
};
struct NeedPass {};

inline double dot6(const V6& a, const V6& b) { double s = 0.0; for (int i = 0; i < 6; i++) s += a[i] * b[i]; return s; }
inline double norm6(const V6& a) { return std::sqrt(dot6(a, a)); }

// applyState(t = identity, x): R = AngleAxisf(x5, Z) * AngleAxisf(x4, Y) * AngleAxisf(x3, X) as float quaternions, then
// toRotationMatrix; translation (float)x0..2
inline void apply_state(const V6& x, float* T) {
  struct Q { float w, x, y, z; };
  auto aa = [](float a, int axis) { const float h = 0.5f * a, s = std::sin(h); Q q{std::cos(h), 0.f, 0.f, 0.f}; (axis == 0 ? q.x : axis == 1 ? q.y : q.z) = s; return q; };
  auto mul = [](const Q& a, const Q& b) {
    return Q{a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
             a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
  };
  const Q q = mul(mul(aa((float)x[5], 2), aa((float)x[4], 1)), aa((float)x[3], 0));
  const float tx = 2.f * q.x, ty = 2.f * q.y, tz = 2.f * q.z;
  const float twx = tx * q.w, twy = ty * q.w, twz = tz * q.w, txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y,
              tzz = tz * q.z;
  const float R[9] = {1.f - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1.f - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1.f - (txx + tyy)};
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[r * 4 + c] = R[r * 3 + c];
    T[r * 4 + 3] = (float)x[r];
  }
  T[12] = T[13] = T[14] = 0.f; T[15] = 1.f;
}

// the pose the functor evaluates at x (row-major float 4x4).  base == nullptr (pcl GICP): applyState(I, x).  Otherwise pclomp's
// applyState(base_transformation_ = guess, x): [R(x) R_g | t_g + t(x)], the 3x3 product in float32 ((a0 b0 + a1 b1) + a2 b2), the
// bottom row the guess's (UPSTREAM-RECALL (DOUBT), tests/gicp_omp_ref.cpp; the device side is OmpPose)
inline void functor_pose(const V6& x, const float* base, float* T) {
  apply_state(x, T);
  if (!base) return;
  float R[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) R[i * 3 + j] = fadd(fadd(fmul(T[i * 4], base[j]), fmul(T[i * 4 + 1], base[4 + j])), fmul(T[i * 4 + 2], base[8 + j]));
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) T[i * 4 + j] = R[i * 3 + j];
    T[i * 4 + 3] = fadd(base[i * 4 + 3], T[i * 4 + 3]);
  }
  for (int j = 0; j < 4; j++) T[12 + j] = base[12 + j];
}

// computeRDerivative: g[3..5] = <dR/dangle, Rsum> with matricesInnerProd(a, b) = sum_i sum_j a(j, i) b(i, j)
inline void r_derivative(const V6& x, const double* Rs, V6& g) {
  const double phi = x[3], theta = x[4], psi = x[5];
  const double cphi = std::cos(phi), sphi = std::sin(phi), ctheta = std::cos(theta), stheta = std::sin(theta), cpsi = std::cos(psi), spsi = std::sin(psi);
  double a[9], b[9], c[9];  // row-major dR_dPhi, dR_dTheta, dR_dPsi
  a[0] = 0.; a[3] = 0.; a[6] = 0.;
  a[1] = sphi * spsi + cphi * cpsi * stheta; a[4] = -cpsi * sphi + cphi * spsi * stheta; a[7] = cphi * ctheta;
  a[2] = cphi * spsi - cpsi * sphi * stheta; a[5] = -cphi * cpsi - sphi * spsi * stheta; a[8] = -ctheta * sphi;
  b[0] = -cpsi * stheta; b[3] = -spsi * stheta; b[6] = -ctheta;
  b[1] = cpsi * ctheta * sphi; b[4] = ctheta * sphi * spsi; b[7] = -sphi * stheta;
  b[2] = cphi * cpsi * ctheta; b[5] = cphi * ctheta * spsi; b[8] = -cphi * stheta;
  c[0] = -ctheta * spsi; c[3] = cpsi * ctheta; c[6] = 0.;
  c[1] = -cphi * cpsi - sphi * spsi * stheta; c[4] = -cphi * spsi + cpsi * sphi * stheta; c[7] = 0.;
  c[2] = cpsi * sphi - cphi * spsi * stheta; c[5] = sphi * spsi + cphi * cpsi * stheta; c[8] = 0.;
  auto inner = [&](const double* m1) {
    double r = 0.;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) r += m1[j * 3 + i] * Rs[i * 3 + j];
    return r;
  };
  g[3] = inner(a); g[4] = inner(b); g[5] = inner(c);
}

// OptimizationFunctorWithIndices over m correspondences; every evaluation is one device pass, except that an evaluation at the pose
// of the pass just before reuses its sums (df after operator() at the same x: the pass would return the same 13 sums)
struct Functor {
  Replay* R = nullptr;
  int m = 0;
  float base[16];            // the guess, when the pose rule is pclomp's (has_base)
  bool has_base = false;
  float lastT[16];
  double last[kGicpPclSums];
  bool have = false;
  int evaluations = 0, passes = 0;
  void sums(const V6& x, double* s) {
    float T[16];
    functor_pose(x, has_base ? base : nullptr, T);
    evaluations++;
    if (!(have && std::memcmp(T, lastT, sizeof(T)) == 0)) {
      if (R->idx == R->log.size()) {
        std::memcpy(R->need_T, T, sizeof(T));
        throw NeedPass{};
      }
      std::memcpy(last, R->log[R->idx++].data(), sizeof(last));
      std::memcpy(lastT, T, sizeof(T));
      have = true;
      passes++;
    }
    std::memcpy(s, last, sizeof(last));
  }
  void grad_from(const V6& x, const double* s, V6& g) {
    g = V6{0, 0, 0, 0, 0, 0};
    const double k = 2.0 / m;
    for (int i = 0; i < 3; i++) g[i] = s[1 + i] * k;
    double R[9];
    for (int i = 0; i < 9; i++) R[i] = s[4 + i] * k;
    r_derivative(x, R, g);
  }
  double f(const V6& x) { double s[kGicpPclSums]; sums(x, s); return s[0] / m; }
  void df(const V6& x, V6& g) { double s[kGicpPclSums]; sums(x, s); grad_from(x, s, g); }
  void fdf(const V6& x, double& fv, V6& g) { double s[kGicpPclSums]; sums(x, s); fv = s[0] / m; grad_from(x, s, g); }
};

enum Status { NegativeGradientEpsilon = -3, NotStarted = -2, Running = -1, Success = 0, NoProgress = 1 };

// pcl/registration/bfgs.h (PCL 1.10): BFGS with Fletcher's bracketing / sectioning line search (after GSL's vector_bfgs2)
struct Bfgs {
  Functor fn;
  double rho = 0.01, sigma = 0.01, tau1 = 9, tau2 = 0.05, tau3 = 0.5, step_size = 1;
  int order = 3, bracket_iters = 100, section_iters = 100;
  double f = 0, delta_f = 0, fp0 = 0, pnorm = 0, g0norm = 0;
  V6 gradient{}, x0{}, dx0{}, dg0{}, g0{}, dx{}, p{}, x_alpha{}, g_alpha{};
  double f_alpha = 0, df_alpha = 0, x_cache_key = 0, f_cache_key = 0, df_cache_key = 0, g_cache_key = 0;
  Bfgs() = default;

  static double poly_eval(const double* c, double x) {  // Eigen::poly_eval of c0 + c1 x + c2 x^2 + c3 x^3
    if (x * x <= 1.0) {
      double v = c[3];
      for (int i = 2; i >= 0; i--) v = v * x + c[i];
      return v;
    }
    double v = c[0];
    const double ix = 1.0 / x;
    for (int i = 1; i < 4; i++) v = v * ix + c[i];
    return std::pow(x, 3.0) * v;
  }
  static int solve_quadratic(double a, double b, double c, double* x0, double* x1) {  // gsl_poly_solve_quadratic
    if (a == 0) {
      if (b == 0) return 0;
      *x0 = -c / b;
      return 1;
    }
    const double disc = b * b - 4 * a * c;
    if (disc > 0) {
      if (b == 0) {
        const double r = std::sqrt(-c / a);
        *x0 = -r; *x1 = r;
      } else {
        const double sgnb = (b > 0 ? 1 : -1);
        const double temp = -0.5 * (b + sgnb * std::sqrt(disc));
        const double r1 = temp / a, r2 = c / temp;
        if (r1 < r2) { *x0 = r1; *x1 = r2; } else { *x0 = r2; *x1 = r1; }
      }
      return 2;
    }
    if (disc == 0) { *x0 = -0.5 * b / a; *x1 = -0.5 * b / a; return 2; }
    return 0;
  }
  static double interpolate(double a, double fa, double fpa, double b, double fb, double fpb, double xmin, double xmax, int order) {
    double ymin = (xmin - a) / (b - a), ymax = (xmax - a) / (b - a), y, fmin;
    if (ymin > ymax) std::swap(ymin, ymax);
    if (order > 2 && !(fpb != fpb) && fpb != std::numeric_limits<double>::infinity()) {
      fpa = fpa * (b - a);
      fpb = fpb * (b - a);
      const double eta = 3 * (fb - fa) - 2 * fpa - fpb, xi = fpa + fpb - 2 * (fb - fa);
      const double c[4] = {fa, fpa, eta, xi};
      y = ymin;
      fmin = poly_eval(c, ymin);
      auto check = [&](double z) { const double v = poly_eval(c, z); if (v < fmin) { y = z; fmin = v; } };
      check(ymax);
      double y0 = 0, y1 = 0;
      const int n = solve_quadratic(3 * c[3], 2 * c[2], c[1], &y0, &y1);
      if (n == 2) {
        if (y0 > y1) std::swap(y0, y1);
        if (y0 > ymin && y0 < ymax) check(y0);
        if (y1 > ymin && y1 < ymax) check(y1);
      } else if (n == 1) {
        if (y0 > ymin && y0 < ymax) check(y0);
      }
    } else {
      fpa = fpa * (b - a);
      const double fl = fa + ymin * (fpa + ymin * (fb - fa - fpa));
      const double fh = fa + ymax * (fpa + ymax * (fb - fa - fpa));
      const double c = 2 * (fb - fa - fpa);
      y = ymin;
      fmin = fl;
      if (fh < fmin) { y = ymax; fmin = fh; }
      if (c > 0) {
        const double z = -fpa / c;
        if (z > ymin && z < ymax) {
          const double fz = fa + z * (fpa + z * (fb - fa - fpa));
          if (fz < fmin) { y = z; fmin = fz; }
        }
      }
    }
    return a + y * (b - a);
  }
  void move_to(double alpha) {
    for (int i = 0; i < 6; i++) x_alpha[i] = x0[i] + alpha * p[i];
    x_cache_key = alpha;
  }
  double slope() const { return dot6(g_alpha, p); }
  double apply_f(double alpha) {
    if (alpha == f_cache_key) return f_alpha;
    move_to(alpha);
    f_alpha = fn.f(x_alpha);
    f_cache_key = alpha;
    return f_alpha;
  }
  double apply_df(double alpha) {
    if (alpha == df_cache_key) return df_alpha;
    move_to(alpha);
    if (alpha != g_cache_key) {
      fn.df(x_alpha, g_alpha);
      g_cache_key = alpha;
    }
    df_alpha = slope();
    df_cache_key = alpha;
    return df_alpha;
  }
  void apply_fdf(double alpha, double& fv, double& dfv) {
    if (alpha == f_cache_key && alpha == df_cache_key) { fv = f_alpha; dfv = df_alpha; return; }
    if (alpha == f_cache_key || alpha == df_cache_key) { fv = apply_f(alpha); dfv = apply_df(alpha); return; }
    move_to(alpha);
    fn.fdf(x_alpha, f_alpha, g_alpha);
    f_cache_key = alpha; g_cache_key = alpha;
    df_alpha = slope();
    df_cache_key = alpha;
    fv = f_alpha; dfv = df_alpha;
  }
  void change_direction() {
    x_alpha = x0; x_cache_key = 0.0;
    f_cache_key = 0.0;
    g_alpha = g0; g_cache_key = 0.0;
    df_alpha = slope(); df_cache_key = 0.0;
  }
  int line_search(double alpha1, double& alpha_new) {
    double f0, fp0l, falpha, falpha_prev, fpalpha, fpalpha_prev, delta, alpha_next;
    double alpha = alpha1, alpha_prev = 0.0, a, b, fa, fb, fpa, fpb;
    int i = 0;
    apply_fdf(0.0, f0, fp0l);
    falpha_prev = f0; fpalpha_prev = fp0l;
    a = 0.0; b = alpha; fa = f0; fb = 0.0; fpa = fp0l; fpb = 0.0;
    while (i++ < bracket_iters) {
      falpha = apply_f(alpha);
      if (falpha > f0 + alpha * rho * fp0l || falpha >= falpha_prev) {
        a = alpha_prev; fa = falpha_prev; fpa = fpalpha_prev;
        b = alpha; fb = falpha; fpb = std::numeric_limits<double>::quiet_NaN();
        break;
      }
      fpalpha = apply_df(alpha);
      if (std::fabs(fpalpha) <= -sigma * fp0l) { alpha_new = alpha; return Success; }
      if (fpalpha >= 0) {
        a = alpha; fa = falpha; fpa = fpalpha;
        b = alpha_prev; fb = falpha_prev; fpb = fpalpha_prev;
        break;
      }
      delta = alpha - alpha_prev;
      alpha_next = interpolate(alpha_prev, falpha_prev, fpalpha_prev, alpha, falpha, fpalpha, alpha + delta, alpha + tau1 * delta, order);
      alpha_prev = alpha; falpha_prev = falpha; fpalpha_prev = fpalpha;
      alpha = alpha_next;
    }
    while (i++ < section_iters) {
      delta = b - a;
      alpha = interpolate(a, fa, fpa, b, fb, fpb, a + tau2 * delta, b - tau3 * delta, order);
      falpha = apply_f(alpha);
      if ((a - alpha) * fpa <= std::numeric_limits<double>::epsilon()) return NoProgress;  // roundoff prevents progress
      if (falpha > f0 + rho * alpha * fp0l || falpha >= fa) {
        b = alpha; fb = falpha; fpb = std::numeric_limits<double>::quiet_NaN();
      } else {
        fpalpha = apply_df(alpha);
        if (std::fabs(fpalpha) <= -sigma * fp0l) { alpha_new = alpha; return Success; }
        if (((b - a) >= 0 && fpalpha >= 0) || ((b - a) <= 0 && fpalpha <= 0)) {
          b = a; fb = fa; fpb = fpa;
          a = alpha; fa = falpha; fpa = fpalpha;
        } else {
          a = alpha; fa = falpha; fpa = fpalpha;
        }
      }
    }
    return Success;
  }
  int minimize_init(const V6& x) {
    delta_f = 0;
    dx = V6{};
    fn.fdf(x, f, gradient);
    x0 = x;
    g0 = gradient;
    g0norm = norm6(g0);
    for (int i = 0; i < 6; i++) p[i] = gradient[i] * -1 / g0norm;
    pnorm = norm6(p);
    fp0 = -g0norm;
    x_alpha = x0; x_cache_key = 0;
    f_alpha = f; f_cache_key = 0;
    g_alpha = g0; g_cache_key = 0;
    df_alpha = slope(); df_cache_key = 0;
    return NotStarted;
  }
  int minimize_one_step(V6& x) {
    double alpha = 0.0, alpha1;
    const double f0 = f;
    if (pnorm == 0.0 || g0norm == 0.0 || fp0 == 0) { dx = V6{}; return NoProgress; }
    if (delta_f < 0) {
      const double del = std::max(-delta_f, 10 * std::numeric_limits<double>::epsilon() * std::fabs(f0));
      alpha1 = std::min(1.0, 2.0 * del / (-fp0));
    } else {
      alpha1 = std::fabs(step_size);
    }
    const int status = line_search(alpha1, alpha);
    if (status != Success) return status;
    {  // updatePosition
      double fv, dfv;
      apply_fdf(alpha, fv, dfv);
      f = f_alpha; x = x_alpha; gradient = g_alpha;
    }
    delta_f = f - f0;
    for (int i = 0; i < 6; i++) { dx0[i] = x[i] - x0[i]; dg0[i] = gradient[i] - g0[i]; }
    dx = dx0;
    const double dxg = dot6(dx0, gradient), dgg = dot6(dg0, gradient), dxdg = dot6(dx0, dg0), dgnorm = norm6(dg0);
    double A = 0, B = 0;
    if (dxdg != 0) {
      B = dxg / dxdg;
      A = -(1.0 + dgnorm * dgnorm / dxdg) * B + dgg / dxdg;
    }
    for (int i = 0; i < 6; i++) { p[i] = -A * dx0[i]; p[i] += -B * dg0[i]; p[i] += gradient[i]; }
    g0 = gradient;
    x0 = x;
    g0norm = norm6(g0);
    pnorm = norm6(p);
    const double dir = (dot6(p, gradient) > 0) ? -1.0 : 1.0;
    for (int i = 0; i < 6; i++) p[i] *= dir / pnorm;
    pnorm = norm6(p);
    fp0 = dot6(p, g0);
    change_direction();
    return Success;
  }
  int test_gradient(double eps) const {
    if (eps < 0) return NegativeGradientEpsilon;
    return norm6(gradient) < eps ? Success : Running;
  }
};

}  // namespace gicp_pcl

// GeneralizedIterativeClosestPoint::computeTransformation (PCL 1.10, and pclomp's copy of it for B2R_METHOD_GICP_OMP, whose cost
// passes are at applyState(guess, x): Functor::base) as a resumable state machine.  next() names the pass the
// registration needs — correspondences at (guess, T()) or a cost pass at T() — and consume_*() hands it the result, so one pair runs
// alone (the single handle) or beside many others whose passes share launches (the batch), through the same statements.
// Inside BFGS the state is checkpointed before every minimizeOneStep: a step that needs a cost pass unwinds and is re-run from its
// checkpoint with the passes answered so far (a few evaluations per step), never from the start of the registration.
class GicpPclPairState {
 public:
  enum Need { CORR, COST, DONE };
  GicpPclPairState() = default;
  void start(const b2r_config& cfg, const float* guess_row) {
    cfg_ = cfg;
    std::memcpy(G_, guess_row, sizeof(G_));
    ck_ = W();
    rep_.log.clear();
    need_ = CORR;
    advance();
  }
  // the pass the registration needs next
  Need next() const { return need_; }
  // CORR: transformation_ (row-major 4x4); COST: the pose of the cost pass
  const float* T() const { return need_ == CORR ? ck_.Tcur : rep_.need_T; }
  const float* guess() const { return G_; }
  // CORR: the top-left 3x3 of double(transformation_) double(guess)
  void rel_rotation(double* R) const { gicp_pcl_rel_rotation(ck_.Tcur, G_, R); }
  void consume_corr(uint64_t m) {
    W& w = ck_;
    std::memcpy(w.Tprev, w.Tcur, sizeof(w.Tprev));  // previous_transformation_ = transformation_
    if (m < 4) { finish(); return; }                  // NotEnoughPointsException, caught as a PCLException: not converged
    // estimateRigidTransformationBFGS: x seeded from transformation_ (atan2 on floats, asin on the promoted double)
    w.x = gicp_pcl::V6{(double)w.Tcur[3], (double)w.Tcur[7], (double)w.Tcur[11], (double)std::atan2(w.Tcur[9], w.Tcur[10]),
                       std::asin(-(double)w.Tcur[8]), (double)std::atan2(w.Tcur[4], w.Tcur[0])};
    w.bfgs = gicp_pcl::Bfgs();
    w.bfgs.fn.m = (int)m;
    if (gicp_pcl_base_pose(cfg_.method)) {  // pclomp: the functor's poses are applyState(guess, x)
      std::memcpy(w.bfgs.fn.base, G_, sizeof(G_));
      w.bfgs.fn.has_base = true;
    }
    w.phase = P_INIT;
    rep_.log.clear();
    advance();
  }
  void consume_cost(const double* sums) {
    gicp_pcl::Sums a;
    std::memcpy(a.data(), sums, sizeof(a));
    rep_.log.push_back(a);
    advance();
  }
  // results (valid at DONE)
  float Tfinal[16];
  bool converged = false;
  int nr_iterations = 0;
  int bfgs_steps = 0, evaluations = 0, corr_passes = 0, cost_passes = 0;

 private:
  enum Phase { P_CORR, P_INIT, P_STEP };
  struct W {
    Phase phase = P_CORR;
    float Tcur[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};  // transformation_
    float Tprev[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};  // previous_transformation_
    int outer = 0, inner = 0, steps = 0, evals = 0, passes = 0, corrs = 0;
    bool conv = false;
    gicp_pcl::V6 x{};
    gicp_pcl::Bfgs bfgs;
  };
  void finish() {
    const W& w = ck_;
    gicp_pcl_mul4f(w.Tprev, G_, Tfinal);  // final_transformation_ = previous_transformation_ * guess
    converged = w.conv;
    nr_iterations = w.outer;
    bfgs_steps = w.steps; evaluations = w.evals; cost_passes = w.passes; corr_passes = w.corrs;
    need_ = DONE;
  }
  // the end of estimateRigidTransformationBFGS and of the outer iteration
  void end_bfgs(W& w, int result) {
    using namespace gicp_pcl;
    w.evals += w.bfgs.fn.evaluations; w.passes += w.bfgs.fn.passes;
    w.bfgs.fn.evaluations = w.bfgs.fn.passes = 0;
    if (!(result == NoProgress || result == Success || w.inner == cfg_.max_optimizer_iterations)) {  // SolverDidntConvergeException
      ck_ = w;
      finish();
      return;
    }
    apply_state(w.x, w.Tcur);
    double delta = 0.;
    for (int k = 0; k < 4; k++)
      for (int l = 0; l < 4; l++) {
        const double ratio = (k < 3 && l < 3) ? 1. / cfg_.rotation_epsilon : 1. / cfg_.transformation_epsilon;
        const double c = ratio * std::fabs(w.Tprev[k * 4 + l] - w.Tcur[k * 4 + l]);
        if (c > delta) delta = c;
      }
    w.outer++;
    if (w.outer >= cfg_.max_iterations || delta < 1) {
      w.conv = true;
      std::memcpy(w.Tprev, w.Tcur, sizeof(w.Tprev));
      ck_ = w;
      finish();
      return;
    }
    w.phase = P_CORR;
    ck_ = w;
  }
  // runs from the checkpoint until the next pass is needed (or the registration ends)
  void advance() {
    using namespace gicp_pcl;
    for (;;) {
      if (ck_.phase == P_CORR) {
        if (need_ != DONE) { ck_.corrs++; need_ = CORR; }
        return;
      }
      W w = ck_;
      w.bfgs.fn.R = &rep_;
      rep_.idx = 0;
      try {
        if (w.phase == P_INIT) {
          w.bfgs.minimize_init(w.x);
          w.inner = 0;
          w.phase = P_STEP;
        } else {
          w.inner++;
          w.steps++;
          int result = w.bfgs.minimize_one_step(w.x);
          if (!result) result = w.bfgs.test_gradient(1e-2);
          if (result != Running || w.inner >= cfg_.max_optimizer_iterations) {
            rep_.log.clear();
            end_bfgs(w, result);
            if (need_ == DONE) return;
            continue;
          }
        }
      } catch (const NeedPass&) {
        need_ = COST;
        return;
      }
      rep_.log.clear();
      ck_ = w;
    }
  }
  b2r_config cfg_{};
  float G_[16];
  W ck_;
  gicp_pcl::Replay rep_;
  Need need_ = DONE;
};

}  // namespace b2r
