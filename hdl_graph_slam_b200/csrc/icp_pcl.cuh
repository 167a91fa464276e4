// icp_pcl.cuh — the factory's `ICP` branch: pcl::IterativeClosestPoint (PCL 1.10) on the device (B2R_METHOD_ICP_PCL).
//
// Re-creates computeTransformation (semantics pinned by tests/icp_pcl_ref.cpp, see its header).  The whole loop stays on the device:
//   k_icp_search   <- transformCloud(input_transformed, transformation_) of the previous step, in place, then determineCorrespondences:
//                     exact 1-NN in the target, accepted when d2 <= max_dist^2 (float64 compare); without the reciprocal check it also
//                     reduces (count, sum d2, sum src, sum tgt) and its last block takes the means
//   k_icp_refit    <- (reciprocal) the tight boxes of the moved source over its unchanged leaves and super-nodes
//   k_icp_reverse  <- (reciprocal) the 1-NN of each accepted pair's target point in the moved source: kept when it is the query itself
//                     within max_dist; then the same reduction as above
//   k_icp_step     <- the demeaned cross products; the last block runs pcl::umeyama (icp_umeyama), final = transformation_ * final,
//                     ++nr_iterations_ and DefaultConvergenceCriteria (icp_has_converged)
// Each pair keeps its moved source in the BVH's own sorted float4 layout, so a warp is still a source leaf.  Every kernel takes one
// pair per blockIdx.y; a finished pair's blocks leave at once, so rounds can be enqueued ahead of the device.
#pragma once
#include <algorithm>
#include <cstring>
#include <vector>
#include "engine.cuh"
#include "gicp.cuh"
#include "gicp_pcl.cuh"
#include "linalg.cuh"

namespace b2r {

constexpr int kIcpThreads = 128;
constexpr int kIcpStats = 8;   // count, sum d2, sum src (3), sum tgt (3)
constexpr int kIcpCross = 9;   // sum (tgt - tmean)_i (src - smean)_j
enum IcpState { ICP_FIRST = 0, ICP_STEP = 1, ICP_DONE = 2 };

struct IcpPairDev {
  Bvh src, tgt;               // the source's own structure (original coordinates) and the target's
  Bvh moved;                  // the moved source: sp = `tsp`, boxes = the refitted ones (reciprocal)
  float4* tsp;                // input_transformed per sorted source position (w = original index bits)
  float4 *leaf_lo, *leaf_hi, *sup_lo, *sup_hi;
  int* corr;                  // per sorted source position: the target SORTED position of the accepted correspondence, -1 = none
  float* d2;                  // per sorted source position: the forward d2
  double* partials;           // [blocks][9]
  unsigned int* counter;
  double* msg;                // [kIcpCross + 2]: the last block's sums (finish_partials' result words and checksum)
  float G[16];                // guess, row-major
  float T[16];                // final_transformation_, row-major
  float inc[16];              // transformation_ of the last step, row-major
  float smean[3], tmean[3];
  double sums[kIcpStats + kIcpCross];
  double thr2, rot_thr, trans_thr, prev_mse, mse;
  int n_corr, max_iterations, iterations, state, converged, reciprocal, guess_identity, nrow, rounds, pad;
};

// input_transformed of sorted position s after this round's transform (written back in place)
__device__ __forceinline__ float4 icp_move(IcpPairDev& p, int s) {
  float4 q;
  if (p.state == ICP_FIRST) {
    q = p.src.sp[s];
    if (idx_bits(q.w) != kPadIdx && !p.guess_identity) {
      const float* G = p.G;
      const float x = q.x, y = q.y, z = q.z;
      q.x = xform_row(G[0], G[1], G[2], G[3], x, y, z); q.y = xform_row(G[4], G[5], G[6], G[7], x, y, z); q.z = xform_row(G[8], G[9], G[10], G[11], x, y, z);
    }
  } else {
    q = p.tsp[s];
    if (idx_bits(q.w) != kPadIdx) {
      const float* M = p.inc;
      const float x = q.x, y = q.y, z = q.z;
      q.x = xform_row(M[0], M[1], M[2], M[3], x, y, z); q.y = xform_row(M[4], M[5], M[6], M[7], x, y, z); q.z = xform_row(M[8], M[9], M[10], M[11], x, y, z);
    }
  }
  p.tsp[s] = q;
  return q;
}

// the correspondence statistics of one round; the last block takes the means (or ends the align below 3 correspondences)
__device__ __forceinline__ void icp_stats(IcpPairDev& p, bool ok, float4 q, int c, float d2) {
  __shared__ double red[kIcpStats * 32];
  __shared__ unsigned long long last;
  double acc[kIcpStats];
#pragma unroll
  for (int i = 0; i < kIcpStats; i++) acc[i] = 0.0;
  if (ok) {
    const float4 t = p.tgt.sp[c];
    acc[0] = 1.0; acc[1] = (double)d2;
    acc[2] = (double)q.x; acc[3] = (double)q.y; acc[4] = (double)q.z;
    acc[5] = (double)t.x; acc[6] = (double)t.y; acc[7] = (double)t.z;
  }
  if (threadIdx.x == 0) last = 0;
  block_reduce<kIcpStats>(acc, red);
  finish_partials<kIcpStats>(acc, p.partials, p.msg, p.counter, &last, 1ull, nullptr, p.nrow);
  __syncthreads();
  if (last == 1ull && threadIdx.x == 0) {
    const double* S = p.msg;
    for (int i = 0; i < kIcpStats; i++) p.sums[i] = S[i];
    const double n = S[0];
    p.n_corr = (int)n;
    p.rounds++;
    if (n < 3.0) {  // min_number_correspondences_: converged_ = false, final_transformation_ as it stands
      p.converged = 0;
      p.state = ICP_DONE;
      return;
    }
    for (int k = 0; k < 3; k++) { p.smean[k] = (float)(S[2 + k] / n); p.tmean[k] = (float)(S[5 + k] / n); }
    p.mse = S[1] / n;
  }
}

// one thread per source sorted position (a warp = a leaf of the source)
__global__ void __launch_bounds__(kIcpThreads) k_icp_search(IcpPairDev* __restrict__ pairs) {
  IcpPairDev& p = pairs[blockIdx.y];
  if (p.state == ICP_DONE || blockIdx.x >= (unsigned)p.nrow) return;
  const int s = blockIdx.x * kIcpThreads + threadIdx.x;
  const float4 q = icp_move(p, s);
  const bool active = idx_bits(q.w) != kPadIdx && finite3(q.x, q.y, q.z);
  Nn1 v;
  v.reset(INFINITY);
  bvh_group_search(p.tgt, q.x, q.y, q.z, active, v, -1);
  const bool ok = active && v.best_pos >= 0 && !((double)v.best_d2() > p.thr2);
  p.corr[s] = ok ? v.best_pos : -1;
  p.d2[s] = v.best_d2();
  if (!p.reciprocal) icp_stats(p, ok, q, v.best_pos, v.best_d2());
}

// one block of 1024 threads per super-node of the moved source: leaf and super-node boxes from the moved coordinates
__global__ void __launch_bounds__(1024) k_icp_refit(IcpPairDev* __restrict__ pairs) {
  IcpPairDev& p = pairs[blockIdx.y];
  if (p.state == ICP_DONE || blockIdx.x >= (unsigned)p.src.nsup) return;
  __shared__ float s_lo[32][3], s_hi[32][3];
  const int s = blockIdx.x * 1024 + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float4 q = p.tsp[s];
  const bool valid = idx_bits(q.w) != kPadIdx;
  float lx = valid ? q.x : INFINITY, ly = valid ? q.y : INFINITY, lz = valid ? q.z : INFINITY;
  float hx = valid ? q.x : -INFINITY, hy = valid ? q.y : -INFINITY, hz = valid ? q.z : -INFINITY;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lx = fminf(lx, __shfl_xor_sync(0xffffffffu, lx, o)); ly = fminf(ly, __shfl_xor_sync(0xffffffffu, ly, o)); lz = fminf(lz, __shfl_xor_sync(0xffffffffu, lz, o));
    hx = fmaxf(hx, __shfl_xor_sync(0xffffffffu, hx, o)); hy = fmaxf(hy, __shfl_xor_sync(0xffffffffu, hy, o)); hz = fmaxf(hz, __shfl_xor_sync(0xffffffffu, hz, o));
  }
  if (lane == 0) {
    const int leaf = blockIdx.x * 32 + warp;
    p.leaf_lo[leaf] = make_float4(lx, ly, lz, 0.f);
    p.leaf_hi[leaf] = make_float4(hx, hy, hz, 0.f);
    s_lo[warp][0] = lx; s_lo[warp][1] = ly; s_lo[warp][2] = lz;
    s_hi[warp][0] = hx; s_hi[warp][1] = hy; s_hi[warp][2] = hz;
  }
  __syncthreads();
  if (warp == 0) {
    float ax = s_lo[lane][0], ay = s_lo[lane][1], az = s_lo[lane][2], bx = s_hi[lane][0], by = s_hi[lane][1], bz = s_hi[lane][2];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ax = fminf(ax, __shfl_xor_sync(0xffffffffu, ax, o)); ay = fminf(ay, __shfl_xor_sync(0xffffffffu, ay, o)); az = fminf(az, __shfl_xor_sync(0xffffffffu, az, o));
      bx = fmaxf(bx, __shfl_xor_sync(0xffffffffu, bx, o)); by = fmaxf(by, __shfl_xor_sync(0xffffffffu, by, o)); bz = fmaxf(bz, __shfl_xor_sync(0xffffffffu, bz, o));
    }
    if (lane == 0) {
      p.sup_lo[blockIdx.x] = make_float4(ax, ay, az, 0.f);
      p.sup_hi[blockIdx.x] = make_float4(bx, by, bz, 0.f);
    }
  }
}

// determineReciprocalCorrespondences' second search: target point j of an accepted pair i -> 1-NN among the moved source
__global__ void __launch_bounds__(kIcpThreads) k_icp_reverse(IcpPairDev* __restrict__ pairs) {
  IcpPairDev& p = pairs[blockIdx.y];
  if (p.state == ICP_DONE || blockIdx.x >= (unsigned)p.nrow) return;
  const int s = blockIdx.x * kIcpThreads + threadIdx.x;
  const int c = p.corr[s];
  const float4 q = p.tsp[s];
  float qx = 0.f, qy = 0.f, qz = 0.f;
  if (c >= 0) { const float4 t = p.tgt.sp[c]; qx = t.x; qy = t.y; qz = t.z; }
  Nn1 v;
  v.reset(INFINITY);
  bvh_group_search(p.moved, qx, qy, qz, c >= 0, v, -1, s >> 5);  // the query's own source leaf first (ordering only)
  const bool ok = c >= 0 && !((double)v.best_d2() > p.thr2) && v.best_idx() == idx_bits(q.w);
  if (!ok) p.corr[s] = -1;
  icp_stats(p, ok, q, c, p.d2[s]);
}

// sigma's float64 sums, then the step in the last block
__global__ void __launch_bounds__(kIcpThreads) k_icp_step(IcpPairDev* __restrict__ pairs) {
  IcpPairDev& p = pairs[blockIdx.y];
  if (p.state == ICP_DONE || blockIdx.x >= (unsigned)p.nrow) return;
  __shared__ double red[kIcpCross * 32];
  __shared__ unsigned long long last;
  const int s = blockIdx.x * kIcpThreads + threadIdx.x;
  const int c = p.corr[s];
  double acc[kIcpCross];
#pragma unroll
  for (int i = 0; i < kIcpCross; i++) acc[i] = 0.0;
  if (c >= 0) {
    const float4 q = p.tsp[s], t = p.tgt.sp[c];
    const double sd[3] = {(double)fsub(q.x, p.smean[0]), (double)fsub(q.y, p.smean[1]), (double)fsub(q.z, p.smean[2])};
    const double dd[3] = {(double)fsub(t.x, p.tmean[0]), (double)fsub(t.y, p.tmean[1]), (double)fsub(t.z, p.tmean[2])};
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
      for (int j = 0; j < 3; j++) acc[i * 3 + j] = dmul(dd[i], sd[j]);
  }
  if (threadIdx.x == 0) last = 0;
  block_reduce<kIcpCross>(acc, red);
  finish_partials<kIcpCross>(acc, p.partials, p.msg, p.counter, &last, 1ull, nullptr, p.nrow);
  __syncthreads();
  if (last == 1ull && threadIdx.x == 0) {
    const double n = p.sums[0];
    float sigma[9], Rt[16], F[16];
    for (int i = 0; i < 9; i++) { p.sums[kIcpStats + i] = p.msg[i]; sigma[i] = (float)(p.msg[i] / n); }
    icp_umeyama(sigma, p.smean, p.tmean, Rt);
    gicp_pcl_mul4f(Rt, p.T, F);
    for (int i = 0; i < 16; i++) { p.inc[i] = Rt[i]; p.T[i] = F[i]; }
    p.iterations++;
    double prev = p.prev_mse;
    const bool conv = icp_has_converged(Rt, p.iterations, p.max_iterations, p.rot_thr, p.trans_thr, p.mse, &prev);
    p.prev_mse = prev;
    p.converged = conv ? 1 : 0;
    p.state = conv ? ICP_DONE : ICP_STEP;
  }
}

// ------------------------------------------------------------------------------------------------ host side
// per pair: moved source, correspondences, d2, refitted boxes, reduction partials, counter and message
struct IcpPairWs { size_t tsp, corr, d2, leaf_lo, leaf_hi, sup_lo, sup_hi, partials, counter, msg, bytes; };
inline size_t icp_align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
inline IcpPairWs icp_pair_ws(const Cloud& s) {
  const size_t n = (size_t)s.nsup * 1024, nl = (size_t)s.nsup * kSuper, ns = (size_t)s.nsup, nb = n / kIcpThreads;
  IcpPairWs w;
  w.tsp = 0;
  w.corr = w.tsp + icp_align_up(n * sizeof(float4), 256);
  w.d2 = w.corr + icp_align_up(n * sizeof(int), 256);
  w.leaf_lo = w.d2 + icp_align_up(n * sizeof(float), 256);
  w.leaf_hi = w.leaf_lo + icp_align_up(nl * sizeof(float4), 256);
  w.sup_lo = w.leaf_hi + icp_align_up(nl * sizeof(float4), 256);
  w.sup_hi = w.sup_lo + icp_align_up(ns * sizeof(float4), 256);
  w.partials = w.sup_hi + icp_align_up(ns * sizeof(float4), 256);
  w.counter = w.partials + icp_align_up((nb + 1) * kIcpCross * sizeof(double), 256);
  w.msg = w.counter + 256;
  w.bytes = w.msg + icp_align_up((kIcpCross + 2) * sizeof(double), 256);
  return w;
}

// the record of pair (s, t) at the column-major float guess, with its workspace at `base` (counter zeroed by the caller)
inline void icp_fill_pair(const b2r_config& cfg, const Cloud& s, const Cloud& t, const float* guess_col, char* base, IcpPairDev& P) {
  std::memset(&P, 0, sizeof(P));
  const IcpPairWs w = icp_pair_ws(s);
  P.src = s.bvh(); P.tgt = t.bvh();
  P.tsp = reinterpret_cast<float4*>(base + w.tsp);
  P.leaf_lo = reinterpret_cast<float4*>(base + w.leaf_lo); P.leaf_hi = reinterpret_cast<float4*>(base + w.leaf_hi);
  P.sup_lo = reinterpret_cast<float4*>(base + w.sup_lo); P.sup_hi = reinterpret_cast<float4*>(base + w.sup_hi);
  P.moved = P.src;
  P.moved.sp = P.tsp; P.moved.leaf_lo = P.leaf_lo; P.moved.leaf_hi = P.leaf_hi; P.moved.sup_lo = P.sup_lo; P.moved.sup_hi = P.sup_hi;
  P.corr = reinterpret_cast<int*>(base + w.corr);
  P.d2 = reinterpret_cast<float*>(base + w.d2);
  P.partials = reinterpret_cast<double*>(base + w.partials);
  P.counter = reinterpret_cast<unsigned int*>(base + w.counter);
  P.msg = reinterpret_cast<double*>(base + w.msg);
  bool ident = true;
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) {
      const float g = guess_col[c * 4 + r];
      P.G[r * 4 + c] = g;
      P.T[r * 4 + c] = g;  // final_transformation_ = guess
      ident = ident && g == (r == c ? 1.0f : 0.0f);
    }
  P.guess_identity = ident ? 1 : 0;
  P.thr2 = cfg.max_correspondence_distance * cfg.max_correspondence_distance;
  P.trans_thr = cfg.transformation_epsilon;
  P.rot_thr = 1.0 - cfg.transformation_epsilon;
  P.prev_mse = DBL_MAX;
  P.max_iterations = cfg.max_iterations;
  P.reciprocal = cfg.use_reciprocal_correspondences ? 1 : 0;
  P.nrow = (int)((size_t)s.nsup * 1024 / kIcpThreads);
  P.state = ICP_FIRST;
}

// one round of computeTransformation for every pair of d_pairs: 2 launches, 4 with the reciprocal check (steps = false: the
// correspondence launches only, as the parity taps want them)
inline int icp_enqueue_round(IcpPairDev* d_pairs, unsigned n, unsigned max_nrow, unsigned max_nsup, bool reciprocal, bool step, Telemetry* tel,
                             cudaStream_t st) {
  TEL_BEGIN(tel, st);
  const dim3 g(max_nrow, n);
  k_icp_search<<<g, kIcpThreads, 0, st>>>(d_pairs);
  if (reciprocal) {
    k_icp_refit<<<dim3(max_nsup, n), 1024, 0, st>>>(d_pairs);
    k_icp_reverse<<<g, kIcpThreads, 0, st>>>(d_pairs);
  }
  if (step) k_icp_step<<<g, kIcpThreads, 0, st>>>(d_pairs);
  TEL_END(tel, KC_ICP_PCL, (reciprocal ? 3 : 1) + (step ? 1 : 0), st);
  B2R_CUDA(cudaGetLastError());
  return B2R_OK;
}

// Run the pairs h_pairs[0..n) (records already at d_pairs) until every one is done.  `predicted` rounds are enqueued at once (the
// previous align's count: consecutive frames need about the same); a finished pair's surplus rounds exit at once, a shortfall is
// topped up after one look at the records, doubling each time.  h_pairs receives the final records.
inline int icp_run(IcpPairDev* d_pairs, IcpPairDev* h_pairs, unsigned n, int predicted, Telemetry* tel, cudaStream_t st, int* rounds_out) {
  unsigned max_nrow = 1, max_nsup = 1;
  bool reciprocal = false;
  int max_it = 1;
  for (unsigned i = 0; i < n; i++) {
    max_nrow = std::max(max_nrow, (unsigned)h_pairs[i].nrow);
    max_nsup = std::max(max_nsup, (unsigned)h_pairs[i].src.nsup);
    reciprocal = reciprocal || h_pairs[i].reciprocal;
    max_it = std::max(max_it, h_pairs[i].max_iterations);
  }
  int enq = 0, batch = std::max(1, std::min(predicted, max_it + 1));
  for (;;) {
    for (int r = 0; r < batch; r++) {
      int rc = icp_enqueue_round(d_pairs, n, max_nrow, max_nsup, reciprocal, true, tel, st);
      if (rc) return rc;
    }
    enq += batch;
    B2R_CUDA(cudaMemcpyAsync(h_pairs, d_pairs, n * sizeof(IcpPairDev), cudaMemcpyDeviceToHost, st));
    B2R_CUDA(cudaStreamSynchronize(st));
    if (tel) tel->d2h += n * sizeof(IcpPairDev);
    bool all = true;
    for (unsigned i = 0; i < n; i++) all = all && h_pairs[i].state == ICP_DONE;
    if (all) break;
    if (enq > max_it + 1) return fail(B2R_ECUDA, "ICP rounds ran past max_iterations without finishing");
    batch = std::min(2 * batch, max_it + 1 - enq + 1);
    batch = std::max(batch, 1);
  }
  if (rounds_out) *rounds_out = enq;
  return B2R_OK;
}

}  // namespace b2r
