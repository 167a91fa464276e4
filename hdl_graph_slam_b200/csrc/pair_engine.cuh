// pair_engine.cuh — device-resident GICP registration of MANY (source, target) pairs per launch.
//
// What it replaces: fast_gicp::LsqRegistration::computeTransformation / step_lm driving FastGICP::linearize / compute_error
// (SURVEY.md A.4), i.e. everything `registration->align()` does for the GICP engine at
// /root/reference/apps/scan_matching_odometry_nodelet.cpp:210 and /root/reference/include/hdl_graph_slam/loop_detector.hpp:143,
// plus the `getFitnessScore(max_range)` that follows every loop-closure align (loop_detector.hpp:146).
//
// Design (GPU-first, SURVEY.md §0.5 / §7 "iteration control on device"):
//   * every pair in flight owns a PairDev record in HBM: the two clouds' search structures, its double-buffered
//     correspondence sets, and the COMPLETE Levenberg-Marquardt state (pose, H, b, lambda, nu, counters);
//   * ONE round = three launches that cover ALL active pairs (blockIdx.y = slot): k_pair_search (exact seeded 1-NN of every
//     transformed source point), k_pair_accumulate (float64 linearisation fused with the trial cost of the previous
//     correspondence set; block partials) and k_pair_lm (one small block per pair: adds the pair's partials in a fixed order
//     and runs the LM step itself — 6x6 LDL^T, se3_exp, rho test, lambda update, convergence test).  The host never sees H or b;
//   * rounds are enqueued ahead; a finished pair's blocks exit at once.  The host reads back one word per round (batch mode:
//     number of pairs still active) or nothing at all until the result record lands in mapped memory (single-pair mode);
//   * reductions depend only on the pair's own geometry, so a pair's result is bitwise identical whether it runs alone
//     (b2r_align), in a batch of 2048, or on another GPU.
#pragma once
#include <cfloat>
#include "gicp.cuh"

namespace b2r {

enum PairMode : int { PM_IDLE = 0, PM_FIRST = 1, PM_FUSED = 2, PM_ERR = 3, PM_FIT = 4, PM_DONE = 5 };

struct LmCfg {
  int max_iterations;      // reg_maximum_iterations (registrations.cpp:32)
  double rot_eps;          // fast_gicp rotation_epsilon_
  double trans_eps;        // reg_transformation_epsilon (:31)
  double thr2;             // reg_max_correspondence_distance^2 (:33), compared with (double)d2
  float lim;               // float >= thr2: range limit of the 1-NN search
  int want_fitness;        // 1: one more round evaluates getFitnessScore(fit_max_range) at the final pose
  double fit_max_range;    // compared with the SQUARED distance (information_matrix_calculator.cpp:69)
  float fit_lim;           // float > fit_max_range (or +inf)
  int index_seed;          // first iteration: seed with the target point of the same firing index
};

// what the host reads back per pair (128 bytes)
struct PairReport {
  b2r_result r;            // 80 bytes: T (column-major float), fitness, converged, iterations
  double y0;               // cost of the last accepted linearisation
  int cur;                 // buffer set holding the correspondences of the last accepted linearisation
  int rounds;              // search+accumulate rounds executed
  int lm_failed;           // "lm not converged!!" exit
  int pad0;
  double tap[3];           // free (keeps the record at 128 bytes)
};
static_assert(sizeof(PairReport) == 128, "PairReport layout");

struct PairDev {
  // geometry (read-only during the registration)
  Bvh src, tgt;
  const double* scov;
  const double* tcov;
  const int* tgt_pos_of;
  int tgt_n;
  int nblk_acc;            // accumulate blocks of this pair = padded source points / kAccThreads
  // workspaces
  int* corr[2];
  int* cpos[2];
  double* mahal[2];
  float* d2;
  double* partials;        // [kAcc][nblk_acc rounded up to 32] (transposed)
  // where results go
  PairReport* report;      // device memory (batch) or host-mapped memory (single pair)
  unsigned long long* flag;      // host-mapped: publication flag of `report` (checksummed message), or nullptr
  unsigned long long* progress;  // host-mapped: (seq << 16) | rounds executed, or nullptr
  double* tap_out;         // parity taps (b2r_gicp_linearize_at / b2r_gicp_error_at): the 29 reduced values go here, no LM step
  unsigned long long seq;
  // control
  unsigned int counter;
  int mode;                // PairMode of the NEXT round
  int tap;
  int rounds;
  // Levenberg-Marquardt state (fast_gicp step_lm)
  double xe[12];           // pose the next round evaluates (rows 0..2 of the 4x4)
  double x0[12];           // last accepted pose
  double H[21], b[6], d[6];
  double y0, lambda, nu;
  int it, li, cur, wc, delta_conv, converged, lm_failed;
  int have_seed;           // 1 once a correspondence set exists in buffer set `cur` (seeds of the next search)
};

// ------------------------------------------------------------------------------------------------ message publication
// (msg_mix, the position-dependent checksum term, lives in common.cuh)

// The LM step functions below are __host__ __device__: the device runs them in the last block of k_pair_accumulate, and
// tests/lm_harness.cu drives their host build on the CPU against the oracle's step_lm (no GPU needed).  The two builds are not the
// same arithmetic: the device may contract the plain float64 products of ldlt6_solve / se3_exp / mul_iso into FMAs.  Replayed over
// the same round sums (tests/test_device_numerics_gpu.py) they take the same decisions, with lambda and nu within 1e-12 relative and
// the pose within 1e-12 of its largest entry.
// report (16 words) -> dst, checksum -> dst[16]; flag = seq.  No system-scope fences: the host accepts the message only when
// it is self-consistent (wait_report).
B2R_HD void publish_report(const PairReport& rep, PairReport* dst, unsigned long long* flag, unsigned long long seq) {
  const unsigned long long* w = reinterpret_cast<const unsigned long long*>(&rep);
  volatile unsigned long long* o = reinterpret_cast<volatile unsigned long long*>(dst);
  unsigned long long x = seq;
#pragma unroll
  for (int i = 0; i < 15; i++) { o[i] = w[i]; x ^= msg_mix(w[i], i); }
  if (flag) {
    o[15] = x;  // last word of the record (tap[2]) carries the checksum in host-mapped publications
    *reinterpret_cast<volatile unsigned long long*>(flag) = seq;
  } else {
    o[15] = w[15];
  }
}

// ------------------------------------------------------------------------------------------------ LM step on the device
__host__ __device__ inline void lm_finish(PairDev& p, const LmCfg& c) {
  p.mode = c.want_fitness ? PM_FIT : PM_DONE;
#pragma unroll
  for (int i = 0; i < 12; i++) p.xe[i] = p.x0[i];  // the fitness round evaluates the final pose
}

__host__ __device__ inline void lm_publish(PairDev& p, double fitness) {
  PairReport rep;
  // final_transformation_ = x0.cast<float>(), handed out column-major like Eigen::Matrix4f::data()
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int cc = 0; cc < 4; cc++) rep.r.T[cc * 4 + r] = (float)p.x0[r * 4 + cc];
  rep.r.T[3] = 0.f; rep.r.T[7] = 0.f; rep.r.T[11] = 0.f; rep.r.T[15] = 1.f;
  rep.r.fitness = fitness;
  rep.r.converged = p.converged;
  rep.r.iterations = p.it;
  rep.y0 = p.y0;
  rep.cur = p.cur;
  rep.rounds = p.rounds;
  rep.lm_failed = p.lm_failed;
  rep.pad0 = 0;
  rep.tap[0] = rep.tap[1] = rep.tap[2] = 0.0;
  publish_report(rep, p.report, p.flag, p.seq);
}

// solve (H + lambda I) d = -b, delta = se3_exp(d), xi = delta * x0; false = singular / non-finite step
__host__ __device__ inline bool lm_propose(PairDev& p, const LmCfg& c) {
  double A[36], nb[6], d[6];
#pragma unroll
  for (int r = 0; r < 6; r++)
#pragma unroll
    for (int cc = r; cc < 6; cc++) {
      const double v = p.H[r * 6 - r * (r - 1) / 2 + (cc - r)];  // upper-triangle packing: row r starts at 6r - r(r-1)/2
      A[r * 6 + cc] = v; A[cc * 6 + r] = v;
    }
#pragma unroll
  for (int i = 0; i < 6; i++) { A[i * 7] += p.lambda; nb[i] = -p.b[i]; }
  bool solved = ldlt6_solve(A, nb, d);
#pragma unroll
  for (int i = 0; i < 6; i++) solved = solved && isfinite(d[i]);
  if (!solved) return false;
  double delta[16], x0[16], xi[16];
  se3_exp(d, delta);
#pragma unroll
  for (int i = 0; i < 12; i++) x0[i] = p.x0[i];
  x0[12] = x0[13] = x0[14] = 0.0; x0[15] = 1.0;
  mul_iso(delta, x0, xi);
#pragma unroll
  for (int i = 0; i < 12; i++) p.xe[i] = xi[i];
#pragma unroll
  for (int i = 0; i < 6; i++) p.d[i] = d[i];
  p.delta_conv = gicp_is_converged(delta, c.rot_eps, c.trans_eps) ? 1 : 0;
  // the next linearisation exists only if this step does not converge and the iteration cap is not reached: then the trial
  // cost and the next linearize(xi) are one fused pass, otherwise only compute_error(xi) runs
  p.wc = (!p.delta_conv && (p.it + 1 < c.max_iterations)) ? 1 : 0;
  // PM_ERR = the LAST trial of the registration unless it is rejected: with want_fitness its round also searches at xi (as the
  // fitness round would) so an accepted final step needs no separate getFitnessScore round
  p.mode = p.wc ? PM_FUSED : PM_ERR;
  return true;
}

// top of LsqRegistration's outer loop: for (it; it < max_iterations && !converged; it++)
__host__ __device__ inline void lm_begin_outer(PairDev& p, const LmCfg& c) {
  if (!(p.it < c.max_iterations) || p.converged) { lm_finish(p, c); return; }
  if (p.lambda < 0.0) {
    double mx = 0.0;
    const int diag[6] = {0, 6, 11, 15, 18, 20};
    for (int i = 0; i < 6; i++) { const double v = fabs(p.H[diag[i]]); mx = (mx < v) ? v : mx; }
    p.lambda = 1e-9 * mx;
  }
  p.nu = 2.0;
  p.li = 0;
  if (!lm_propose(p, c)) {  // "lm not converged!!": the pose keeps its last valid value
    p.it++;
    p.lm_failed = 1;
    lm_finish(p, c);
  }
}

// r[0..20] upper H, r[21..26] b, r[27] cost of the new linearisation, r[28] trial cost with the previous correspondences
// (PM_FIT: r[0] = sum of squared NN distances within range, r[1] = their count)
__host__ __device__ inline void lm_advance(PairDev& p, const double* r, const LmCfg& c) {
  const int mode = p.mode;
  p.rounds++;
  if (p.tap) {  // parity tap: hand the reduced values out, no LM step
    for (int i = 0; i < kAcc; i++) p.tap_out[i] = r[i];
    p.mode = PM_DONE;
    lm_publish(p, NAN);
    return;
  }
  if (mode == PM_FIT) {
    p.mode = PM_DONE;
    lm_publish(p, r[1] > 0.0 ? r[0] / r[1] : DBL_MAX);
    return;
  }
  if (mode == PM_FIRST) {
    p.have_seed = 1;
    for (int i = 0; i < 21; i++) p.H[i] = r[i];
    for (int i = 0; i < 6; i++) p.b[i] = r[21 + i];
    p.y0 = r[27];
    lm_begin_outer(p, c);
  } else {  // PM_FUSED / PM_ERR: one LM trial has been evaluated at xe
    const double yi = r[28];
    const bool fit_ready = (mode == PM_ERR) && c.want_fitness;  // r[0], r[1] = fitness sums at xe (valid if xe becomes the final pose)
    double den = 0.0;
    for (int i = 0; i < 6; i++) den += p.d[i] * (p.lambda * p.d[i] - p.b[i]);
    const double rho = (p.y0 - yi) / den;
    bool outer_done = false, accepted = false;
    if (rho < 0.0) {
      if (p.delta_conv) {
        outer_done = true;  // ok = true, x0 unchanged
      } else {
        p.lambda = p.nu * p.lambda;
        p.nu = 2.0 * p.nu;
        p.li++;
        if (p.li >= 10 || !lm_propose(p, c)) {  // inner loop exhausted or singular step: "lm not converged!!"
          p.it++;
          p.lm_failed = 1;
          lm_finish(p, c);
        }
        // else: the speculative linearisation in the other buffer set is simply dropped; next trial next round
      }
    } else {
      const double tt = 2.0 * rho - 1.0;
      const double f = 1.0 - tt * tt * tt;
      p.lambda = p.lambda * ((1.0 / 3.0 < f) ? f : 1.0 / 3.0);
      accepted = true;
      for (int i = 0; i < 12; i++) p.x0[i] = p.xe[i];
      if (p.wc) {  // adopt the linearisation at the accepted pose: it IS the next iteration's linearize(x0)
        p.cur ^= 1;
        for (int i = 0; i < 21; i++) p.H[i] = r[i];
        for (int i = 0; i < 6; i++) p.b[i] = r[21 + i];
        p.y0 = r[27];
      }
      outer_done = true;
    }
    if (outer_done) {
      p.converged = p.delta_conv;
      p.it++;
      lm_begin_outer(p, c);
      // the registration ended with xe accepted as the final pose: its fitness sums are already in hand
      if (p.mode == PM_FIT && fit_ready && accepted) {
        p.mode = PM_DONE;
        lm_publish(p, r[1] > 0.0 ? r[0] / r[1] : DBL_MAX);
        if (p.progress) *reinterpret_cast<volatile unsigned long long*>(p.progress) = (p.seq << 16) | (unsigned long long)(p.rounds & 0xffff);
        return;
      }
    }
  }
  if (p.mode == PM_DONE) lm_publish(p, NAN);
  if (p.progress) *reinterpret_cast<volatile unsigned long long*>(p.progress) = (p.seq << 16) | (unsigned long long)(p.rounds & 0xffff);
}

#ifdef __CUDACC__
// ------------------------------------------------------------------------------------------------ round kernels
// update_correspondences for every active pair: exact 1-NN of every transformed source point in the pair's target.
// C lanes per query (bvh.cuh): C = 4 shortens the per-warp chain (single pair: the kernel time is the slowest warp),
// C = 1 minimises instructions per query (batches: thousands of warps per SM-slot, throughput is what counts).
#ifndef B2R_SEARCH_MINBLOCKS
#define B2R_SEARCH_MINBLOCKS 8
#endif
template <int C>
__global__ void __launch_bounds__(kLinThreads, B2R_SEARCH_MINBLOCKS) k_pair_search(PairDev* pairs, const int* __restrict__ active, const __grid_constant__ LmCfg cfg) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  // batch mode: active[0] = number of pairs still in flight, active[1..] = their indices (k_pair_compact, previous round); the host
  // sizes grid.y from a count that may be one round stale, so surplus rows exit here
  if (active && (int)blockIdx.y >= active[0]) return;
  PairDev& p = pairs[active ? active[1 + blockIdx.y] : blockIdx.y];
  const int mode = p.mode;
  // PM_ERR (compute_error only) has no correspondence update; with want_fitness it runs the fitness search at the same pose
  const bool fit_search = mode == PM_FIT || (mode == PM_ERR && cfg.want_fitness);
  if (mode != PM_FIRST && mode != PM_FUSED && !fit_search) return;
  constexpr int Q = 32 / C;
  const int gt = blockIdx.x * blockDim.x + threadIdx.x;
  const int n_sorted = p.src.nleaf * kLeaf;
  const int s = (gt >> 5) * Q + (gt & (Q - 1));
  if ((gt >> 5) * Q >= n_sorted) return;  // whole warps only
  const bool writer = (gt & 31) < Q;
  const int cur = p.cur;
  const int wset = (mode == PM_FIRST) ? cur : (cur ^ 1);
  const bool use_seed = p.have_seed != 0;  // false in the first round of an align and in a stand-alone fitness evaluation
  const float lim = fit_search ? cfg.fit_lim : cfg.lim;
  const double thr2 = fit_search ? (double)INFINITY : cfg.thr2;
  Bvh tgt = p.tgt;
  const float4 pt = p.src.sp[s];
  const bool is_point = idx_bits(pt.w) != kPadIdx;
  float qx = 0.f, qy = 0.f, qz = 0.f;
  Nn1K v;  // packed-key visitor: the position of the winner comes from the target's pos_of table afterwards
  v.reset(lim);
  bool active_q = false;
  int sp0 = -1;
  if (is_point) {
    // fast_gicp: trans.cast<float>() * point (float32, no FMA)
    qx = xform_row((float)p.xe[0], (float)p.xe[1], (float)p.xe[2], (float)p.xe[3], pt.x, pt.y, pt.z);
    qy = xform_row((float)p.xe[4], (float)p.xe[5], (float)p.xe[6], (float)p.xe[7], pt.x, pt.y, pt.z);
    qz = xform_row((float)p.xe[8], (float)p.xe[9], (float)p.xe[10], (float)p.xe[11], pt.x, pt.y, pt.z);
    if (finite3(qx, qy, qz)) {
      active_q = true;
      // a seed is a REAL candidate (its exact distance and index enter the visitor like any other): a tight upper bound from
      // the last accepted correspondences, or a heuristic one from the firing order on the first iteration
      if (use_seed) sp0 = p.cpos[cur][s];
      else if (cfg.index_seed) { const int oi = idx_bits(pt.w); if (oi < p.tgt_n) sp0 = p.tgt_pos_of[oi]; }
      if (sp0 >= 0) {
        const float4 t = tgt.sp[sp0];
        v.seed(dist2_f32(qx, qy, qz, t.x, t.y, t.z), idx_bits(t.w), sp0);
      }
    }
  }
  int hint = -1;
  {
    const bool good = sp0 >= 0 && (use_seed || v.best_d2() < 1.0f);
    const unsigned hm = __ballot_sync(0xffffffffu, good);
    if (hm) hint = __shfl_sync(0xffffffffu, sp0, __fns(hm, 0, (__popc(hm) + 1) / 2)) >> 5;
  }
  bvh_group_search<C>(tgt, qx, qy, qz, active_q, v, -1, hint);  // all 32 lanes participate
  if (is_point && writer) {
    const bool valid = active_q && v.found() && ((double)v.best_d2() < thr2);
    if (!fit_search) p.corr[wset][idx_bits(pt.w)] = valid ? v.best_idx() : -1;
    p.cpos[wset][s] = valid ? p.tgt_pos_of[v.best_idx()] : -1;
    p.d2[s] = v.best_d2();
  }
}

// One value of the block reduction, consumed as soon as it is produced.  (Streaming the 29 values instead of holding 29 float64
// accumulators until the end keeps the kernel under 96 registers: 3 blocks of 256 threads per SM instead of 2 — the pass is
// bound by gather latency, so residency is throughput.)  A butterfly per value is 10 SHFL per lane and value: 290 per warp, which
// saturated the shared-memory / shuffle data path (ncu r2g: l1tex data-pipe wavefronts 81 % of peak, half of them shuffles).
// Instead the warp TRANSPOSES through shared memory: every lane stores its value into row (i mod 8) of the warp's tile; after 8
// values, lane l adds elements q, q + 4, ..., q + 28 (q = l & 3) of row l >> 2 and two shuffle levels join the four partial
// sums — 2 store + 2 load + 0.5 shuffle wavefronts per value instead of 10.  The order of the additions is fixed.
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
constexpr int kRedRow = 36;  // float64 elements per tile row: rows 0..3 of a half-warp start 4 banks apart
__device__ __forceinline__ void red_flush(int phase, int count, double* tile, double* red, int lane, int warp) {
  __syncwarp();
  const int r = lane >> 2, q = lane & 3;
  double v = 0.0;
  if (r < count) {
    const double* row = tile + r * kRedRow + q;
#pragma unroll
    for (int t = 0; t < 8; t++) v += row[4 * t];
  }
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  if (q == 0 && r < count) red[(phase * 8 + r) * 8 + warp] = v;
  __syncwarp();
}
template <int I, int LAST>
__device__ __forceinline__ void red_emit(double v, double* tile, double* red, int lane, int warp) {
  tile[(I & 7) * kRedRow + lane] = v;
  if ((I & 7) == 7 || I == LAST) red_flush(I >> 3, (I & 7) + 1, tile, red, lane, warp);
}

// linearize (float64) at xe into the write set + compute_error of the previous set, per active pair.  Every block leaves its
// 29 partial sums in the pair's `partials`; k_pair_lm (next launch) adds them in a fixed order and takes the LM step.
#ifndef B2R_ACC_MINBLOCKS
#define B2R_ACC_MINBLOCKS 4  // 64 registers, 32 warps per SM: the pass is bound by gather latency
#endif
__global__ void __launch_bounds__(kAccThreads, B2R_ACC_MINBLOCKS) k_pair_accumulate(PairDev* pairs, const int* __restrict__ active, const __grid_constant__ LmCfg cfg) {
  __shared__ double red[kAcc * 8];
  __shared__ double tiles[(kAccThreads / 32) * 8 * kRedRow];
  asm volatile("griddepcontrol.wait;" ::: "memory");
  // single-pair mode: let the (tiny) LM kernel of this round become resident now, so that it starts the moment this grid drains
  if (!active) asm volatile("griddepcontrol.launch_dependents;");
  if (active && (int)blockIdx.y >= active[0]) return;
  PairDev& p = pairs[active ? active[1 + blockIdx.y] : blockIdx.y];
  const int mode = p.mode;
  if (mode < PM_FIRST || mode > PM_FIT) return;
  const int nblk = p.nblk_acc;
  if ((int)blockIdx.x >= nblk) return;
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* tile = tiles + warp * 8 * kRedRow;
  const int cur = p.cur;
  const int wset = (mode == PM_FIRST) ? cur : (cur ^ 1);
  float4 pt = make_float4(0.f, 0.f, 0.f, bits_idx(kPadIdx));
  if (s < p.src.nleaf * kLeaf) pt = p.src.sp[s];
  const bool is_point = idx_bits(pt.w) != kPadIdx;
  if (!is_point) { pt.x = 0.f; pt.y = 0.f; pt.z = 0.f; }  // padding entries carry +inf coordinates: inf * 0 would poison the sums below
  // The pass is bound by memory latency (ncu r2k: long-scoreboard stalls 16 per issued instruction): a point's loads form the chain
  // pair record -> cpos -> gathers (target point, target covariance), twice (trial cost, then linearisation).  Read both cpos
  // entries first and PREFETCH every record the two parts will touch, so the chain is paid once, not per part.
  const bool do_trial = (mode == PM_FUSED || mode == PM_ERR) && is_point;
  const bool do_lin = (mode == PM_FIRST || mode == PM_FUSED) && is_point;
  const bool fit = mode == PM_FIT || (mode == PM_ERR && cfg.want_fitness);
  const int tp = do_trial ? p.cpos[cur][s] : -1;
  const int wpos = ((do_lin || fit) && is_point) ? p.cpos[wset][s] : -1;
  if (tp >= 0) {
    prefetch_l1(p.tgt.sp + tp);
    prefetch_l1(p.mahal[cur] + (size_t)s * 6);
    prefetch_l1(p.mahal[cur] + (size_t)s * 6 + 5);
  }
  if (do_lin && wpos >= 0) {
    prefetch_l1(p.tgt.sp + wpos);
    prefetch_l1(p.tcov + (size_t)wpos * 6);
    prefetch_l1(p.tcov + (size_t)wpos * 6 + 5);  // a 48-byte record can straddle two 32-byte sectors
    prefetch_l1(p.scov + (size_t)s * 6);
    prefetch_l1(p.scov + (size_t)s * 6 + 5);
  }
  double T[12];
#pragma unroll
  for (int i = 0; i < 12; i++) T[i] = p.xe[i];
  const double ax = (double)pt.x, ay = (double)pt.y, az = (double)pt.z;
  const double tx = T[0] * ax + T[1] * ay + T[2] * az + T[3];
  const double ty = T[4] * ax + T[5] * ay + T[6] * az + T[7];
  const double tz = T[8] * ax + T[9] * ay + T[10] * az + T[11];
  // ---- trial cost: FastGICP::compute_error at xe with the previous correspondences / mahalanobis
  double trial = 0.0;
  {
    if (tp >= 0) {
      const float4 tb = p.tgt.sp[tp];
      const double* m = p.mahal[cur] + (size_t)s * 6;
      const double ex = (double)tb.x - tx, ey = (double)tb.y - ty, ez = (double)tb.z - tz;
      const double Mex = m[0] * ex + m[1] * ey + m[2] * ez;
      const double Mey = m[1] * ex + m[3] * ey + m[4] * ez;
      const double Mez = m[2] * ex + m[4] * ey + m[5] * ez;
      trial = ex * Mex + ey * Mey + ez * Mez;
    }
  }
  // ---- getFitnessScore sums (fitness round, or the final compute_error round of a registration that wants its fitness):
  // mean of the squared NN distances with d2 <= max_range (information_matrix_calculator.cpp:66-75)
  double fit_sum = 0.0, fit_cnt = 0.0;
  if (fit && wpos >= 0) {
    const float dd = p.d2[s];
    if ((double)dd <= cfg.fit_max_range) { fit_sum = (double)dd; fit_cnt = 1.0; }
  }
  // ---- FastGICP::linearize over the correspondences just written
  double m00 = 0, m01 = 0, m02 = 0, m11 = 0, m12 = 0, m22 = 0, ex = 0, ey = 0, ez = 0;
  if (do_lin) {
    const int best_pos = wpos;
    if (best_pos >= 0) {
      const double* ca = p.scov + (size_t)s * 6;
      const double* cb = p.tcov + (size_t)best_pos * 6;
      const float4 tb = p.tgt.sp[best_pos];
      const double CA[9] = {ca[0], ca[1], ca[2], ca[1], ca[3], ca[4], ca[2], ca[4], ca[5]};
      const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
      double tmp[9], rcr[9], M[9];
      mul3(R, CA, tmp);
      // rcr = CB + tmp * R^T  (symmetric; build the upper part and mirror so the inverse is exactly symmetric)
      double u[6];
      u[0] = tmp[0] * R[0] + tmp[1] * R[1] + tmp[2] * R[2];
      u[1] = tmp[0] * R[3] + tmp[1] * R[4] + tmp[2] * R[5];
      u[2] = tmp[0] * R[6] + tmp[1] * R[7] + tmp[2] * R[8];
      u[3] = tmp[3] * R[3] + tmp[4] * R[4] + tmp[5] * R[5];
      u[4] = tmp[3] * R[6] + tmp[4] * R[7] + tmp[5] * R[8];
      u[5] = tmp[6] * R[6] + tmp[7] * R[7] + tmp[8] * R[8];
      rcr[0] = cb[0] + u[0]; rcr[1] = cb[1] + u[1]; rcr[2] = cb[2] + u[2];
      rcr[4] = cb[3] + u[3]; rcr[5] = cb[4] + u[4]; rcr[8] = cb[5] + u[5];
      rcr[3] = rcr[1]; rcr[6] = rcr[2]; rcr[7] = rcr[5];
      inv3(rcr, M);
      double* mo = p.mahal[wset] + (size_t)s * 6;
      mo[0] = M[0]; mo[1] = M[1]; mo[2] = M[2]; mo[3] = M[4]; mo[4] = M[5]; mo[5] = M[8];
      m00 = M[0]; m01 = M[1]; m02 = M[2]; m11 = M[4]; m12 = M[5]; m22 = M[8];
      ex = (double)tb.x - tx; ey = (double)tb.y - ty; ez = (double)tb.z - tz;
    }
  }
  // a point without correspondence has M = 0, e = 0: every term below is an exact zero, as if it had been skipped
  const double Mex = m00 * ex + m01 * ey + m02 * ez;
  const double Mey = m01 * ex + m11 * ey + m12 * ez;
  const double Mez = m02 * ex + m12 * ey + m22 * ez;
  // S = skew(tA) = [[0,-tz,ty],[tz,0,-tx],[-ty,tx,0]];  MS = M*S;  H = [S^T M S, -S^T M; -M S, M] (upper), b = J^T M e = [S^T Me ; -Me]
  const double ms00 = m01 * tz - m02 * ty, ms01 = -m00 * tz + m02 * tx, ms02 = m00 * ty - m01 * tx;
  const double ms10 = m11 * tz - m12 * ty, ms11 = -m01 * tz + m12 * tx, ms12 = m01 * ty - m11 * tx;
  const double ms20 = m12 * tz - m22 * ty, ms21 = -m02 * tz + m22 * tx, ms22 = m02 * ty - m12 * tx;
  const bool lin = mode == PM_FIRST || mode == PM_FUSED;
  // slots 0 and 1 carry the fitness sums in the rounds that do not linearise (PM_FIT, PM_ERR)
  red_emit<0, 28>(lin ? tz * ms10 - ty * ms20 : fit_sum, tile, red, lane, warp);   // (0,0)
  red_emit<1, 28>(lin ? tz * ms11 - ty * ms21 : fit_cnt, tile, red, lane, warp);   // (0,1)
  red_emit<2, 28>(tz * ms12 - ty * ms22, tile, red, lane, warp);   // (0,2)
  red_emit<3, 28>(-ms00, tile, red, lane, warp);                   // (0,3) = -(MS)[0][0]
  red_emit<4, 28>(-ms10, tile, red, lane, warp);                   // (0,4)
  red_emit<5, 28>(-ms20, tile, red, lane, warp);                   // (0,5)
  red_emit<6, 28>(-tz * ms01 + tx * ms21, tile, red, lane, warp);  // (1,1)
  red_emit<7, 28>(-tz * ms02 + tx * ms22, tile, red, lane, warp);  // (1,2)
  red_emit<8, 28>(-ms01, tile, red, lane, warp);                   // (1,3)
  red_emit<9, 28>(-ms11, tile, red, lane, warp);                   // (1,4)
  red_emit<10, 28>(-ms21, tile, red, lane, warp);                  // (1,5)
  red_emit<11, 28>(ty * ms02 - tx * ms12, tile, red, lane, warp);  // (2,2)
  red_emit<12, 28>(-ms02, tile, red, lane, warp);                  // (2,3)
  red_emit<13, 28>(-ms12, tile, red, lane, warp);                  // (2,4)
  red_emit<14, 28>(-ms22, tile, red, lane, warp);                  // (2,5)
  red_emit<15, 28>(m00, tile, red, lane, warp); red_emit<16, 28>(m01, tile, red, lane, warp); red_emit<17, 28>(m02, tile, red, lane, warp);  // (3,3..5)
  red_emit<18, 28>(m11, tile, red, lane, warp); red_emit<19, 28>(m12, tile, red, lane, warp);                                      // (4,4..5)
  red_emit<20, 28>(m22, tile, red, lane, warp);                                                                         // (5,5)
  red_emit<21, 28>(tz * Mey - ty * Mez, tile, red, lane, warp);
  red_emit<22, 28>(-tz * Mex + tx * Mez, tile, red, lane, warp);
  red_emit<23, 28>(ty * Mex - tx * Mey, tile, red, lane, warp);
  red_emit<24, 28>(-Mex, tile, red, lane, warp); red_emit<25, 28>(-Mey, tile, red, lane, warp); red_emit<26, 28>(-Mez, tile, red, lane, warp);
  red_emit<27, 28>(ex * Mex + ey * Mey + ez * Mez, tile, red, lane, warp);
  red_emit<28, 28>(trial, tile, red, lane, warp);
  __syncthreads();
  // the block's sums: value i = sum over the 8 warps, added in warp order by one thread each
  if (threadIdx.x < kAcc) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < kAccThreads / 32; w++) v += red[threadIdx.x * 8 + w];
    p.partials[(size_t)threadIdx.x * (((unsigned)nblk + 31u) & ~31u) + blockIdx.x] = v;  // transposed: value i of block b at [i * stride + b] (k_pair_lm)
  }
}
static_assert(kAccThreads == 256, "red_emit parks 8 warp sums per value");

// The LM step of every active pair (one block per pair): add the pair's block partials in a fixed order (depends only on the
// pair's own block count => bitwise reproducible, independent of which other pairs share the launch), then thread 0 runs
// fast_gicp's step_lm logic on a SHARED-MEMORY copy of the pair's state (one coalesced load, one coalesced store; the scalar
// chain itself never waits on HBM) and publishes the record when the registration ends.
constexpr int kLmThreads = 256;
__global__ void __launch_bounds__(kLmThreads, 1) k_pair_lm(PairDev* pairs, const int* __restrict__ active, const __grid_constant__ LmCfg cfg) {
  __shared__ double r[kAcc];
  __shared__ PairDev sp;
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (!active) asm volatile("griddepcontrol.launch_dependents;");  // single pair: the next round's search may queue up behind this block
  if (active && (int)blockIdx.x >= active[0]) return;
  PairDev* gp = pairs + (active ? active[1 + blockIdx.x] : blockIdx.x);
  // Two dependent memory round trips instead of six: (1) the whole record (mode, partials pointer and block count included) comes in
  // with one coalesced copy, (2) every load of the reduction is issued before the first one is consumed.
  {
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(gp);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(&sp);
    for (int i = threadIdx.x; i < (int)(sizeof(PairDev) / 8); i += blockDim.x) dst[i] = src[i];
  }
  __syncthreads();
  const int mode = sp.mode;
  if (mode < PM_FIRST || mode > PM_FIT) return;  // block-uniform
  const double* partials = sp.partials;
  const unsigned int nrow = (unsigned int)sp.nblk_acc;
  {
    // the partials are stored transposed ([value][block], stride = blocks rounded up to 32): warp w sums the values w, w + 8, ...;
    // one coalesced load covers 32 blocks of a value, lane l adds blocks l, l + 32, ... in ascending order and a fixed butterfly
    // joins the lanes.  The loads of ALL the warp's values go out first (up to 4 values x 8 rows in flight per lane).
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int nw = kLmThreads / 32;
    constexpr int kVals = (kAcc + nw - 1) / nw;  // values per warp
    const unsigned int stride = (nrow + 31u) & ~31u;
    if (nrow <= 8u * 32u) {
      double t[kVals][8];
#pragma unroll
      for (int q = 0; q < kVals; q++) {
        const int i = warp + q * nw;
#pragma unroll
        for (int u = 0; u < 8; u++) {
          const unsigned int row = lane + 32u * u;
          t[q][u] = (i < kAcc && row < nrow) ? __ldcg(partials + (size_t)i * stride + row) : 0.0;
        }
      }
#pragma unroll
      for (int q = 0; q < kVals; q++) {
        const int i = warp + q * nw;
        double sacc = 0.0;
#pragma unroll
        for (int u = 0; u < 8; u++) if (lane + 32u * u < nrow) sacc += t[q][u];  // same additions, same order as the general loop below
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sacc += __shfl_xor_sync(0xffffffffu, sacc, o);
        if (lane == 0 && i < kAcc) r[i] = sacc;
      }
    } else {
      for (int i = warp; i < kAcc; i += nw) {
        const double* col = partials + (size_t)i * stride;
        double sacc = 0.0;
        unsigned int row = lane;
        for (; row + 7 * 32 < nrow; row += 8 * 32) {
          double t[8];
#pragma unroll
          for (int u = 0; u < 8; u++) t[u] = __ldcg(col + row + u * 32);
#pragma unroll
          for (int u = 0; u < 8; u++) sacc += t[u];
        }
        for (; row < nrow; row += 32) sacc += __ldcg(col + row);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sacc += __shfl_xor_sync(0xffffffffu, sacc, o);
        if (lane == 0) r[i] = sacc;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) lm_advance(sp, r, cfg);
  __syncthreads();
  {
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&sp);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(gp);
    for (int i = threadIdx.x; i < (int)(sizeof(PairDev) / 8); i += blockDim.x) dst[i] = src[i];
  }
}

// After a round: active_out[0] = number of pairs that still need rounds, active_out[1..] = their indices in ascending order;
// (seq << 32 | count) also lands in host-mapped memory so the host can shrink grid.y and stop enqueueing.
__global__ void __launch_bounds__(1024) k_pair_compact(const PairDev* pairs, int n, int* active_out, unsigned long long* h_word, unsigned long long seq) {
  __shared__ int wsum[32];
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int per = (n + 1023) / 1024;
  const int i0 = threadIdx.x * per;
  int cnt = 0;
  for (int i = i0; i < i0 + per && i < n; i++) { const int m = pairs[i].mode; cnt += (m >= PM_FIRST && m <= PM_FIT); }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = wsum[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += v; }
    wsum[lane] = w;
  }
  __syncthreads();
  int pos = incl - cnt + (warp ? wsum[warp - 1] : 0);
  for (int i = i0; i < i0 + per && i < n; i++) { const int m = pairs[i].mode; if (m >= PM_FIRST && m <= PM_FIT) active_out[1 + pos++] = i; }
  if (threadIdx.x == 1023) {
    active_out[0] = wsum[31];
    *reinterpret_cast<volatile unsigned long long*>(h_word) = (seq << 32) | (unsigned long long)(unsigned int)wsum[31];
  }
}
#endif  // __CUDACC__

}  // namespace b2r
