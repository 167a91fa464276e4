// bvh.cuh — exact nearest-neighbour search over a two-level implicit BVH (Hilbert-ordered 32-point leaves).
//
// Replaces the FLANN kd-tree queries the reference's registration handle performs (fast_gicp update_correspondences /
// calculate_covariances, pcl::Registration::getFitnessScore; call sites apps/scan_matching_odometry_nodelet.cpp:210,307,316,
// include/hdl_graph_slam/loop_detector.hpp:143,146) and the kd-tree builds at setInputSource/Target (:172,177,246; :122,136).
//
// Structure (per cloud): points sorted by (30-bit Hilbert key, original index); leaf L = sorted[32L .. 32L+31] with a tight
// AABB; super-node S = leaves [32S .. 32S+31] with a tight AABB.  LiDAR density varies by 3 orders of magnitude between the
// near and the far field; fixed-size leaves adapt to it (a uniform grid does not).
//
// Search = "warp group": the 32 lanes of a warp hold 32 queries that are neighbours in space (a leaf of the query cloud).
// A leaf of the target is visited if ANY lane still needs it; its 32 points are then tested by all lanes (all-pairs tile).
//
// Result contract (oracle/kdtree.hpp): the lexicographically smallest (d2, original index), d2 = ((dx*dx+dy*dy)+dz*dz) in
// non-contracted float32.  Exactness: the AABB bound is assembled from face distances in the same operation order, so by
// monotone rounding it never exceeds the d2 of any point inside the box; a leaf is skipped for a lane only if
// bound > worst (strict) — equal-distance lower-index candidates stay reachable.  No cell quantisation is involved in the
// decision logic (the Morton key only orders the points), so no representability argument is needed.
#pragma once
#include <type_traits>
#include "common.cuh"

// The warp-level code below is device code; tests/warp_harness.cpp also compiles it for the CPU on an emulated 32-lane warp
// (tests/warp_emu.hpp supplies the built-ins) with -DB2R_WARP_EMU.
#if defined(__CUDACC__) || defined(B2R_WARP_EMU)
#define B2R_WARP_CODE 1
#endif

namespace b2r {

constexpr int kLeaf = 32;
constexpr int kSuper = 32;  // leaves per super-node
constexpr int kPadIdx = 0x7fffffff;

struct Bvh {
  const float4* sp;       // [nleaf*32] (x,y,z,bits(orig idx)); padding = (+inf,+inf,+inf, kPadIdx)
  const float4* leaf_lo;  // [nleaf]
  const float4* leaf_hi;
  const float4* sup_lo;   // [nsup]
  const float4* sup_hi;
  int nleaf, nsup, n;
};

// 30-bit 3-D Hilbert index of 10-bit cell coordinates (Skilling's transpose algorithm).  A Hilbert curve has no long jumps,
// so 32 consecutive points stay compact (CPU probe on a VLP-16 frame: max leaf visits per group 74 vs 386 with Morton).
// The key only ORDERS points; exactness never depends on it.
B2R_HD unsigned int hilbert_spread10(unsigned int v) {  // bit i of v -> bit 3 i
  v &= 0x3ffu;
  v = (v | (v << 16)) & 0x030000ffu;
  v = (v | (v << 8)) & 0x0300f00fu;
  v = (v | (v << 4)) & 0x030c30c3u;
  v = (v | (v << 2)) & 0x09249249u;
  return v;
}
B2R_HD unsigned int hilbert30(unsigned int x, unsigned int y, unsigned int z) {
  unsigned int X0 = x & 0x3ffu, X1 = y & 0x3ffu, X2 = z & 0x3ffu;
#pragma unroll
  for (unsigned int Q = 1u << 9; Q > 1; Q >>= 1) {  // inverse undo of the excess work (Skilling): per level, per axis, invert or exchange the low bits
    const unsigned int P = Q - 1;
    if (X0 & Q) X0 ^= P;
    if (X1 & Q) X0 ^= P; else { const unsigned int t = (X0 ^ X1) & P; X0 ^= t; X1 ^= t; }
    if (X2 & Q) X0 ^= P; else { const unsigned int t = (X0 ^ X2) & P; X0 ^= t; X2 ^= t; }
  }
  X1 ^= X0;  // Gray encode
  X2 ^= X1;
  unsigned int t = X2 >> 1;  // bit j of t = xor of the bits of X2 above j: a prefix xor from the top
  t ^= t >> 1; t ^= t >> 2; t ^= t >> 4; t ^= t >> 8;
  X0 ^= t; X1 ^= t; X2 ^= t;
  return (hilbert_spread10(X0) << 2) | (hilbert_spread10(X1) << 1) | hilbert_spread10(X2);  // x bit above y bit above z bit, level by level
}

// lower bound of dist2_f32(q, p) for every p inside [lo, hi] (same association as dist2_f32)
B2R_HD float aabb_bound2(float qx, float qy, float qz, float lx, float ly, float lz, float hx, float hy, float hz) {
  float bx = 0.f, by = 0.f, bz = 0.f;
  if (qx < lx) bx = fsub(lx, qx); else if (qx > hx) bx = fsub(qx, hx);
  if (qy < ly) by = fsub(ly, qy); else if (qy > hy) by = fsub(qy, hy);
  if (qz < lz) bz = fsub(lz, qz); else if (qz > hz) bz = fsub(qz, hz);
  return fadd(fadd(fmul(bx, bx), fmul(by, by)), fmul(bz, bz));
}

// Candidates are ranked by the 64-bit key (float bits of d2) << 32 | original index: d2 >= 0, so integer order of the key ==
// lexicographic order of (d2, idx) — one compare, and a candidate met twice (seed, overlapping parts) is rejected for free.
B2R_HD unsigned long long nn_key(float d2, int idx) {
#ifdef __CUDA_ARCH__
  return ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned int)idx;
#else
  union { float f; unsigned int u; } c; c.f = d2;
  return ((unsigned long long)c.u << 32) | (unsigned int)idx;
#endif
}
B2R_HD float nn_key_d2(unsigned long long k) {
#ifdef __CUDA_ARCH__
  return __uint_as_float((unsigned int)(k >> 32));
#else
  union { float f; unsigned int u; } c; c.u = (unsigned int)(k >> 32); return c.f;
#endif
}
constexpr unsigned long long kKeyInf = 0x7f8000007fffffffull;  // (+inf, kPadIdx)

// 1-NN visitor: (d2, idx) kept in two registers — one float compare per candidate, the index only breaks exact ties
struct Nn1 {
  static constexpr int kTileLanes = 8;   // below 8 interested lanes the cooperative mode (1 step per lane) beats the 32-step tile
  static constexpr int kTileUnroll = 8;  // tiny visitor body: unroll the all-pairs tile loop
  static constexpr bool kTwoPhase = false;
#ifdef B2R_KNN_PROFILE
  int n_tile = 0, n_coop = 0, n_try = 0;
#endif
  float bd2;       // +inf = nothing yet
  int bidx;        // kPadIdx = nothing yet
  int best_pos;
  float lim;
  B2R_HD void reset(float limit_) { bd2 = INFINITY; bidx = kPadIdx; best_pos = -1; lim = limit_; }
  B2R_HD void seed(float d2, int idx, int pos) { bd2 = d2; bidx = idx; best_pos = pos; }
  B2R_HD float worst() const { return bd2; }
  B2R_HD float limit() const { return lim; }
  B2R_HD void visit(float d2, int idx, int pos) {
    // padding entries carry (+inf, kPadIdx): never better than anything, so no explicit padding test is needed
    if (d2 < bd2 || (d2 == bd2 && idx < bidx)) { bd2 = d2; bidx = idx; best_pos = pos; }
  }
  // the same as a predicated update (three selects, no branch): the all-pairs tile loop runs it 32 times per lane and visited leaf,
  // and a divergent `if` there costs a BSSY / BRA / BSYNC triple per candidate (ncu: 20 % of the search kernel's instructions)
  B2R_HD void visit_if(bool on, float d2, int idx, int pos) {
    const bool b = on & ((d2 < bd2) | ((d2 == bd2) & (idx < bidx)));
    bd2 = b ? d2 : bd2; bidx = b ? idx : bidx; best_pos = b ? pos : best_pos;
  }
  B2R_HD float best_d2() const { return bd2; }
  B2R_HD int best_idx() const { return bidx; }
#ifdef B2R_WARP_CODE
  // C copies of one query sit in lanes q, q + 32/C, ...; each saw a different 1/C of the candidates: all adopt the best result
  template <int C>
  __device__ __forceinline__ void merge_copies() {
#pragma unroll
    for (int off = 32 / C; off < 32; off <<= 1) {
      const float od = __shfl_xor_sync(0xffffffffu, bd2, off);
      const int oi = __shfl_xor_sync(0xffffffffu, bidx, off);
      const int op = __shfl_xor_sync(0xffffffffu, best_pos, off);
      if (od < bd2 || (od == bd2 && oi < bidx)) { bd2 = od; bidx = oi; best_pos = op; }
    }
  }
#endif
};

// 1-NN visitor on ONE packed key (nn_key): the lexicographic (d2, index) rule is a single unsigned 64-bit compare, so the all-pairs
// tile loop costs 2 ISETP + 2 SEL per candidate instead of FSETP.NEU + ISETP + FSETP.LT + PLOP3 + FSEL + SEL (+ SEL for the position);
// the `pass` predicate is folded into the start key (key 0 beats everything) instead of being and-ed into every candidate's
// decision.  No position is tracked: the caller maps the winning index through the target's pos_of table.  Same candidates, same
// rule => the same answers as Nn1 (tests/warp_harness.cpp runs both on the emulated warp).
#ifndef B2R_NN1K_TILE_LANES
#define B2R_NN1K_TILE_LANES 8
#endif
struct Nn1K {
  static constexpr int kTileLanes = B2R_NN1K_TILE_LANES;
  static constexpr int kTileUnroll = 8;
  static constexpr bool kTwoPhase = false;
  static constexpr bool kKeyed = true;
#ifdef B2R_KNN_PROFILE
  int n_tile = 0, n_coop = 0, n_try = 0;
#endif
  unsigned long long key;  // kKeyInf = nothing yet
  float lim;
  B2R_HD void reset(float limit_) { key = kKeyInf; lim = limit_; }
  B2R_HD void seed(float d2, int idx, int) { key = nn_key(d2, idx); }
  B2R_HD float worst() const { return nn_key_d2(key); }
  B2R_HD float limit() const { return lim; }
  B2R_HD void visit(float d2, int idx, int) {
    const unsigned long long kq = nn_key(d2, idx);  // padding = kKeyInf: never below any key
    key = kq < key ? kq : key;
  }
  B2R_HD unsigned long long tile_begin(bool pass) const { return pass ? key : 0ull; }
  B2R_HD void tile_end(bool pass, unsigned long long k) { key = pass ? k : key; }
  B2R_HD float best_d2() const { return nn_key_d2(key); }
  B2R_HD int best_idx() const { return (int)(unsigned int)(key & 0xffffffffull); }
  B2R_HD bool found() const { return (unsigned int)(key & 0xffffffffull) != (unsigned int)kPadIdx; }
#ifdef B2R_WARP_CODE
  template <int C>
  __device__ __forceinline__ void merge_copies() {
#pragma unroll
    for (int off = 32 / C; off < 32; off <<= 1) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, key, off);
      key = o < key ? o : key;
    }
  }
#endif
};
template <class V, class = void> struct keyed_visitor : std::false_type {};
template <class V> struct keyed_visitor<V, std::void_t<decltype(V::kKeyed)>> : std::integral_constant<bool, V::kKeyed> {};

// host/device serial reference of the traversal for ONE query (used by tests/host_harness.cu and as documentation of the
// pruning rule; the device path below makes the same per-lane decisions, only warp-wide)
template <class Visitor>
B2R_HD void bvh_search_one(const Bvh& b, float qx, float qy, float qz, Visitor& v) {
  for (int s = 0; s < b.nsup; s++) {
    const float4 slo = b.sup_lo[s], shi = b.sup_hi[s];
    const float sb = aabb_bound2(qx, qy, qz, slo.x, slo.y, slo.z, shi.x, shi.y, shi.z);
    if (sb > v.worst() || !(sb < v.limit())) continue;
    const int l1 = (s + 1) * kSuper < b.nleaf ? (s + 1) * kSuper : b.nleaf;
    for (int l = s * kSuper; l < l1; l++) {
      const float4 lo = b.leaf_lo[l], hi = b.leaf_hi[l];
      const float lb = aabb_bound2(qx, qy, qz, lo.x, lo.y, lo.z, hi.x, hi.y, hi.z);
      if (lb > v.worst() || !(lb < v.limit())) continue;
      for (int t = 0; t < kLeaf; t++) {
        const float4 p = b.sp[l * kLeaf + t];
        const int idx = idx_bits(p.w);
        if (idx == kPadIdx) continue;
        v.visit(dist2_f32(qx, qy, qz, p.x, p.y, p.z), idx, l * kLeaf + t);
      }
    }
  }
}

#ifdef B2R_WARP_CODE
// ------------------------------------------------------------------------------------------------ build kernels
__global__ void k_morton_keys(const float* __restrict__ raw, int stride_f, int n, const int* __restrict__ mm, unsigned int* keys, int* vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = raw + (size_t)i * stride_f;
  const float x = p[0], y = p[1], z = p[2];
  unsigned int key = 0xffffffffu;  // non-finite points sort last and are dropped from the structure
  if (finite3(x, y, z)) {
    const float mnx = ord2f(mm[0]), mny = ord2f(mm[1]), mnz = ord2f(mm[2]);
    const float ext = fmaxf(fmaxf(ord2f(mm[3]) - mnx, ord2f(mm[4]) - mny), fmaxf(ord2f(mm[5]) - mnz, 1.0e-6f));
    const float sc = 1023.0f / ext;
    const unsigned int ix = (unsigned int)fminf(fmaxf((x - mnx) * sc, 0.f), 1023.f);
    const unsigned int iy = (unsigned int)fminf(fmaxf((y - mny) * sc, 0.f), 1023.f);
    const unsigned int iz = (unsigned int)fminf(fmaxf((z - mnz) * sc, 0.f), 1023.f);
    key = hilbert30(ix, iy, iz);
  }
  keys[i] = key;
  vals[i] = i;
}

// one block = 1024 threads = 32 leaves = one super-node
__global__ void __launch_bounds__(1024) k_bvh_leaves(const float* __restrict__ raw, int stride_f, int n, const unsigned int* __restrict__ keys_sorted,
                                                     const int* __restrict__ vals_sorted, float4* sorted, int* pos_of, float4* leaf_lo,
                                                     float4* leaf_hi, float4* sup_lo, float4* sup_hi) {
  __shared__ float s_lo[32][3], s_hi[32][3];
  const int s = blockIdx.x * 1024 + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float x = INFINITY, y = INFINITY, z = INFINITY;
  int idx = kPadIdx;
  if (s < n && keys_sorted[s] != 0xffffffffu) {
    idx = vals_sorted[s];
    const float* p = raw + (size_t)idx * stride_f;
    x = p[0]; y = p[1]; z = p[2];
    pos_of[idx] = s;
  }
  sorted[s] = make_float4(x, y, z, bits_idx(idx));
  const bool valid = idx != kPadIdx;
  float lx = valid ? x : INFINITY, ly = valid ? y : INFINITY, lz = valid ? z : INFINITY;
  float hx = valid ? x : -INFINITY, hy = valid ? y : -INFINITY, hz = valid ? z : -INFINITY;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lx = fminf(lx, __shfl_xor_sync(0xffffffffu, lx, o)); ly = fminf(ly, __shfl_xor_sync(0xffffffffu, ly, o)); lz = fminf(lz, __shfl_xor_sync(0xffffffffu, lz, o));
    hx = fmaxf(hx, __shfl_xor_sync(0xffffffffu, hx, o)); hy = fmaxf(hy, __shfl_xor_sync(0xffffffffu, hy, o)); hz = fmaxf(hz, __shfl_xor_sync(0xffffffffu, hz, o));
  }
  const int leaf = blockIdx.x * 32 + warp;
  if (lane == 0) {
    leaf_lo[leaf] = make_float4(lx, ly, lz, 0.f);
    leaf_hi[leaf] = make_float4(hx, hy, hz, 0.f);
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
      sup_lo[blockIdx.x] = make_float4(ax, ay, az, 0.f);
      sup_hi[blockIdx.x] = make_float4(bx, by, bz, 0.f);
    }
  }
}


// ------------------------------------------------------------------------------------------------ warp-group traversal
// Group-level masks are cheap but only as good as the group's box: a group that straddles a jump of the Hilbert curve has a box
// of tens of metres and would send every leaf in range to bvh_try_leaf (one such warp, with hundreds of leaf tests, can set the
// kernel time).  When a group mask keeps more than kRefineAbove nodes, every lane re-tests the survivors against ITS OWN query
// (uniform loads, no ballot in the loop) and the warp keeps the union.
constexpr int kRefineAbove = 4;
template <class Visitor>
__device__ __forceinline__ unsigned refine_node_mask(unsigned gmask, const float4* __restrict__ nlo, const float4* __restrict__ nhi, float qx, float qy,
                                                     float qz, bool active, const Visitor& v) {
  if (__popc(gmask) <= kRefineAbove) return gmask;
  unsigned mine = 0;
  const float w = v.worst(), lim = v.limit();
  if (active) {
    for (unsigned m = gmask; m; m &= m - 1) {
      const int j = __ffs(m) - 1;
      const float4 lo = __ldg(nlo + j), hi = __ldg(nhi + j);
      const float lb = aabb_bound2(qx, qy, qz, lo.x, lo.y, lo.z, hi.x, hi.y, hi.z);
      if (!(lb > w) && lb < lim) mine |= 1u << j;
    }
  }
  return __reduce_or_sync(0xffffffffu, mine);
}

// All 32 lanes call this together.  Lane l holds query (qx,qy,qz) (active) and its own visitor.
//   own_leaf >= 0 : the queries ARE that leaf of this same structure (k-NN of a cloud against itself): visited first.
// Order: own leaf, then the super-node nearest to the group's AABB, then all remaining super-nodes by index.
// Visit one leaf for the lanes flagged `pass`.  Two modes (a Morton leaf at a curve discontinuity can
// span 100 m; its 32 queries then want DIFFERENT leaves and a pure all-pairs tile wastes 31/32 of the work):
//   tile mode  (>= kTileLanes lanes interested): every lane tests all 32 candidates (broadcast loads);
//   coop mode  (few lanes interested): for each interested lane L the 32 lanes evaluate the leaf's 32 candidates in ONE
//              step (lane t owns candidate t), then L's visitor consumes the acceptable ones best-first.
// Both feed exactly the same (d2, idx) candidates to the same visitors, so the result is identical.

// C > 1: the warp carries Q = 32/C queries; lanes q, q+Q, q+2Q, ... hold the SAME query and identical visitor state between
// visits.  In tile mode each copy scans 1/C of the leaf and the copies merge afterwards: C times the warps, 1/C of the chain per
// warp — the searches are latency-bound and their kernel time is the slowest warp, i.e. the heaviest query.
// Candidates and tie rule are unchanged, so results are identical.
template <int C = 1, class Visitor>
__device__ __forceinline__ bool bvh_visit_leaf(const Bvh& b, int l, float qx, float qy, float qz, bool pass, Visitor& v) {
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  unsigned mask = __ballot_sync(FULL, pass);
  constexpr int Q = 32 / C;                                                        // distinct queries per warp
#ifdef B2R_TILE_AT  // offline experiments (tools/warp_cost.cpp)
  constexpr int kTile = B2R_TILE_AT;
#else
  constexpr int kTile = C == 1 ? Visitor::kTileLanes : (Visitor::kTileLanes / C > 1 ? Visitor::kTileLanes / C : 1);
#endif
  if (C > 1) mask &= (Q == 32 ? 0xffffffffu : ((1u << Q) - 1u));
  if (mask == 0) return false;  // warp-uniform: nobody wanted the leaf
  const float4* __restrict__ lp = b.sp + (size_t)l * kLeaf;
#ifdef B2R_KNN_PROFILE
  if (__popc(mask) >= kTile) v.n_tile++; else v.n_coop += __popc(mask);
#ifdef B2R_WARP_EMU
  if (lane == 0) g_visit_hist[__popc(mask)]++;  // offline model only (tools/warp_cost.cpp): how many queries wanted each visited leaf
#endif
#endif
  if (__popc(mask) >= kTile) {
    // (dynamic regrouping of sparse visits — the r-th interested query served by 2 or 4 adjacent lanes sweeping a half / a quarter of the
    // leaf each — is exact but was no faster out of line and slower inlined at every visit site)
    if constexpr (C > 1) {
      const int t0 = (lane / Q) * (kLeaf / C);
      if constexpr (keyed_visitor<Visitor>::value) {
        unsigned long long k = v.tile_begin(pass);
#pragma unroll
        for (int t = 0; t < kLeaf / C; t++) {
          const float4 p = __ldg(lp + t0 + t);
          const unsigned long long kq = nn_key(dist2_f32(qx, qy, qz, p.x, p.y, p.z), idx_bits(p.w));
          k = kq < k ? kq : k;
        }
        v.tile_end(pass, k);
      } else {
#pragma unroll
        for (int t = 0; t < kLeaf / C; t++) {
          const float4 p = __ldg(lp + t0 + t);  // C addresses per warp
          v.visit_if(pass, dist2_f32(qx, qy, qz, p.x, p.y, p.z), idx_bits(p.w), l * kLeaf + t0 + t);
        }
      }
      v.template merge_copies<C>();
    } else if constexpr (Visitor::kTwoPhase) {
      // list visitors (an accepted candidate costs ~100 instructions for the whole warp): first mark the candidates that can
      // still beat the lane's current worst (cheap, branch-free), then let every lane walk ITS OWN marks — the number of
      // insertion rounds is max-over-lanes of the marks, not the number of steps in which any lane accepts.  Per lane the
      // candidates arrive in the same ascending order and visit() re-tests exactly, so the lists are identical.
      unsigned m = 0;
      const float w = v.worst();
#pragma unroll 8
      for (int t = 0; t < kLeaf; t++) {
        const float4 p = __ldg(lp + t);
        if (dist2_f32(qx, qy, qz, p.x, p.y, p.z) <= w) m |= 1u << t;
      }
      if (!pass) m = 0;
      while (__any_sync(FULL, m != 0)) {
        if (m) {
          const int t = __ffs(m) - 1;
          m &= m - 1;
          const float4 p = __ldg(lp + t);
          v.visit(dist2_f32(qx, qy, qz, p.x, p.y, p.z), idx_bits(p.w), l * kLeaf + t);
        }
      }
    } else {
      // (a minimum-first variant — one sweep that keeps only the smallest distance, the exact (d2, index) sweep only when some lane can
      // improve — was no faster on the 4-lane odometry search and slower on the 1-lane batch search, where some lane of
      // the 32 nearly always needs the second sweep)
      if constexpr (keyed_visitor<Visitor>::value) {
        unsigned long long k = v.tile_begin(pass);
#pragma unroll Visitor::kTileUnroll
        for (int t = 0; t < kLeaf; t++) {
          const float4 p = __ldg(lp + t);
          const unsigned long long kq = nn_key(dist2_f32(qx, qy, qz, p.x, p.y, p.z), idx_bits(p.w));
          k = kq < k ? kq : k;
        }
        v.tile_end(pass, k);
      } else {
#pragma unroll Visitor::kTileUnroll
        for (int t = 0; t < kLeaf; t++) {
          const float4 p = __ldg(lp + t);  // same address on every lane: one broadcast transaction
          v.visit_if(pass, dist2_f32(qx, qy, qz, p.x, p.y, p.z), idx_bits(p.w), l * kLeaf + t);  // padding = (+inf, kPadIdx): rejected by the visitor
        }
      }
    }
    return true;
  }
  const float4 mine = __ldg(lp + lane);  // coalesced: candidate `lane`
  const int my_idx = idx_bits(mine.w);
  while (mask) {
    const int L = __ffs(mask) - 1;
    mask &= mask - 1;
    const float ax = __shfl_sync(FULL, qx, L), ay = __shfl_sync(FULL, qy, L), az = __shfl_sync(FULL, qz, L);
    const float d2 = dist2_f32(ax, ay, az, mine.x, mine.y, mine.z);
    float wL = __shfl_sync(FULL, v.worst(), L);
    bool ok = (my_idx != kPadIdx) && !(d2 > wL);
    while (__ballot_sync(FULL, ok)) {
      // best acceptable candidate: min d2 (non-negative floats order like unsigned ints), then min index among equals
      const unsigned int du = ok ? __float_as_uint(d2) : 0xffffffffu;
      const unsigned int dmin = __reduce_min_sync(FULL, du);
      const unsigned int iu = (ok && du == dmin) ? (unsigned int)my_idx : 0xffffffffu;
      const unsigned int imin = __reduce_min_sync(FULL, iu);
      const int bl = __ffs(__ballot_sync(FULL, ok && du == dmin && iu == imin)) - 1;
      const float bd = __uint_as_float(dmin);
      const int bi = (int)imin;
      if ((lane & (Q - 1)) == L) v.visit(bd, bi, l * kLeaf + bl);
      if (lane == bl) ok = false;
      wL = __shfl_sync(FULL, v.worst(), L);
      ok = ok && !(d2 > wL);
    }
  }
  return true;
}

// lower bound of dist2_f32(q, p) for every q inside box G and p inside box N (gap per axis, same association): it never
// exceeds aabb_bound2(q, N) for a q in G (monotone rounding), so pruning a node for the whole GROUP with it is safe.
__device__ __forceinline__ float aabb_aabb_bound2(float glx, float gly, float glz, float ghx, float ghy, float ghz, const float4& lo, const float4& hi) {
  float bx = 0.f, by = 0.f, bz = 0.f;
  if (ghx < lo.x) bx = fsub(lo.x, ghx); else if (glx > hi.x) bx = fsub(glx, hi.x);
  if (ghy < lo.y) by = fsub(lo.y, ghy); else if (gly > hi.y) by = fsub(gly, hi.y);
  if (ghz < lo.z) bz = fsub(lo.z, ghz); else if (glz > hi.z) bz = fsub(glz, hi.z);
  return fadd(fadd(fmul(bx, bx), fmul(by, by)), fmul(bz, bz));
}

// exact per-lane test + visit of one leaf
// exact = false: every active lane takes the leaf without a bound test (the queries' own leaf in a self k-NN)
template <int C = 1, class Visitor>
__device__ __forceinline__ bool bvh_try_leaf(const Bvh& b, int l, float qx, float qy, float qz, bool active, Visitor& v, bool exact = true) {
#ifdef B2R_KNN_PROFILE
  v.n_try++;
#endif
  const float4 lo = __ldg(b.leaf_lo + l), hi = __ldg(b.leaf_hi + l);
  const float lb = aabb_bound2(qx, qy, qz, lo.x, lo.y, lo.z, hi.x, hi.y, hi.z);
  const bool pass = active && (!exact || (!(lb > v.worst()) && (lb < v.limit())));
  return bvh_visit_leaf<C>(b, l, qx, qy, qz, pass, v);
}

// loosest bound of the group as ordered bits (non-negative floats order like unsigned ints): one REDUX instruction
template <class Visitor>
__device__ __forceinline__ float group_max_worst_fast(bool active, const Visitor& v) {
  const float w = fminf(v.worst(), v.limit());  // >= 0 or +inf
  return __uint_as_float(__reduce_max_sync(0xffffffffu, active ? __float_as_uint(w) : 0u));
}

// All 32 lanes call this together.  Lane l holds query (qx,qy,qz) (active) and its own visitor.
//   own_leaf >= 0 : the queries ARE that leaf of this same structure (k-NN of a cloud against itself): visited first.
//   own_leaf <  0 : `hint_leaf` >= 0 names a leaf that probably holds the answers (last iteration's correspondent); else the
//                   leaf nearest to the group's centre is looked up.
// Node tests are lane-parallel against the GROUP's AABB and loosest bound (lane j tests node j: 32 nodes per step, no
// dependent-load chain, conservative); the survivors get the exact per-lane test inside bvh_try_leaf at visit time.
// Order: own/hinted leaf, the 32-leaf window centred on it by index distance, then the remaining super-nodes by index.
template <int C = 1, class Visitor>
__device__ __forceinline__ void bvh_group_search(const Bvh& b, float qx, float qy, float qz, bool active, Visitor& v, int own_leaf,
                                                 int hint_leaf = -1) {
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  if (__ballot_sync(FULL, active) == 0 || b.nleaf <= 0) return;
  // group AABB of the active queries
  float glx = active ? qx : INFINITY, gly = active ? qy : INFINITY, glz = active ? qz : INFINITY;
  float ghx = active ? qx : -INFINITY, ghy = active ? qy : -INFINITY, ghz = active ? qz : -INFINITY;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    glx = fminf(glx, __shfl_xor_sync(FULL, glx, o)); gly = fminf(gly, __shfl_xor_sync(FULL, gly, o)); glz = fminf(glz, __shfl_xor_sync(FULL, glz, o));
    ghx = fmaxf(ghx, __shfl_xor_sync(FULL, ghx, o)); ghy = fmaxf(ghy, __shfl_xor_sync(FULL, ghy, o)); ghz = fmaxf(ghz, __shfl_xor_sync(FULL, ghz, o));
  }
  // The first leaf — the queries' own one, the hinted one, or the one nearest to the group's centre — is visited at ONE call site, and
  // so are the leaves of pass 1 and of pass 2: every site inlines the whole leaf visit (for the list visitors two copies of the
  // 80-instruction insertion network), and six of them made the k-NN kernel 6 000 instructions long.
  int first = own_leaf >= 0 ? own_leaf : hint_leaf;
  const bool first_exact = own_leaf < 0;
  // no own leaf, no hint: the leaf nearest to the group's centre inside the nearest super-node (ordering heuristic only)
  if (first < 0) {
    const float gcx = 0.5f * (glx + ghx), gcy = 0.5f * (gly + ghy), gcz = 0.5f * (glz + ghz);
    float bd = INFINITY;
    int bs = 0;
    for (int s = lane; s < b.nsup; s += 32) {
      const float4 slo = __ldg(b.sup_lo + s), shi = __ldg(b.sup_hi + s);
      const float d = aabb_bound2(gcx, gcy, gcz, slo.x, slo.y, slo.z, shi.x, shi.y, shi.z);
      if (d < bd) { bd = d; bs = s; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float od = __shfl_xor_sync(FULL, bd, o);
      const int os = __shfl_xor_sync(FULL, bs, o);
      if (od < bd || (od == bd && os < bs)) { bd = od; bs = os; }
    }
    const int l = bs * kSuper + lane;
    float ld = INFINITY;
    if (l < b.nleaf) {
      const float4 lo = __ldg(b.leaf_lo + l), hi = __ldg(b.leaf_hi + l);
      ld = aabb_bound2(gcx, gcy, gcz, lo.x, lo.y, lo.z, hi.x, hi.y, hi.z);
    }
    int ll = l;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float od = __shfl_xor_sync(FULL, ld, o);
      const int ol = __shfl_xor_sync(FULL, ll, o);
      if (od < ld || (od == ld && ol < ll)) { ld = od; ll = ol; }
    }
    if (ld < INFINITY) first = ll;
  }
  if (first >= 0) { bvh_try_leaf<C>(b, first, qx, qy, qz, active, v, first_exact); own_leaf = first; }  // from here on `own_leaf` = already visited
  // pass 1: the window of 32 leaves CENTRED on the already-visited leaf, in order of index distance from it (Hilbert order:
  // index neighbours are space neighbours), so the bound is tight before anything else is looked at.  The window ignores
  // super-node borders: a leaf that straddles a jump of the curve at the end of its super-node has half of its true
  // neighbours in the next one (such a leaf alone can set the kernel time).
  int win0 = -1;  // first leaf of the pass-1 window
  if (own_leaf >= 0) {
    win0 = own_leaf - kSuper / 2;
    if (win0 > b.nleaf - kSuper) win0 = b.nleaf - kSuper;
    if (win0 < 0) win0 = 0;
    const float gw = group_max_worst_fast(active, v);
    const float4 lo = __ldg(b.leaf_lo + win0 + lane), hi = __ldg(b.leaf_hi + win0 + lane);
    const float lgb = aabb_aabb_bound2(glx, gly, glz, ghx, ghy, ghz, lo, hi);
    unsigned lmask = __ballot_sync(FULL, !(lgb > gw) && lgb < INFINITY) & ~(1u << (own_leaf - win0));
    lmask = refine_node_mask(lmask, b.leaf_lo + win0, b.leaf_hi + win0, qx, qy, qz, active, v);
    const int c = own_leaf - win0;
#pragma unroll 1
    for (int e = 2; e < 2 * kSuper && lmask; e++) {  // e = 2 d + side: c - 1, c + 1, c - 2, c + 2, ...
      const int d = e >> 1;
      const int j = (e & 1) ? c + d : c - d;
      if (j >= 0 && j < kSuper && ((lmask >> j) & 1u)) { lmask &= ~(1u << j); bvh_try_leaf<C>(b, win0 + j, qx, qy, qz, active, v); }
    }
  }
  // pass 2: every super-node, 32 per step, then the leaves of each survivor, 32 per step — all against the group's box and
  // its CURRENT loosest bound (one REDUX); leaves inside the pass-1 window are done (visited, or pruned for good).
  for (int sbase = 0; sbase < b.nsup; sbase += 32) {
    unsigned smask;
    {
      const float gw = group_max_worst_fast(active, v);
      const int sg = sbase + lane;
      float sgb = INFINITY;
      if (sg < b.nsup) {
        const float4 slo = __ldg(b.sup_lo + sg), shi = __ldg(b.sup_hi + sg);
        sgb = aabb_aabb_bound2(glx, gly, glz, ghx, ghy, ghz, slo, shi);
      }
      smask = __ballot_sync(FULL, !(sgb > gw) && sgb < INFINITY);
    }
    if (win0 >= 0 && (win0 % kSuper) == 0 && win0 / kSuper >= sbase && win0 / kSuper < sbase + 32) smask &= ~(1u << (win0 / kSuper - sbase));  // window == one whole super-node
    smask = refine_node_mask(smask, b.sup_lo + sbase, b.sup_hi + sbase, qx, qy, qz, active, v);
    while (smask) {
      const int sj = __ffs(smask) - 1;
      smask &= smask - 1;
      const int l0 = (sbase + sj) * kSuper;
      const float gw = group_max_worst_fast(active, v);
      const float4 lo = __ldg(b.leaf_lo + l0 + lane), hi = __ldg(b.leaf_hi + l0 + lane);
      const float lgb = aabb_aabb_bound2(glx, gly, glz, ghx, ghy, ghz, lo, hi);
      unsigned lmask = __ballot_sync(FULL, !(lgb > gw) && lgb < INFINITY);
      const int rel = win0 - l0;
      if (win0 >= 0 && rel > -kSuper && rel < kSuper) lmask &= ~(rel >= 0 ? (0xffffffffu << rel) : (0xffffffffu >> (-rel)));
      lmask = refine_node_mask(lmask, b.leaf_lo + l0, b.leaf_hi + l0, qx, qy, qz, active, v);
      while (lmask) {
        const int lj = __ffs(lmask) - 1;
        lmask &= lmask - 1;
        bvh_try_leaf<C>(b, l0 + lj, qx, qy, qz, active, v);
      }
    }
  }
}
#endif

}  // namespace b2r
