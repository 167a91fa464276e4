// bvh_build.cuh — the whole implicit-BVH build of a cloud as ONE kernel on a thread-block cluster.
//
// What it replaces: the kd-tree builds the reference pays at every setInputSource / setInputTarget (pcl::search::KdTree inside
// fast_gicp, pcl::Registration::initCompute's FLANN tree; call sites /root/reference/apps/scan_matching_odometry_nodelet.cpp:
// 172,177,246 and /root/reference/include/hdl_graph_slam/loop_detector.hpp:122,136) — and, in this engine, a chain of eleven
// launches (bbox, fill, keys, six cub::DeviceRadixSort kernels, leaves).
//
// Design: a cloud of up to 131 072 points lives ENTIRELY in the distributed shared memory of one cluster
// (CL = 1/2/4/8 CTAs x PER = 1..16 (key, index) pairs per thread, at most 128 KB per CTA).  The cluster computes the bounding box, the 30-bit Hilbert
// keys, runs a stable 4-pass LSD radix sort whose scatter writes straight into the PEER CTAs' shared memory (DSMEM stores,
// cluster barriers between passes — no global-memory round trip, no histogram/offset kernels), and finally each CTA emits its
// contiguous slice of the structure: sorted float4 points, pos_of, leaf boxes, super-node boxes.
// blockIdx.x / CL selects the cloud: a whole set of keyframe clouds is built by one launch.
//
// Order contract (unchanged): ascending (Hilbert key, original index); non-finite points dropped (pos_of = -1); padding
// entries (+inf, kPadIdx) up to a multiple of 1024.
#pragma once
#include <cooperative_groups.h>
#include "bvh.cuh"
#include "grid.cuh"

namespace b2r {

constexpr int kBuildThreads = 1024;
constexpr int kBuildMaxPer = 16;                        // (key, index) pairs per thread at most: 16 384 per CTA, 128 KB of shared memory
constexpr int kBuildMaxPoints = 8 * kBuildMaxPer * kBuildThreads;  // 131 072: the largest cloud a cluster of 8 holds
// PER pairs per thread => a CTA holds PER * 1024 pairs.  The kernels are latency bound (one cluster per cloud), so a cloud is spread over
// as MANY CTAs as the portable cluster size allows (8) with as FEW pairs per thread as that needs: 65 536 points = 8 CTAs x 8 per
// thread, 24 000 points = 8 x 4 (every phase except the barriers scales with the pairs per thread).
template <int PER>
struct BuildGeom {
  static_assert(PER == 1 || PER == 2 || PER == 4 || PER == 8 || PER == 16, "pairs per thread: a power of two up to 16");
  static constexpr int kCap = PER * kBuildThreads;                                                     // pairs held by one CTA
  static constexpr int kShift = PER == 1 ? 10 : PER == 2 ? 11 : PER == 4 ? 12 : PER == 8 ? 13 : 14;     // log2(kCap)
  static constexpr size_t kSmem = (size_t)kCap * 8 + 32 * 256 * 2 + 256 * 4 * 2 + 64 * 4;
};
// the (cluster size, pairs per thread) of a cloud of n points: 0 = too large for a cluster.  `wide` = clusters of 16 CTAs may be
// launched (non-portable size, opt-in per kernel, probed once: cluster16_allowed()): clouds above 65 536 points then take
// 16 CTAs x 8 pairs instead of 8 x 16.
struct BuildShape { int cl, per; };
inline BuildShape build_shape_for(size_t n, bool wide) {
  if (n > (size_t)kBuildMaxPoints) return {0, 0};
  const int slices = (int)((n + kBuildThreads - 1) / kBuildThreads) > 0 ? (int)((n + kBuildThreads - 1) / kBuildThreads) : 1;
  if (wide && slices > 64) return {16, 8};
  int per = 1;
  while (per * 8 < slices) per *= 2;
  int cl = 1;
  while (cl * per < slices) cl *= 2;
  return {cl, per};
}
// index of a shape in the instantiation table: (1,1) (2,1) (4,1) (8,1) (8,2) (8,4) (8,8) (8,16) (16,8)
inline int build_shape_index(BuildShape s) {
  if (s.cl == 16) return 8;
  return s.per == 1 ? (s.cl == 1 ? 0 : s.cl == 2 ? 1 : s.cl == 4 ? 2 : 3) : (s.per == 2 ? 4 : s.per == 4 ? 5 : s.per == 8 ? 6 : 7);
}
constexpr int kBuildShapes = 9;

struct BuildItem {   // one cloud of a batched build
  const float* raw;
  float4* sorted;
  int* pos_of;
  float4* leaf_lo;
  float4* leaf_hi;
  float4* sup_lo;
  float4* sup_hi;
  int stride_f;
  int n;
};

#ifdef __CUDACC__
namespace cg = cooperative_groups;

// -DB2R_BUILD_PROFILE (tools/build_variant.sh): thread 0 of CTA 0 prints the cycles between the marks of one build
#ifdef B2R_BUILD_PROFILE
#define B2R_MARK(k) do { if (threadIdx.x == 0 && blockIdx.x == 0) b2r_marks[k] = clock64(); } while (0)
#else
#define B2R_MARK(k) do { } while (0)
#endif

#ifdef B2R_BUILD_PROFILE
__device__ long long b2r_marks[16];
#endif

// ---- shared-memory layout and the two cluster-wide building blocks (also used by the voxel-grid kernel, voxelgrid.cuh)
struct ClusterSmem {
  uint2* buf;            // [PER * 1024] (key, original index)
  unsigned short* wh;    // [32 warps][256 digits]
  int* cta_cnt;          // [256] digit counts of this CTA
  int* base;             // [256] first destination of (digit, this CTA)
  int* s_mm;             // [6] bbox as ordered ints, [8..63] scratch
};
template <int PER>
__device__ __forceinline__ ClusterSmem cluster_smem(unsigned char* smem_raw) {
  constexpr size_t cap = BuildGeom<PER>::kCap;
  ClusterSmem S;
  S.buf = reinterpret_cast<uint2*>(smem_raw);
  S.wh = reinterpret_cast<unsigned short*>(smem_raw + cap * 8);
  S.cta_cnt = reinterpret_cast<int*>(smem_raw + cap * 8 + 32 * 256 * 2);
  S.base = S.cta_cnt + 256;
  S.s_mm = S.base + 256;
  return S;
}

// bounding box of the finite points of a cloud spread over the cluster (element i of CTA `rank` = point g0 + i), as ordered ints
template <int CL, int PER>
__device__ __forceinline__ void cluster_bbox(cg::cluster_group& cluster, const ClusterSmem& S, const float* __restrict__ raw, int stride_f, int n, int g0, int* mm) {
  int* s_mm = S.s_mm;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < 6) s_mm[tid] = tid < 3 ? 0x7fffffff : (int)0x80000000;
  __syncthreads();
  {
    int mn0 = 0x7fffffff, mn1 = 0x7fffffff, mn2 = 0x7fffffff, mx0 = (int)0x80000000, mx1 = (int)0x80000000, mx2 = (int)0x80000000;
#pragma unroll
    for (int b = 0; b < PER; b++) {
      const int i = g0 + warp * (32 * PER) + b * 32 + lane;
      if (i < n) {
        const float* p = raw + (size_t)i * stride_f;
        const float x = p[0], y = p[1], z = p[2];
        if (finite3(x, y, z)) {
          const int ox = f2ord(x), oy = f2ord(y), oz = f2ord(z);
          mn0 = min(mn0, ox); mn1 = min(mn1, oy); mn2 = min(mn2, oz);
          mx0 = max(mx0, ox); mx1 = max(mx1, oy); mx2 = max(mx2, oz);
        }
      }
    }
    mn0 = __reduce_min_sync(0xffffffffu, mn0); mn1 = __reduce_min_sync(0xffffffffu, mn1); mn2 = __reduce_min_sync(0xffffffffu, mn2);
    mx0 = __reduce_max_sync(0xffffffffu, mx0); mx1 = __reduce_max_sync(0xffffffffu, mx1); mx2 = __reduce_max_sync(0xffffffffu, mx2);
    if (lane == 0) {
      atomicMin(&s_mm[0], mn0); atomicMin(&s_mm[1], mn1); atomicMin(&s_mm[2], mn2);
      atomicMax(&s_mm[3], mx0); atomicMax(&s_mm[4], mx1); atomicMax(&s_mm[5], mx2);
    }
  }
  cluster.sync();
  {
#pragma unroll
    for (int d = 0; d < 6; d++) mm[d] = d < 3 ? 0x7fffffff : (int)0x80000000;
    for (int c = 0; c < CL; c++) {
      const int* peer = cluster.map_shared_rank(s_mm, c);
#pragma unroll
      for (int d = 0; d < 3; d++) { mm[d] = min(mm[d], peer[d]); mm[3 + d] = max(mm[3 + d], peer[3 + d]); }
    }
  }
}

// stable LSD radix sort of the (key, value) pairs held in the cluster's distributed shared memory (CL x PER x 1024 pairs, every CTA
// full), ascending by the 32-bit key: 4 passes of 8 bits; the scatter writes straight into the peer CTAs' shared memory
template <int CL, int PER>
__device__ __forceinline__ void cluster_radix_sort(cg::cluster_group& cluster, const ClusterSmem& S, int rank) {
  uint2* buf = S.buf;
  unsigned short* wh = S.wh;
  int* cta_cnt = S.cta_cnt;
  int* base = S.base;
  int* s_mm = S.s_mm;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned int lt = (1u << lane) - 1u;
#pragma unroll 1
  for (int pass = 0; pass < 4; pass++) {
    const int shift = 8 * pass;
#ifdef B2R_BUILD_PROFILE
    if (pass == 0) B2R_MARK(3);
#endif
    for (int i = tid; i < 32 * 256 / 2; i += kBuildThreads) reinterpret_cast<unsigned int*>(wh)[i] = 0u;
    __syncthreads();
    // every warp ranks its own contiguous 32 * PER elements in order, 32 at a time: rank inside (warp, digit) = running count of the
    // digit in this warp + number of equal digits in lower lanes (stable).  The MATCH.ANY of a step does not depend on the running
    // counts, so the masks of up to 8 steps are taken first (independent, pipelined) and only the count updates — a shared-memory
    // read-modify-write by the digit's leader lane — run one after the other (the serial match + update chain was a large share of a pass
    // at 16 pairs per thread).
    uint2 e[PER];
    unsigned short off[PER];
    unsigned short* mywh = wh + warp * 256;
    constexpr int kHalf = PER < 8 ? PER : 8;
#pragma unroll
    for (int b0 = 0; b0 < PER; b0 += kHalf) {
      unsigned int peers[kHalf];
#pragma unroll
      for (int k = 0; k < kHalf; k++) {
        e[b0 + k] = buf[warp * (32 * PER) + (b0 + k) * 32 + lane];
        peers[k] = __match_any_sync(0xffffffffu, (e[b0 + k].x >> shift) & 255u);
      }
#pragma unroll
      for (int k = 0; k < kHalf; k++) {
        const unsigned int d = (e[b0 + k].x >> shift) & 255u;
        const int leader = __ffs(peers[k]) - 1;
        unsigned int bs = 0;
        if (lane == leader) { bs = mywh[d]; mywh[d] = (unsigned short)(bs + __popc(peers[k])); }
        bs = __shfl_sync(0xffffffffu, bs, leader);
        off[b0 + k] = (unsigned short)(bs + __popc(peers[k] & lt));
        __syncwarp();
      }
    }
    __syncthreads();
#ifdef B2R_BUILD_PROFILE
    if (pass == 0) B2R_MARK(4);
#endif
    // per digit: exclusive prefix over the warps (in place) and the CTA's count
    if (tid < 256) {
      int run = 0;
#pragma unroll 8
      for (int w = 0; w < 32; w++) { const int c = wh[w * 256 + tid]; wh[w * 256 + tid] = (unsigned short)run; run += c; }
      cta_cnt[tid] = run;
    }
#ifdef B2R_BUILD_PROFILE
    if (pass == 0) B2R_MARK(5);
#endif
    cluster.sync();  // every CTA has its elements in registers (its buffer may be overwritten) and its digit counts published
#ifdef B2R_BUILD_PROFILE
    if (pass == 0) B2R_MARK(6);
#endif
    if (tid < 256) {
      int tot = 0, before = 0;
      for (int c = 0; c < CL; c++) {
        const int v = cluster.map_shared_rank(cta_cnt, c)[tid];
        tot += v;
        if (c < rank) before += v;
      }
      // exclusive scan of the digit totals over the 256 digits (8 warps)
      int inc = tot;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
      if (lane == 31) s_mm[8 + warp] = inc;
      // (threads 0..255 are warps 0..7: a named barrier over them would do; the block barrier below is simpler)
      base[tid] = inc - tot + before;  // completed with the warp offsets after the barrier
    }
    __syncthreads();
    if (tid < 256) {
      int woff = 0;
      for (int w = 0; w < warp; w++) woff += s_mm[8 + w];
      base[tid] += woff;
    }
    __syncthreads();
#ifdef B2R_BUILD_PROFILE
    if (pass == 0) B2R_MARK(7);
#endif
#pragma unroll
    for (int b = 0; b < PER; b++) {
      const unsigned int d = (e[b].x >> shift) & 255u;
      const int dst = base[d] + (int)mywh[d] + (int)off[b];
      uint2* peer = cluster.map_shared_rank(buf, dst >> BuildGeom<PER>::kShift);
      peer[dst & (BuildGeom<PER>::kCap - 1)] = e[b];
    }
#ifdef B2R_BUILD_PROFILE
    if (pass == 0) B2R_MARK(8);
#endif
    cluster.sync();  // all scatters have landed before anybody reads its buffer again
#ifdef B2R_BUILD_PROFILE
    if (pass == 0) B2R_MARK(9);
#endif
  }

}

// SINGLE: the one cloud travels as a kernel parameter (no descriptor upload); else blockIdx.x / CL indexes the descriptor list.
// (Two instantiations rather than a run-time select between a parameter-space struct and a global one.)
template <int CL, int PER, bool SINGLE>
__global__ void __launch_bounds__(kBuildThreads, 1) k_bvh_build_cluster(const BuildItem* __restrict__ items, const __grid_constant__ BuildItem single) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int kCap = BuildGeom<PER>::kCap;
  const ClusterSmem S = cluster_smem<PER>(smem_raw);
  uint2* buf = S.buf;
  unsigned short* wh = S.wh;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  BuildItem it;
  if constexpr (SINGLE) it = single;
  else it = items[blockIdx.x / CL];
  const int n = it.n;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int padded = ((n + 1023) / 1024) * 1024;
  const int g0 = rank * kCap;  // first global position / element index of this CTA's slice

  B2R_MARK(0);
  int mm[6];
  cluster_bbox<CL, PER>(cluster, S, it.raw, it.stride_f, n, g0, mm);
  B2R_MARK(1);
  // ---- 30-bit Hilbert keys (k_morton_keys's arithmetic) into this CTA's slice
  {
    const float mnx = ord2f(mm[0]), mny = ord2f(mm[1]), mnz = ord2f(mm[2]);
    const float ext = fmaxf(fmaxf(ord2f(mm[3]) - mnx, ord2f(mm[4]) - mny), fmaxf(ord2f(mm[5]) - mnz, 1.0e-6f));
    const float sc = 1023.0f / ext;
#pragma unroll 4
    for (int b = 0; b < PER; b++) {
      const int e = warp * (32 * PER) + b * 32 + lane;
      const int i = g0 + e;
      unsigned int key = 0xffffffffu;  // non-finite points and the padding sort last
      if (i < n) {
        const float* p = it.raw + (size_t)i * it.stride_f;
        const float x = p[0], y = p[1], z = p[2];
        if (finite3(x, y, z)) {
          const unsigned int ix = (unsigned int)fminf(fmaxf((x - mnx) * sc, 0.f), 1023.f);
          const unsigned int iy = (unsigned int)fminf(fmaxf((y - mny) * sc, 0.f), 1023.f);
          const unsigned int iz = (unsigned int)fminf(fmaxf((z - mnz) * sc, 0.f), 1023.f);
          key = hilbert30(ix, iy, iz);
        }
      }
      buf[e] = make_uint2(key, i < n ? (unsigned int)i : 0xffffffffu);
    }
  }
  __syncthreads();
  B2R_MARK(2);

  cluster_radix_sort<CL, PER>(cluster, S, rank);
  B2R_MARK(10);

  // ---- emit this CTA's slice of the structure (k_bvh_leaves's work): one super-node (1024 positions, 32 leaves) per step.
  // The point of step j + 1 is gathered while step j is reduced (the gather is an L2 round trip), and the boxes are reduced with
  // REDUX on order-preserving ints: 6 instructions per warp instead of 30 shuffle + min/max pairs (min / max are exact either way).
  float* s_lo = reinterpret_cast<float*>(wh);        // [32][3] leaf boxes of the current super-node (the histogram area is free now)
  float* s_hi = s_lo + 96;
  const int nstep = min(kCap / 1024, max(0, (padded - g0 + 1023) / 1024));
  uint2 kv = nstep > 0 ? buf[tid] : make_uint2(0xffffffffu, 0xffffffffu);
  float nx = INFINITY, ny = INFINITY, nz = INFINITY;
  if (kv.x != 0xffffffffu) { const float* p = it.raw + (size_t)kv.y * it.stride_f; nx = p[0]; ny = p[1]; nz = p[2]; }
  for (int j = 0; j < nstep; j++) {
    const int sg = g0 + j * 1024 + tid;              // global sorted position
    const uint2 cur = kv;
    const float x = nx, y = ny, z = nz;
    if (j + 1 < nstep) {                             // next step's record in flight during this step's reductions
      kv = buf[(j + 1) * 1024 + tid];
      nx = ny = nz = INFINITY;
      if (kv.x != 0xffffffffu) { const float* p = it.raw + (size_t)kv.y * it.stride_f; nx = p[0]; ny = p[1]; nz = p[2]; }
    }
    int idx = kPadIdx;
    if (cur.x != 0xffffffffu) {
      idx = (int)cur.y;
      it.pos_of[idx] = sg;
    } else if (cur.y != 0xffffffffu) {
      it.pos_of[cur.y] = -1;                         // a non-finite point of the cloud: dropped from the structure
    }
    it.sorted[sg] = make_float4(x, y, z, bits_idx(idx));
    const bool valid = idx != kPadIdx;
    const int kInfP = f2ord(INFINITY), kInfN = f2ord(-INFINITY);
    const int lx = __reduce_min_sync(0xffffffffu, valid ? f2ord(x) : kInfP), ly = __reduce_min_sync(0xffffffffu, valid ? f2ord(y) : kInfP),
              lz = __reduce_min_sync(0xffffffffu, valid ? f2ord(z) : kInfP);
    const int hx = __reduce_max_sync(0xffffffffu, valid ? f2ord(x) : kInfN), hy = __reduce_max_sync(0xffffffffu, valid ? f2ord(y) : kInfN),
              hz = __reduce_max_sync(0xffffffffu, valid ? f2ord(z) : kInfN);
    const int leaf = sg >> 5;
    int* s_lo_i = reinterpret_cast<int*>(s_lo);
    int* s_hi_i = reinterpret_cast<int*>(s_hi);
    if (lane == 0) {
      it.leaf_lo[leaf] = make_float4(ord2f(lx), ord2f(ly), ord2f(lz), 0.f);
      it.leaf_hi[leaf] = make_float4(ord2f(hx), ord2f(hy), ord2f(hz), 0.f);
      s_lo_i[warp * 3 + 0] = lx; s_lo_i[warp * 3 + 1] = ly; s_lo_i[warp * 3 + 2] = lz;
      s_hi_i[warp * 3 + 0] = hx; s_hi_i[warp * 3 + 1] = hy; s_hi_i[warp * 3 + 2] = hz;
    }
    __syncthreads();
    if (warp == 0) {
      const int ax = __reduce_min_sync(0xffffffffu, s_lo_i[lane * 3 + 0]), ay = __reduce_min_sync(0xffffffffu, s_lo_i[lane * 3 + 1]),
                az = __reduce_min_sync(0xffffffffu, s_lo_i[lane * 3 + 2]);
      const int bx = __reduce_max_sync(0xffffffffu, s_hi_i[lane * 3 + 0]), by = __reduce_max_sync(0xffffffffu, s_hi_i[lane * 3 + 1]),
                bz = __reduce_max_sync(0xffffffffu, s_hi_i[lane * 3 + 2]);
      if (lane == 0) {
        it.sup_lo[sg >> 10] = make_float4(ord2f(ax), ord2f(ay), ord2f(az), 0.f);
        it.sup_hi[sg >> 10] = make_float4(ord2f(bx), ord2f(by), ord2f(bz), 0.f);
      }
    }
    __syncthreads();
  }
#ifdef B2R_BUILD_PROFILE
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    const long long t = clock64();
    printf("build n=%d CL=%d PER=%d cycles: bbox %lld keys %lld | pass0: zero+rank %lld warp-prefix %lld sync %lld digit-scan %lld scatter %lld sync %lld | sort total %lld | emit %lld | all %lld\n",
           n, CL, PER, b2r_marks[1] - b2r_marks[0], b2r_marks[2] - b2r_marks[1], b2r_marks[4] - b2r_marks[3], b2r_marks[5] - b2r_marks[4], b2r_marks[6] - b2r_marks[5],
           b2r_marks[7] - b2r_marks[6], b2r_marks[8] - b2r_marks[7], b2r_marks[9] - b2r_marks[8], b2r_marks[10] - b2r_marks[2], t - b2r_marks[10], t - b2r_marks[0]);
  }
#endif
}
#endif  // __CUDACC__

}  // namespace b2r
