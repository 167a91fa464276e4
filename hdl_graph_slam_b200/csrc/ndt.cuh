// ndt.cuh — NDT kernels and host driver.
//
// Re-creates, GPU-first, pclomp::NormalDistributionsTransform + pclomp::VoxelGridCovariance (koide3/ndt_omp; SURVEY.md
// A.2/A.3) — the reference factory's default engine (/root/reference/src/hdl_graph_slam/registrations.cpp:26,101-120):
//   ndt_build_map (k_vox_*)   <- setInputTarget -> VoxelGridCovariance::filter/applyFilter (voxel Gaussians: mean, cov, icov)
//   k_ndt_derivatives         <- computeDerivatives + computePointDerivatives + updateDerivatives, DIRECT1 / DIRECT7
//                                (sum of full Gaussians of the containing cell and its 6 face neighbours, NOT trilinear)
//   k_ndt_hessian             <- computeHessian / updateHessian (float64 path, reached only when the More-Thuente loop ran)
//   ndt_align                 <- computeTransformation + computeStepLengthMT (+ trialValueSelectionMT / updateIntervalMT)
// Per-(point,cell) math is float32 in exactly the operation order of oracle/ndt.cpp::ndt_point_cell (non-contracted
// intrinsics), exp as (float)exp((double)x); accumulation float64 with a fixed reduction tree.
#pragma once
#include <cmath>
#include <cstring>
#include <vector>
#include <algorithm>
#include "engine.cuh"
#include "gicp.cuh"  // block_reduce / finish_partials
#include "linalg.cuh"

namespace b2r {

struct VoxGeom {
  float leaf, inv_leaf;
  int min_b[3], max_b[3], div_b[3];
  int ok;       // 0: dx*dy*dz exceeds int32 (PCL's own limit: "Leaf size is too small for the input dataset")
  int empty;    // no finite points
};

struct __align__(16) NdtVoxel {  // full float64 record (parity dump, float64 Hessian pass)
  double mean[3];
  double icov[9];
  int npts;     // number of points, -1 = invalidated (bad eigenvalues / infinite icov)
  int pad[3];
};  // 112 bytes

struct __align__(16) NdtCell {   // what a derivative pass reads per (point, cell): 64 bytes, staged in shared memory
  double mean[3];
  float icov[9];                 // (float)icov: exactly the cast ndt_omp / the oracle apply per (point, cell)
  int npts;
};
static_assert(sizeof(NdtCell) == 64, "NdtCell layout");

constexpr unsigned long long kNdtEmpty = 0xffffffffffffffffull;

// Sparse voxel map: the reference's VoxelGridCovariance keeps its leaves in a std::map keyed by the linearised ijk, limited only by
// int32 indices.  Here: points radix-sorted by that key, one record per occupied voxel at the sorted position of its first point,
// and an open-addressing hash table (key -> position).  No dense table: a 200 m extent at 0.5 m resolution (16 M cells, the
// effective setting of hdl_graph_slam_imu.launch) costs what its ~10^4 occupied voxels cost.
struct NdtVoxelMap {
  VoxGeom* geom = nullptr;      // device
  VoxGeom h_geom;               // host copy (valid after ndt_sync_geom)
  bool h_geom_valid = false;
  DevBuf<unsigned int> keys;    // sorted voxel keys (n), 0xffffffff = dropped (non-finite) point
  DevBuf<float4> sorted;        // (x,y,z,bits(idx)) ascending (voxel key, index)
  DevBuf<NdtVoxel> vox;         // record of a voxel lives at the sorted position of its first point
  DevBuf<NdtCell> cells;        // compact twin of vox
  DevBuf<unsigned long long> table;  // (pos << 32) | key, kNdtEmpty = free
  unsigned int mask = 0;
  size_t n = 0;
};

struct NdtWork {
  DevBuf<double> partials;
  DevBuf<double> grows;           // derivative pass: group rows of the two-level sum
  DevBuf<unsigned int> gcount;    // derivative pass: per-group arrival counters (zero between launches)
  unsigned long long* d_queue = nullptr;  // chunk ticket counter, monotone over launches
  unsigned long long qnext = 0;   // first ticket of the next launch
  double* d_out = nullptr;        // 64 doubles
  unsigned int* d_counter = nullptr;
  double* h_out = nullptr;        // pinned + mapped: kernels write their results here directly
  double* h_out_dev = nullptr;    // device alias of h_out
  unsigned long long* h_flag = nullptr; unsigned long long* h_flag_dev = nullptr; unsigned long long seq = 0;
  VoxGeom* h_geom_pinned = nullptr;
  unsigned long long* d_pairs = nullptr;
  BuildCtx* bc = nullptr;         // build scratch of the handle's main stream (keys / values / sort space)
  Telemetry* tel = nullptr;
  void release() {
    partials.release(); grows.release(); gcount.release();
    if (d_queue) cudaFree(d_queue);
    d_queue = nullptr;
    if (d_out) cudaFree(d_out);
    if (d_counter) cudaFree(d_counter);
    if (h_out) cudaFreeHost(h_out);
    if (h_geom_pinned) cudaFreeHost(h_geom_pinned);
    if (d_pairs) cudaFree(d_pairs);
    d_out = nullptr; d_counter = nullptr; h_out = nullptr; h_geom_pinned = nullptr; d_pairs = nullptr;
  }
};

inline void ndt_free_map(NdtVoxelMap* m) {
  if (!m) return;
  if (m->geom) cudaFree(m->geom);
  m->keys.release(); m->sorted.release(); m->vox.release(); m->cells.release(); m->table.release();
  delete m;
}

// ------------------------------------------------------------------------------------------------ voxel build kernels
// VoxelGridCovariance::applyFilter geometry (A.3): min_b = floor(min_p * inv_leaf) ...
__global__ void k_vox_params(const int* mm, VoxGeom* vg, int n, float leaf) {
  VoxGeom V;
  V.leaf = leaf;
  V.inv_leaf = 1.0f / leaf;
  V.ok = 1;
  V.empty = 0;
  if (n <= 0 || mm[0] == 0x7fffffff) {
    V.empty = 1;
    for (int d = 0; d < 3; d++) { V.min_b[d] = 0; V.max_b[d] = 0; V.div_b[d] = 1; }
    *vg = V;
    return;
  }
  double cells = 1.0;
  for (int d = 0; d < 3; d++) {
    float mn = ord2f(mm[d]), mx = ord2f(mm[3 + d]);
    float a = floorf(fmul(mn, V.inv_leaf)), b = floorf(fmul(mx, V.inv_leaf));
    if (!(a > -1.0e9f && b < 1.0e9f)) { V.ok = 0; a = 0.f; b = 0.f; }
    V.min_b[d] = (int)a;
    V.max_b[d] = (int)b;
    V.div_b[d] = V.max_b[d] - V.min_b[d] + 1;
    cells *= (double)V.div_b[d];
  }
  if (cells > 2147483647.0) V.ok = 0;  // int32 linear index, as PCL
  *vg = V;
}

__device__ __forceinline__ unsigned int vox_key_of_point(const VoxGeom& V, float x, float y, float z) {
  // ijk = (int)(floor(p * inv_leaf) - (float)min_b)   (float32, as in VoxelGridCovariance / VoxelGrid)
  int i0 = (int)fsub(floorf(fmul(x, V.inv_leaf)), (float)V.min_b[0]);
  int i1 = (int)fsub(floorf(fmul(y, V.inv_leaf)), (float)V.min_b[1]);
  int i2 = (int)fsub(floorf(fmul(z, V.inv_leaf)), (float)V.min_b[2]);
  i0 = clampi(i0, 0, V.div_b[0] - 1); i1 = clampi(i1, 0, V.div_b[1] - 1); i2 = clampi(i2, 0, V.div_b[2] - 1);
  return (unsigned int)i0 + (unsigned int)i1 * (unsigned int)V.div_b[0] + (unsigned int)i2 * (unsigned int)V.div_b[0] * (unsigned int)V.div_b[1];
}

__global__ void k_vox_keys(const float* __restrict__ raw, int stride_f, int n, const VoxGeom* __restrict__ vg, unsigned int* keys, int* vals) {
  const VoxGeom V = *vg;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float* p = raw + (size_t)i * stride_f;
    const float x = p[0], y = p[1], z = p[2];
    unsigned int k = 0xffffffffu;  // dropped points sort last
    if (finite3(x, y, z)) k = V.ok ? vox_key_of_point(V, x, y, z) : 0u;
    keys[i] = k;
    vals[i] = i;
  }
}

__global__ void k_vox_gather(const float* __restrict__ raw, int stride_f, int n, const unsigned int* __restrict__ keys_sorted, const int* __restrict__ vals_sorted,
                             float4* sorted) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
    const int i = vals_sorted[s];
    const float* p = raw + (size_t)i * stride_f;
    sorted[s] = (keys_sorted[s] != 0xffffffffu) ? make_float4(p[0], p[1], p[2], bits_idx(i)) : make_float4(0.f, 0.f, 0.f, bits_idx(kPadIdx));
  }
}

__device__ __forceinline__ unsigned int ndt_hash(unsigned int key) {
  key ^= key >> 16; key *= 0x7feb352du; key ^= key >> 15; key *= 0x846ca68bu; key ^= key >> 16;
  return key;
}

// One thread per voxel (the thread at the sorted position of the voxel's first point): sequential float64 moments in
// ascending point index, the finalisation of VoxelGridCovariance::applyFilter, and the hash-table insert.
__global__ void k_vox_finalize(const unsigned int* __restrict__ keys_sorted, const float4* __restrict__ sorted, NdtVoxel* vox, NdtCell* cells,
                               unsigned long long* table, unsigned int mask, int n) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const unsigned int key = keys_sorted[s];
  if (key == 0xffffffffu) return;
  if (s > 0 && keys_sorted[s - 1] == key) return;  // not the first point of its voxel
  int cnt = 0;
  double sx = 0, sy = 0, sz = 0, cxx = 0, cxy = 0, cxz = 0, cyy = 0, cyz = 0, czz = 0;
  for (int j = s; j < n && keys_sorted[j] == key; j++) {
    const float4 p = sorted[j];
    const double x = (double)p.x, y = (double)p.y, z = (double)p.z;
    sx += x; sy += y; sz += z;
    // products of two float32 values are exact in float64, so contraction cannot change these sums
    cxx += x * x; cxy += x * y; cxz += x * z; cyy += y * y; cyz += y * z; czz += z * z;
    cnt++;
  }
  NdtVoxel R;
  const double nn = (double)cnt;
  R.mean[0] = sx / nn; R.mean[1] = sy / nn; R.mean[2] = sz / nn;
  R.npts = cnt;
  R.pad[0] = R.pad[1] = R.pad[2] = 0;
  for (int k = 0; k < 9; k++) R.icov[k] = 0.0;
  if (cnt >= 6) {
    const double S[3] = {sx, sy, sz};
    const double S2[9] = {cxx, cxy, cxz, cxy, cyy, cyz, cxz, cyz, czz};
    double cov[9];
    const double f = __ddiv_rn(__dsub_rn(nn, 1.0), nn);
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
      for (int bb = 0; bb < 3; bb++) {
        // cov = (S2 - 2*(sum*mean^T))/n + mean*mean^T ; cov *= (n-1)/n       (non-contracted, as the oracle)
        double t = __dmul_rn(2.0, __dmul_rn(S[a], R.mean[bb]));
        t = __ddiv_rn(__dsub_rn(S2[a * 3 + bb], t), nn);
        t = __dadd_rn(t, __dmul_rn(R.mean[a], R.mean[bb]));
        cov[a * 3 + bb] = __dmul_rn(t, f);
      }
    double w[3], V[9];
    sym_eigen3(cov, w, V);
    if (w[0] < 0 || w[1] < 0 || w[2] <= 0) {
      R.npts = -1;
    } else {
      const double minv = 0.01 * w[2];
      if (w[0] < minv) {
        w[0] = minv;
        if (w[1] < minv) w[1] = minv;
        double Vi[9], VD[9];
        inv3(V, Vi);
#pragma unroll
        for (int a = 0; a < 3; a++)
#pragma unroll
          for (int bb = 0; bb < 3; bb++) VD[a * 3 + bb] = V[a * 3 + bb] * w[bb];
        mul3(VD, Vi, cov);
      }
      inv3(cov, R.icov);
      double mxv = -INFINITY, mnv = INFINITY;
      bool nan_in = false;
#pragma unroll
      for (int a = 0; a < 9; a++) { mxv = fmax(mxv, R.icov[a]); mnv = fmin(mnv, R.icov[a]); nan_in |= (R.icov[a] != R.icov[a]); }
      if (mxv == INFINITY || mnv == -INFINITY || nan_in) R.npts = -1;
    }
  }
  vox[s] = R;
  NdtCell C;
  C.mean[0] = R.mean[0]; C.mean[1] = R.mean[1]; C.mean[2] = R.mean[2];
#pragma unroll
  for (int k = 0; k < 9; k++) C.icov[k] = (float)R.icov[k];
  C.npts = R.npts;
  cells[s] = C;
  // insert (key -> s): every key is inserted exactly once, so the first free slot of the probe sequence is taken with one CAS
  const unsigned long long entry = ((unsigned long long)(unsigned int)s << 32) | (unsigned long long)key;
  unsigned int h = ndt_hash(key) & mask;
  while (atomicCAS(table + h, kNdtEmpty, entry) != kNdtEmpty) h = (h + 1) & mask;
}

// ------------------------------------------------------------------------------------------------ derivative kernel
constexpr int kNdtThreads = 128;
constexpr int kNdtAccA = 28;   // first sweep over a point's cells: score, g[6], upper triangle of H (21)
constexpr int kNdtAccB = 15;   // second sweep: strict lower triangle of H (ndt_omp's float32 Hessian is NOT symmetric to the last bit)
constexpr int kNdtAcc = kNdtAccA + kNdtAccB;
constexpr int kNdtSlots = 320; // voxel records staged per block (20 KB)

struct NdtArgs {
  const float4* src;           // the source's Hilbert-sorted points (bvh.cuh): a block's 128 points are spatial neighbours
  int n_sorted;
  const VoxGeom* geom;
  const unsigned long long* table;
  unsigned int mask;
  const NdtCell* cells;
  const NdtVoxel* vox;
  float Tf[12];
  float jang[8][3];
  float hang[15][3];
  double jang_d[8][3];
  double hang_d[15][3];
  double d1, d2;
  int ncell_search;  // 1 or 7
  int compute_hessian;
  double* partials;            // derivative pass: one row of kNdtAcc sums per 128-point chunk; Hessian pass: [blocks][36]
  double* grows;               // derivative pass: one row per group of 32 chunks
  unsigned int* gcount;        // chunks of a group that have delivered their row (zero between launches)
  unsigned long long* queue;   // chunk tickets: monotone over launches, this launch's start at qbase
  unsigned long long qbase;
  double* out;
  unsigned int* counter;
  unsigned long long* pairs;
  unsigned long long* flag;  // host-mapped completion flag
  unsigned long long seq;
};

__device__ __forceinline__ float dot3f(const float* a, float x, float y, float z) {
  return fadd(fadd(fmul(a[0], x), fmul(a[1], y)), fmul(a[2], z));
}

__constant__ int c_off7[7][3] = {{0, 0, 0}, {1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};

// VoxelGridCovariance::getNeighborhoodAtPoint's leaf lookup: in-bounds test against min_b / max_b, then leaves_.find(idx).
// Returns the position of the voxel record or -1.
__device__ __forceinline__ int ndt_find(const unsigned long long* __restrict__ table, unsigned int mask, const VoxGeom& V, int cx, int cy, int cz) {
  if (cx < V.min_b[0] || cx > V.max_b[0] || cy < V.min_b[1] || cy > V.max_b[1] || cz < V.min_b[2] || cz > V.max_b[2]) return -1;
  const unsigned int key = (unsigned int)(cx - V.min_b[0]) + (unsigned int)(cy - V.min_b[1]) * (unsigned int)V.div_b[0] +
                           (unsigned int)(cz - V.min_b[2]) * (unsigned int)V.div_b[0] * (unsigned int)V.div_b[1];
  unsigned int h = ndt_hash(key) & mask;
  for (;;) {
    const unsigned long long e = __ldg(table + h);
    if ((unsigned int)e == key) return (int)(e >> 32);
    if (e == kNdtEmpty) return -1;
    h = (h + 1) & mask;
  }
}

// computeDerivatives (DIRECT1 / DIRECT7) over the Hilbert-sorted source.  A block's 128 points are neighbours in space, so
// the voxel records they need (<= 7 per point) form a small box of cells: the block looks every cell of that box up ONCE,
// stages the 64-byte records in shared memory, and the per-(point, cell) loop then runs without a global load.  Blocks
// whose points are spread too wide for the staging area (far-field leaves, jumps of the curve) fall back to direct lookups.
//
// Work distribution and summation order (round 2, late): the 128-point CHUNKS of the source are handed out through a ticket
// counter (a resident block takes the next chunk when it is done with its own), every chunk reduces to its OWN row of 43
// float64 sums, and the rows are added by a fixed two-level tree (32 chunk rows -> one group row by whichever block completes
// the group, group rows -> result by whichever block completes the last group).  The sums therefore do not depend on which
// block processed which chunk — bitwise reproducible — while no SM waits for a statically assigned heavy block (with a static
// persistent grid the slowest SM sub-partition ran far longer than the mean, much of it the single last block adding its rows of
// partials in a chain of dependent memory round trips).
// (Tried and dropped: fully warp-autonomous 32-point sub-chunks with warp tickets and a three-level tree — no block barrier at
// all — was slower per pass than this version: the barrier stalls turn into long-scoreboard and fence stalls, and the tail does
// not shrink because it is set by work units per resident slot, not by the unit's size.)
constexpr int kNdtRow = 136;  // float64 elements per shared-memory row of per-thread values (128 + 8: half-warps hit distinct banks)

// sums of R (<= 16) rows of 128 per-thread values -> dst[0..R): thread (row = tid >> 3, part = tid & 7) adds the elements part,
// part + 8, ... of its row in ascending order, three butterfly levels join the 8 parts.  The order is fixed.
__device__ __forceinline__ void ndt_rows_sum(const double* rows, int R, double* dst) {
  const int row = threadIdx.x >> 3, part = threadIdx.x & 7;
  double s = 0.0;
  if (row < R) {
    const double* p = rows + row * kNdtRow + part;
#pragma unroll
    for (int j = 0; j < 16; j++) s += p[8 * j];
  }
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  if (row < R && part == 0) dst[row] = s;
}

template <bool HESS>
__global__ void __launch_bounds__(kNdtThreads, 4) k_ndt_derivatives(const __grid_constant__ NdtArgs A) {
  __shared__ __align__(16) NdtCell s_cell[kNdtSlots];  // staged voxel records; after the pair loop: rows of the register sums
  __shared__ double s_low[kNdtAccB][kNdtRow];          // strict lower triangle of H: one float64 column per thread (no conflicts, no sync)
  __shared__ double s_fin[kNdtAcc];
  __shared__ int s_box[6];
  __shared__ int s_chunk, s_role;
  static_assert(sizeof(NdtCell) * kNdtSlots >= sizeof(double) * 14 * kNdtRow, "the reduction rows reuse the staging area");
  constexpr int NV = HESS ? kNdtAcc : 7;  // values that carry information (score + gradient without the Hessian)
  const int lane = threadIdx.x & 31;
  const VoxGeom V = *A.geom;
  const int nchunks = A.n_sorted / kNdtThreads;  // n_sorted is a multiple of 1024
  const int p1 = A.n_sorted;
  for (;;) {
  if (threadIdx.x == 0) s_chunk = (int)(atomicAdd(A.queue, 1ull) - A.qbase);  // tickets of this launch start at qbase (ndt_run_pass)
  __syncthreads();
#ifdef B2R_NDT_STRIDE  // experiment: visit the chunks in a scattered order (heavy regions of the Hilbert order spread over the pass)
  const int chunk = s_chunk >= nchunks ? s_chunk : (int)(((long long)s_chunk * B2R_NDT_STRIDE) % nchunks);
#else
  const int chunk = s_chunk;
#endif
  if (chunk >= nchunks) break;  // block-uniform
  double acc[kNdtAccA];
#pragma unroll
  for (int k = 0; k < kNdtAccA; k++) acc[k] = 0.0;
  if (HESS) {
#pragma unroll
    for (int q = 0; q < kNdtAccB; q++) s_low[q][threadIdx.x] = 0.0;
  }
  unsigned int npairs = 0;
  const int base = chunk * kNdtThreads;
  const int s = base + threadIdx.x;
  float4 pt = make_float4(0.f, 0.f, 0.f, bits_idx(kPadIdx));
  if (s < p1) pt = A.src[s];
  const float x = pt.x, y = pt.y, z = pt.z;
  float xt = 0.f, yt = 0.f, zt = 0.f;
  int ci = 0, cj = 0, ck = 0;
  bool valid = false;
  if (idx_bits(pt.w) != kPadIdx && !V.empty && V.ok) {
    xt = xform_row(A.Tf[0], A.Tf[1], A.Tf[2], A.Tf[3], x, y, z);
    yt = xform_row(A.Tf[4], A.Tf[5], A.Tf[6], A.Tf[7], x, y, z);
    zt = xform_row(A.Tf[8], A.Tf[9], A.Tf[10], A.Tf[11], x, y, z);
    if (finite3(xt, yt, zt)) {
      // getNeighborhoodAtPoint{1,7}: ijk = floor(pt / leaf)   (float32 DIVISION here, multiply-by-inverse at build)
      const float fi = floorf(__fdiv_rn(xt, V.leaf)), fj = floorf(__fdiv_rn(yt, V.leaf)), fk = floorf(__fdiv_rn(zt, V.leaf));
      if (fabsf(fi) < 1.0e9f && fabsf(fj) < 1.0e9f && fabsf(fk) < 1.0e9f) { ci = (int)fi; cj = (int)fj; ck = (int)fk; valid = true; }
    }
  }
  // ---- the block's box of base cells (+-1 for the face neighbours)
  if (threadIdx.x < 6) s_box[threadIdx.x] = threadIdx.x < 3 ? 0x7fffffff : (int)0x80000000;
  __syncthreads();
  {
    int lo0 = valid ? ci : 0x7fffffff, lo1 = valid ? cj : 0x7fffffff, lo2 = valid ? ck : 0x7fffffff;
    int hi0 = valid ? ci : (int)0x80000000, hi1 = valid ? cj : (int)0x80000000, hi2 = valid ? ck : (int)0x80000000;
    lo0 = __reduce_min_sync(0xffffffffu, lo0); lo1 = __reduce_min_sync(0xffffffffu, lo1); lo2 = __reduce_min_sync(0xffffffffu, lo2);
    hi0 = __reduce_max_sync(0xffffffffu, hi0); hi1 = __reduce_max_sync(0xffffffffu, hi1); hi2 = __reduce_max_sync(0xffffffffu, hi2);
    if (lane == 0 && lo0 <= hi0) {
      atomicMin(&s_box[0], lo0); atomicMin(&s_box[1], lo1); atomicMin(&s_box[2], lo2);
      atomicMax(&s_box[3], hi0); atomicMax(&s_box[4], hi1); atomicMax(&s_box[5], hi2);
    }
  }
  __syncthreads();
  const bool any = s_box[0] <= s_box[3];
  const int bx0 = s_box[0] - 1, by0 = s_box[1] - 1, bz0 = s_box[2] - 1;
  const long long ex = any ? (long long)s_box[3] - s_box[0] + 3 : 0, ey = any ? (long long)s_box[4] - s_box[1] + 3 : 0, ez = any ? (long long)s_box[5] - s_box[2] + 3 : 0;
  const bool staged = any && ex <= kNdtSlots && ey <= kNdtSlots && ez <= kNdtSlots && ex * ey * ez <= kNdtSlots;
  const int dx = (int)ex, dxy = (int)(ex * ey);
  if (staged) {
    const int vol = dxy * (int)ez;
    for (int slot = threadIdx.x; slot < vol; slot += blockDim.x) {
      const int cz = slot / dxy, r = slot - cz * dxy, cy = r / dx, cx = r - cy * dx;
      const int pos = ndt_find(A.table, A.mask, V, bx0 + cx, by0 + cy, bz0 + cz);
      if (pos >= 0) {
        const uint4* g = reinterpret_cast<const uint4*>(A.cells + pos);
        uint4* d = reinterpret_cast<uint4*>(&s_cell[slot]);
        d[0] = __ldg(g); d[1] = __ldg(g + 1); d[2] = __ldg(g + 2); d[3] = __ldg(g + 3);
      } else {
        s_cell[slot].npts = -1;
      }
    }
  }
  __syncthreads();
  if (valid) {
    bool have_pd = false;
    float j13 = 0, j23 = 0, j04 = 0, j14 = 0, j24 = 0, j05 = 0, j15 = 0, j25 = 0;
    float ha1 = 0, ha2 = 0, hb1 = 0, hb2 = 0, hc1 = 0, hc2 = 0, hd0 = 0, hd1 = 0, hd2 = 0, he0 = 0, he1 = 0, he2 = 0, hf0 = 0, hf1 = 0, hf2 = 0;
    const float d2f = (float)A.d2;
    for (int c = 0; c < A.ncell_search; c++) {
      const int cx = ci + c_off7[c][0], cy = cj + c_off7[c][1], cz = ck + c_off7[c][2];
      const NdtCell* L;
      if (staged) {
        L = &s_cell[(cx - bx0) + (cy - by0) * dx + (cz - bz0) * dxy];
      } else {
        const int pos = ndt_find(A.table, A.mask, V, cx, cy, cz);
        if (pos < 0) continue;
        L = A.cells + pos;
      }
      if (L->npts < 6) continue;  // fewer than min_points_per_voxel, or invalidated (bad eigenvalues / infinite icov)
      npairs++;
      if (!have_pd) {  // computePointDerivatives(x): original point only
        j13 = dot3f(A.jang[0], x, y, z); j23 = dot3f(A.jang[1], x, y, z);
        j04 = dot3f(A.jang[2], x, y, z); j14 = dot3f(A.jang[3], x, y, z); j24 = dot3f(A.jang[4], x, y, z);
        j05 = dot3f(A.jang[5], x, y, z); j15 = dot3f(A.jang[6], x, y, z); j25 = dot3f(A.jang[7], x, y, z);
        if (HESS) {
          ha1 = dot3f(A.hang[0], x, y, z); ha2 = dot3f(A.hang[1], x, y, z);
          hb1 = dot3f(A.hang[2], x, y, z); hb2 = dot3f(A.hang[3], x, y, z);
          hc1 = dot3f(A.hang[4], x, y, z); hc2 = dot3f(A.hang[5], x, y, z);
          hd0 = dot3f(A.hang[6], x, y, z); hd1 = dot3f(A.hang[7], x, y, z); hd2 = dot3f(A.hang[8], x, y, z);
          he0 = dot3f(A.hang[9], x, y, z); he1 = dot3f(A.hang[10], x, y, z); he2 = dot3f(A.hang[11], x, y, z);
          hf0 = dot3f(A.hang[12], x, y, z); hf1 = dot3f(A.hang[13], x, y, z); hf2 = dot3f(A.hang[14], x, y, z);
        }
        have_pd = true;
      }
      const float q0 = (float)((double)xt - L->mean[0]), q1 = (float)((double)yt - L->mean[1]), q2 = (float)((double)zt - L->mean[2]);
      float C[9];
#pragma unroll
      for (int k = 0; k < 9; k++) C[k] = L->icov[k];
      // qC = q^T C ; gq[0..2] == qC
      float gq[6];
#pragma unroll
      for (int j = 0; j < 3; j++) gq[j] = fadd(fadd(fmul(q0, C[0 * 3 + j]), fmul(q1, C[1 * 3 + j])), fmul(q2, C[2 * 3 + j]));
      const float qCq = fadd(fadd(fmul(q0, gq[0]), fmul(q1, gq[1])), fmul(q2, gq[2]));
      const float arg = fmul(fmul(-d2f, qCq), 0.5f);
      float exv = (float)exp((double)arg);
      const float score_inc = (float)(-A.d1 * (double)exv);
      exv = fmul(d2f, exv);
      if (exv > 1.f || exv < 0.f || exv != exv) continue;  // contributes nothing (score_inc dropped as well)
      exv = (float)((double)exv * A.d1);
      // CJ columns 3..5 (columns 0..2 are C itself)
      float CJ3[3], CJ4[3], CJ5[3];
#pragma unroll
      for (int r = 0; r < 3; r++) {
        CJ3[r] = fadd(fmul(C[r * 3 + 1], j13), fmul(C[r * 3 + 2], j23));
        CJ4[r] = fadd(fadd(fmul(C[r * 3 + 0], j04), fmul(C[r * 3 + 1], j14)), fmul(C[r * 3 + 2], j24));
        CJ5[r] = fadd(fadd(fmul(C[r * 3 + 0], j05), fmul(C[r * 3 + 1], j15)), fmul(C[r * 3 + 2], j25));
      }
      gq[3] = fadd(fadd(fmul(q0, CJ3[0]), fmul(q1, CJ3[1])), fmul(q2, CJ3[2]));
      gq[4] = fadd(fadd(fmul(q0, CJ4[0]), fmul(q1, CJ4[1])), fmul(q2, CJ4[2]));
      gq[5] = fadd(fadd(fmul(q0, CJ5[0]), fmul(q1, CJ5[1])), fmul(q2, CJ5[2]));
      acc[0] += (double)score_inc;
#pragma unroll
      for (int k = 0; k < 6; k++) acc[1 + k] += (double)fmul(exv, gq[k]);
      if (HESS) {
        // All 36 entries of H exactly as ndt_omp writes them: its float32 expression is not symmetric to the last bit
        // ((-d2 g_i) g_j vs (-d2 g_j) g_i, J_j^T C J_i vs J_i^T C J_j) and the Newton iteration is sensitive to it.  The 21 upper
        // entries accumulate in float64 registers, the 15 strictly lower ones in a float64 shared-memory column per thread (43
        // register accumulators would spill).  The term J_jj^T C J_ii is P[jj][ii] with
        // P[a][b] = J[:,a] . CJ[:,b], CJ[r][b]: b<3 -> C[r][b]; b=3 -> CJ3[r]; b=4 -> CJ4[r]; b=5 -> CJ5[r]
#define B2R_CJ(r, b) ((b) < 3 ? C[(r) * 3 + (b)] : ((b) == 3 ? CJ3[r] : ((b) == 4 ? CJ4[r] : CJ5[r])))
        // second-derivative terms qC . v_ij  (i,j in 3..5); a=(0,ha1,ha2) b=(0,hb1,hb2) c=(0,hc1,hc2) d,e,f full
        const float xa = fadd(fadd(fmul(gq[0], 0.f), fmul(gq[1], ha1)), fmul(gq[2], ha2));
        const float xb = fadd(fadd(fmul(gq[0], 0.f), fmul(gq[1], hb1)), fmul(gq[2], hb2));
        const float xc = fadd(fadd(fmul(gq[0], 0.f), fmul(gq[1], hc1)), fmul(gq[2], hc2));
        const float xd = fadd(fadd(fmul(gq[0], hd0), fmul(gq[1], hd1)), fmul(gq[2], hd2));
        const float xe = fadd(fadd(fmul(gq[0], he0), fmul(gq[1], he1)), fmul(gq[2], he2));
        const float xf = fadd(fadd(fmul(gq[0], hf0), fmul(gq[1], hf1)), fmul(gq[2], hf2));
        const float XH[3][3] = {{xa, xb, xc}, {xb, xd, xe}, {xc, xe, xf}};
        int hk = 7, lk = 0;
#pragma unroll
        for (int ii = 0; ii < 6; ii++) {
#pragma unroll
          for (int jj = 0; jj < 6; jj++) {
            float u = fmul(fmul(-d2f, gq[ii]), gq[jj]);
            const float xh = (ii >= 3 && jj >= 3) ? XH[ii - 3][jj - 3] : 0.f;
            u = fadd(u, xh);
            // P[jj][ii] = J[:,jj] . CJ[:,ii]
            float pj;
            if (jj < 3) pj = B2R_CJ(jj, ii);
            else if (jj == 3) pj = fadd(fmul(j13, B2R_CJ(1, ii)), fmul(j23, B2R_CJ(2, ii)));
            else if (jj == 4) pj = fadd(fadd(fmul(j04, B2R_CJ(0, ii)), fmul(j14, B2R_CJ(1, ii))), fmul(j24, B2R_CJ(2, ii)));
            else pj = fadd(fadd(fmul(j05, B2R_CJ(0, ii)), fmul(j15, B2R_CJ(1, ii))), fmul(j25, B2R_CJ(2, ii)));
            u = fadd(u, pj);
            const double w = (double)fmul(exv, u);
            if (jj >= ii) { acc[hk] += w; hk++; }                     // upper triangle + diagonal: registers
            else { s_low[lk][threadIdx.x] += w; lk++; }              // strict lower triangle: this thread's shared-memory column
          }
        }
#undef B2R_CJ
      }
    }
  }
  __syncthreads();  // the pair loop is over: s_cell becomes the reduction rows
  // pair count (integer, exact) through a warp reduction + one atomic per warp
  npairs = __reduce_add_sync(0xffffffffu, npairs);
  if (lane == 0 && npairs) atomicAdd(A.pairs, (unsigned long long)npairs);
  // ---- this chunk's row of sums
  double* tile = reinterpret_cast<double*>(s_cell);
  double* my_row = A.partials + (size_t)chunk * kNdtAcc;
#pragma unroll
  for (int k = 0; k < 14; k++) tile[k * kNdtRow + threadIdx.x] = acc[k];
  __syncthreads();
  ndt_rows_sum(tile, HESS ? 14 : 7, my_row);
  if (HESS) {
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 14; k++) tile[k * kNdtRow + threadIdx.x] = acc[14 + k];
    __syncthreads();
    ndt_rows_sum(tile, 14, my_row + 14);
    ndt_rows_sum(&s_low[0][0], kNdtAccB, my_row + kNdtAccA);
  }
  __syncthreads();  // the row is written (by several threads); s_cell / s_low / s_box are free for the next chunk
  // ---- fixed two-level tree over the chunk rows
  const int g = chunk >> 5;
  const int gsize = min(32, nchunks - (g << 5));
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int t = atomicAdd(A.gcount + g, 1u);
    const bool closes = t == (unsigned int)(gsize - 1);
    if (closes) A.gcount[g] = 0;  // all increments of this group are in: ready for the next launch
    s_role = closes ? 1 : 0;
  }
  __syncthreads();
  if (s_role) {  // block-uniform: this block completed group g and adds its rows in ascending chunk order
    __threadfence();
    if (threadIdx.x < NV) {
      const double* col = A.partials + (size_t)(g << 5) * kNdtAcc + threadIdx.x;
      double t[32];
#pragma unroll
      for (int u = 0; u < 32; u++) t[u] = (u < gsize) ? __ldcg(col + (size_t)u * kNdtAcc) : 0.0;  // 32 independent loads: one round trip
      double sum = 0.0;
#pragma unroll
      for (int u = 0; u < 32; u++) sum += t[u];
      A.grows[(size_t)g * kNdtAcc + threadIdx.x] = sum;
    }
    __syncthreads();
    const unsigned int ngroups = (unsigned int)((nchunks + 31) >> 5);
    if (threadIdx.x == 0) {
      __threadfence();
      const unsigned int t2 = atomicAdd(A.counter, 1u);
      const bool last = t2 == ngroups - 1;
      if (last) *A.counter = 0;
      s_role = last ? 2 : 0;
    }
    __syncthreads();
    if (s_role == 2) {  // the last group is in: add the group rows in ascending order and publish
      __threadfence();
      if (threadIdx.x < kNdtAcc) {
        double sum = 0.0;
        if (threadIdx.x < NV) {
          const double* col = A.grows + threadIdx.x;
          unsigned int r = 0;
          for (; r + 32 <= ngroups; r += 32) {
            double t[32];
#pragma unroll
            for (int u = 0; u < 32; u++) t[u] = __ldcg(col + (size_t)(r + u) * kNdtAcc);
#pragma unroll
            for (int u = 0; u < 32; u++) sum += t[u];
          }
          for (; r < ngroups; r++) sum += __ldcg(col + (size_t)r * kNdtAcc);
        }
        A.out[threadIdx.x] = sum;
        s_fin[threadIdx.x] = sum;
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        unsigned long long x = A.seq;
        const unsigned long long e = *reinterpret_cast<volatile unsigned long long*>(A.pairs);
        *A.pairs = 0;
        reinterpret_cast<unsigned long long*>(A.out)[kNdtAcc] = e;
        x ^= msg_mix(e, kNdtAcc);
        for (int i = 0; i < kNdtAcc; i++) x ^= msg_mix((unsigned long long)__double_as_longlong(s_fin[i]), i);
        reinterpret_cast<unsigned long long*>(A.out)[kNdtAcc + 1] = x;
        *reinterpret_cast<volatile unsigned long long*>(A.flag) = A.seq;
      }
    }
  }
  }
}


// float64 Hessian-only pass (ndt_omp computeHessian/updateHessian)
__global__ void __launch_bounds__(kNdtThreads) k_ndt_hessian(const __grid_constant__ NdtArgs A) {
  __shared__ double red[36 * 32];
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  double acc[36];
#pragma unroll
  for (int k = 0; k < 36; k++) acc[k] = 0.0;
  float4 pt = make_float4(0.f, 0.f, 0.f, bits_idx(kPadIdx));
  if (s < A.n_sorted) pt = A.src[s];
  if (idx_bits(pt.w) != kPadIdx) {
    const VoxGeom V = *A.geom;
    const float xf = pt.x, yf = pt.y, zf = pt.z;
    const float xt = xform_row(A.Tf[0], A.Tf[1], A.Tf[2], A.Tf[3], xf, yf, zf);
    const float yt = xform_row(A.Tf[4], A.Tf[5], A.Tf[6], A.Tf[7], xf, yf, zf);
    const float zt = xform_row(A.Tf[8], A.Tf[9], A.Tf[10], A.Tf[11], xf, yf, zf);
    if (!V.empty && V.ok && finite3(xt, yt, zt)) {
      const float fi = floorf(__fdiv_rn(xt, V.leaf)), fj = floorf(__fdiv_rn(yt, V.leaf)), fk = floorf(__fdiv_rn(zt, V.leaf));
      if (fabsf(fi) < 1.0e9f && fabsf(fj) < 1.0e9f && fabsf(fk) < 1.0e9f) {
        const int ci = (int)fi, cj = (int)fj, ck = (int)fk;
        const double x = (double)xf, y = (double)yf, z = (double)zf;
        double J[3][6] = {{1, 0, 0, 0, 0, 0}, {0, 1, 0, 0, 0, 0}, {0, 0, 1, 0, 0, 0}};
#define B2R_DJ(r) (x * A.jang_d[r][0] + y * A.jang_d[r][1] + z * A.jang_d[r][2])
#define B2R_DH(r) (x * A.hang_d[r][0] + y * A.hang_d[r][1] + z * A.hang_d[r][2])
        J[1][3] = B2R_DJ(0); J[2][3] = B2R_DJ(1); J[0][4] = B2R_DJ(2); J[1][4] = B2R_DJ(3); J[2][4] = B2R_DJ(4);
        J[0][5] = B2R_DJ(5); J[1][5] = B2R_DJ(6); J[2][5] = B2R_DJ(7);
        const double va[3] = {0, B2R_DH(0), B2R_DH(1)}, vb[3] = {0, B2R_DH(2), B2R_DH(3)}, vc[3] = {0, B2R_DH(4), B2R_DH(5)};
        const double vd[3] = {B2R_DH(6), B2R_DH(7), B2R_DH(8)}, ve[3] = {B2R_DH(9), B2R_DH(10), B2R_DH(11)}, vf[3] = {B2R_DH(12), B2R_DH(13), B2R_DH(14)};
#undef B2R_DJ
#undef B2R_DH
        for (int c = 0; c < A.ncell_search; c++) {
          const int pos = ndt_find(A.table, A.mask, V, ci + c_off7[c][0], cj + c_off7[c][1], ck + c_off7[c][2]);
          if (pos < 0) continue;
          const NdtVoxel* L = A.vox + pos;
          if (L->npts < 6) continue;
          const double q[3] = {(double)xt - L->mean[0], (double)yt - L->mean[1], (double)zt - L->mean[2]};
          const double* C = L->icov;
          double Cq[3];
          for (int r = 0; r < 3; r++) Cq[r] = C[r * 3 + 0] * q[0] + C[r * 3 + 1] * q[1] + C[r * 3 + 2] * q[2];
          double ex = A.d2 * exp(-A.d2 * (q[0] * Cq[0] + q[1] * Cq[1] + q[2] * Cq[2]) / 2);
          if (ex > 1 || ex < 0 || ex != ex) continue;
          ex *= A.d1;
          double CJ[3][6], qCJ[6];
          for (int r = 0; r < 3; r++)
            for (int k = 0; k < 6; k++) CJ[r][k] = C[r * 3 + 0] * J[0][k] + C[r * 3 + 1] * J[1][k] + C[r * 3 + 2] * J[2][k];
          for (int k = 0; k < 6; k++) qCJ[k] = q[0] * CJ[0][k] + q[1] * CJ[1][k] + q[2] * CJ[2][k];
#pragma unroll
          for (int ii = 0; ii < 6; ii++)
#pragma unroll
            for (int jj = 0; jj < 6; jj++) {
              double xh = 0;
              if (ii >= 3 && jj >= 3) {
                const int key = (ii - 3) * 3 + (jj - 3);
                const double* v = (key == 0) ? va : (key == 1 || key == 3) ? vb : (key == 2 || key == 6) ? vc : (key == 4) ? vd : (key == 5 || key == 7) ? ve : vf;
                double Cv[3];
                for (int r = 0; r < 3; r++) Cv[r] = C[r * 3 + 0] * v[0] + C[r * 3 + 1] * v[1] + C[r * 3 + 2] * v[2];
                xh = q[0] * Cv[0] + q[1] * Cv[1] + q[2] * Cv[2];
              }
              const double jcj = J[0][jj] * CJ[0][ii] + J[1][jj] * CJ[1][ii] + J[2][jj] * CJ[2][ii];
              acc[ii * 6 + jj] += ex * (-A.d2 * qCJ[ii] * qCJ[jj] + xh + jcj);
            }
        }
      }
    }
  }
  block_reduce<36>(acc, red);
  finish_partials<36>(acc, A.partials, A.out, A.counter, A.flag, A.seq);
}

// ------------------------------------------------------------------------------------------------ host side
inline int ndt_init_work(NdtWork& W) {
  if (W.d_out) return B2R_OK;
  B2R_CUDA(cudaMalloc(&W.d_out, 64 * sizeof(double)));
  B2R_CUDA(cudaMalloc(&W.d_counter, 4 * sizeof(unsigned int)));
  B2R_CUDA(cudaMemset(W.d_counter, 0, 4 * sizeof(unsigned int)));
  B2R_CUDA(cudaMalloc(&W.d_pairs, sizeof(unsigned long long)));
  B2R_CUDA(cudaMemset(W.d_pairs, 0, sizeof(unsigned long long)));
  B2R_CUDA(cudaMalloc(&W.d_queue, sizeof(unsigned long long)));
  B2R_CUDA(cudaMemset(W.d_queue, 0, sizeof(unsigned long long)));
  W.qnext = 0;
  B2R_CUDA(cudaHostAlloc(&W.h_out, 72 * sizeof(double), cudaHostAllocMapped));
  B2R_CUDA(cudaHostGetDevicePointer((void**)&W.h_out_dev, W.h_out, 0));
  W.h_flag = reinterpret_cast<unsigned long long*>(W.h_out + 64);
  W.h_flag_dev = reinterpret_cast<unsigned long long*>(W.h_out_dev + 64);
  *W.h_flag = 0;
  B2R_CUDA(cudaMallocHost(&W.h_geom_pinned, sizeof(VoxGeom)));
  return B2R_OK;
}

inline int ndt_ensure_map(const b2r_config& cfg, Cloud& c, NdtWork& W, cudaStream_t st) {
  if (c.ndt_ready) return B2R_OK;
  int rc = ndt_init_work(W);
  if (rc) return rc;
  BuildCtx* B = W.bc;
  if (!B) return fail(B2R_ESTATE, "internal: NDT build scratch not attached");
  if (!c.ndt) {
    c.ndt = new NdtVoxelMap();
    B2R_CUDA(cudaMalloc(&c.ndt->geom, sizeof(VoxGeom)));
  }
  NdtVoxelMap& M = *c.ndt;
  const int n = (int)c.n;
  M.n = c.n;
  M.h_geom_valid = false;
  size_t tsize = 1024;
  while (tsize < 2 * c.n) tsize <<= 1;
  M.mask = (unsigned int)(tsize - 1);
  B2R_CUDA(M.keys.reserve(c.n + 1));
  B2R_CUDA(M.sorted.reserve(c.n + 1));
  B2R_CUDA(M.vox.reserve(c.n + 1));
  B2R_CUDA(M.cells.reserve(c.n + 1));
  B2R_CUDA(M.table.reserve(tsize));
  B2R_CUDA(B->keys_a.reserve(c.n + 1)); B2R_CUDA(B->vals_a.reserve(c.n + 1)); B2R_CUDA(B->vals_b.reserve(c.n + 1));
  size_t tmp_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, B->keys_a.p, M.keys.p, B->vals_a.p, B->vals_b.p, n, 0, 32, st);
  B2R_CUDA(B->sort_tmp.reserve(tmp_bytes + 256));
  TEL_BEGIN(W.tel, st);
  k_grid_reset<<<1, 32, 0, st>>>(B->mm);
  int nb = n > 0 ? (n + 255) / 256 : 1;
  if (nb > 1184) nb = 1184;
  if (n > 0) k_bbox<<<nb, 256, 0, st>>>(c.raw_view, c.stride_f, n, B->mm);
  k_vox_params<<<1, 1, 0, st>>>(B->mm, M.geom, n, (float)cfg.ndt_resolution);
  B2R_CUDA(cudaMemsetAsync(M.table.p, 0xff, tsize * sizeof(unsigned long long), st));
  if (n > 0) {
    k_vox_keys<<<nb, 256, 0, st>>>(c.raw_view, c.stride_f, n, M.geom, B->keys_a.p, B->vals_a.p);
    size_t tb = B->sort_tmp.cap;
    // stable LSD radix sort by voxel key: inside a voxel the points stay in ascending index, the order the moments are summed in
    cub::DeviceRadixSort::SortPairs(B->sort_tmp.p, tb, B->keys_a.p, M.keys.p, B->vals_a.p, B->vals_b.p, n, 0, 32, st);
    k_vox_gather<<<nb, 256, 0, st>>>(c.raw_view, c.stride_f, n, M.keys.p, B->vals_b.p, M.sorted.p);
    k_vox_finalize<<<(n + 127) / 128, 128, 0, st>>>(M.keys.p, M.sorted.p, M.vox.p, M.cells.p, M.table.p, M.mask, n);
  }
  TEL_END(W.tel, KC_NDT_BUILD, n > 0 ? 10 : 4, st);
  B2R_CUDA(cudaGetLastError());
  c.ndt_ready = true;
  return B2R_OK;
}

inline int ndt_sync_geom(NdtVoxelMap& M, NdtWork& W, cudaStream_t st) {
  if (M.h_geom_valid) return B2R_OK;
  B2R_CUDA(cudaMemcpyAsync(W.h_geom_pinned, M.geom, sizeof(VoxGeom), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaStreamSynchronize(st));
  M.h_geom = *W.h_geom_pinned;
  M.h_geom_valid = true;
  if (!M.h_geom.ok) return fail(B2R_EUNSUPPORTED, "NDT voxel grid exceeds int32 indices (leaf size too small for the extent; PCL refuses the same input)");
  return B2R_OK;
}

inline int ndt_dump(Cloud& c, NdtWork& W, cudaStream_t st, size_t capacity, size_t* n_voxels, int64_t* keys, int32_t* npts, double* mean,
                    double* icov, int32_t* min_b, int32_t* div_b) {
  NdtVoxelMap& M = *c.ndt;
  int rc = ndt_sync_geom(M, W, st);
  if (rc) return rc;
  std::vector<unsigned int> ks(M.n + 1);
  std::vector<NdtVoxel> vox(M.n + 1);
  if (M.n) {
    B2R_CUDA(cudaMemcpyAsync(ks.data(), M.keys.p, M.n * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    B2R_CUDA(cudaMemcpyAsync(vox.data(), M.vox.p, M.n * sizeof(NdtVoxel), cudaMemcpyDeviceToHost, st));
  }
  B2R_CUDA(cudaStreamSynchronize(st));
  size_t V = 0;
  for (size_t s = 0; s < M.n; s++) {  // keys ascending: one record per run of equal keys, at the run's first position
    if (ks[s] == 0xffffffffu) break;
    if (s > 0 && ks[s - 1] == ks[s]) continue;
    if (V < capacity) {
      const NdtVoxel& L = vox[s];
      if (keys) keys[V] = (int64_t)ks[s];
      if (npts) npts[V] = L.npts;
      if (mean) std::memcpy(mean + V * 3, L.mean, 3 * sizeof(double));
      if (icov) std::memcpy(icov + V * 9, L.icov, 9 * sizeof(double));
    }
    V++;
  }
  *n_voxels = V;
  if (min_b) for (int d = 0; d < 3; d++) min_b[d] = M.h_geom.empty ? 0 : M.h_geom.min_b[d];
  if (div_b) for (int d = 0; d < 3; d++) div_b[d] = M.h_geom.empty ? 0 : M.h_geom.div_b[d];
  return B2R_OK;
}

// ---- scalar pose algebra, float32 exactly as oracle/ndt.cpp (host libm on both sides)
struct NdtScalars {
  double d1, d2;
  float jang[8][3], hang[15][3];
  double jang_d[8][3], hang_d[15][3];
};

inline void ndt_gauss(const b2r_config& c, NdtScalars& K) {
  double gauss_c1 = 10 * (1 - c.ndt_outlier_ratio);
  double gauss_c2 = c.ndt_outlier_ratio / std::pow(c.ndt_resolution, 3);
  double gauss_d3 = -std::log(gauss_c2);
  K.d1 = -std::log(gauss_c1 + gauss_c2) - gauss_d3;
  K.d2 = -2 * std::log((-std::log(gauss_c1 * std::exp(-0.5) + gauss_c2) - gauss_d3) / K.d1);
}

inline void ndt_angle_derivs(const double* p, NdtScalars& K) {
  double cx, cy, cz, sx, sy, sz;
  if (std::fabs(p[3]) < 10e-5) { cx = 1.0; sx = 0.0; } else { cx = std::cos(p[3]); sx = std::sin(p[3]); }
  if (std::fabs(p[4]) < 10e-5) { cy = 1.0; sy = 0.0; } else { cy = std::cos(p[4]); sy = std::sin(p[4]); }
  if (std::fabs(p[5]) < 10e-5) { cz = 1.0; sz = 0.0; } else { cz = std::cos(p[5]); sz = std::sin(p[5]); }
  // Magnusson 2009 eq. 6.19 / 6.21 (SURVEY A.2)
  const double J[8][3] = {
      {(-sx * sz + cx * sy * cz), (-sx * cz - cx * sy * sz), (-cx * cy)},
      {(cx * sz + sx * sy * cz), (cx * cz - sx * sy * sz), (-sx * cy)},
      {(-sy * cz), sy * sz, cy},
      {sx * cy * cz, (-sx * cy * sz), sx * sy},
      {(-cx * cy * cz), cx * cy * sz, (-cx * sy)},
      {(-cy * sz), (-cy * cz), 0},
      {(cx * cz - sx * sy * sz), (-cx * sz - sx * sy * cz), 0},
      {(sx * cz + cx * sy * sz), (cx * sy * cz - sx * sz), 0}};
  const double Hh[15][3] = {
      {(-cx * sz - sx * sy * cz), (-cx * cz + sx * sy * sz), sx * cy},
      {(-sx * sz + cx * sy * cz), (-cx * sy * sz - sx * cz), (-cx * cy)},
      {(cx * cy * cz), (-cx * cy * sz), (cx * sy)},
      {(sx * cy * cz), (-sx * cy * sz), (sx * sy)},
      {(-sx * cz - cx * sy * sz), (sx * sz - cx * sy * cz), 0},
      {(cx * cz - sx * sy * sz), (-sx * sy * cz - cx * sz), 0},
      {(-cy * cz), (cy * sz), (sy)},
      {(-sx * sy * cz), (sx * sy * sz), (sx * cy)},
      {(cx * sy * cz), (-cx * sy * sz), (-cx * cy)},
      {(sy * sz), (sy * cz), 0},
      {(-sx * cy * sz), (-sx * cy * cz), 0},
      {(cx * cy * sz), (cx * cy * cz), 0},
      {(-cy * cz), (cy * sz), 0},
      {(-cx * sz - sx * sy * cz), (-cx * cz + sx * sy * sz), 0},
      {(-sx * sz + cx * sy * cz), (-cx * sy * sz - sx * cz), 0}};
  for (int r = 0; r < 8; r++)
    for (int c = 0; c < 3; c++) { K.jang_d[r][c] = J[r][c]; K.jang[r][c] = (float)J[r][c]; }
  for (int r = 0; r < 15; r++)
    for (int c = 0; c < 3; c++) { K.hang_d[r][c] = Hh[r][c]; K.hang[r][c] = (float)Hh[r][c]; }
}

// Translation * AngleAxis(rx, X) * AngleAxis(ry, Y) * AngleAxis(rz, Z) in float32 (Eigen composition order, no FMA:
// this translation unit is compiled for x86-64 without -mfma, host products are separate mul/add)
inline void ndt_pose_to_matrix(const double* p, float* T) {
  float ang[3] = {(float)p[3], (float)p[4], (float)p[5]};
  float R[3][9];
  for (int a = 0; a < 3; a++) {
    float s = (float)std::sin((double)ang[a]);
    float c = (float)std::cos((double)ang[a]);
    float omc = 1.0f - c;
    volatile float diag_axis_v = omc + c;
    float diag_axis = diag_axis_v;
    float m[9] = {c, 0, 0, 0, c, 0, 0, 0, c};
    if (a == 0) { m[0] = diag_axis; m[5] = 0.f - s; m[7] = 0.f + s; }
    if (a == 1) { m[4] = diag_axis; m[2] = 0.f + s; m[6] = 0.f - s; }
    if (a == 2) { m[8] = diag_axis; m[1] = 0.f - s; m[3] = 0.f + s; }
    std::memcpy(R[a], m, sizeof(m));
  }
  auto mm = [](const float* A, const float* B, float* O) {
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) {
        volatile float u = A[r * 3 + 0] * B[0 * 3 + c];
        volatile float v = A[r * 3 + 1] * B[1 * 3 + c];
        volatile float w = u + v;
        volatile float v2 = A[r * 3 + 2] * B[2 * 3 + c];
        O[r * 3 + c] = w + v2;
      }
  };
  float xy[9], xyz[9];
  mm(R[0], R[1], xy);
  mm(xy, R[2], xyz);
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[r * 4 + c] = xyz[r * 3 + c];
    T[r * 4 + 3] = (float)p[r];
  }
  T[12] = T[13] = T[14] = 0.f;
  T[15] = 1.f;
}

// Eigen 3.3 Matrix3f::eulerAngles(0,1,2), float32, first angle in [0, pi] (what the reference's distro Eigen does)
inline void ndt_euler_xyz(const float* T, float* out) {
  auto m = [&](int r, int c) { return T[r * 4 + c]; };
  float res0 = std::atan2(m(1, 2), m(2, 2));
  volatile float a2 = m(0, 0) * m(0, 0);
  volatile float b2 = m(0, 1) * m(0, 1);
  float c2 = std::sqrt(a2 + b2);
  float res1;
  if (res0 > 0.f) {
    res0 -= (float)M_PI;
    res1 = std::atan2(-m(0, 2), -c2);
  } else {
    res1 = std::atan2(-m(0, 2), c2);
  }
  float s1 = std::sin(res0), c1 = std::cos(res0);
  volatile float n1 = s1 * m(2, 0);
  volatile float n2 = c1 * m(1, 0);
  volatile float d1 = c1 * m(1, 1);
  volatile float d2 = s1 * m(2, 1);
  float res2 = std::atan2(n1 - n2, d1 - d2);
  out[0] = -res0; out[1] = -res1; out[2] = -res2;
}

// JacobiSVD(H).solve(rhs) for symmetric H: pseudo-inverse via a 6x6 cyclic Jacobi eigen-decomposition
inline void ndt_svd6_solve(const double* H, const double* rhs, double* x) {
  double A[36], V[36], w[6];
  std::memcpy(A, H, sizeof(A));
  bool nan_in = false;
  for (int i = 0; i < 36; i++) nan_in |= (H[i] != H[i]);
  for (int i = 0; i < 6; i++) nan_in |= (rhs[i] != rhs[i]);
  if (nan_in) { for (int i = 0; i < 6; i++) x[i] = NAN; return; }
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 6; j++) V[i * 6 + j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 64; sweep++) {
    double off = 0;
    for (int p = 0; p < 6; p++)
      for (int q = p + 1; q < 6; q++) off += A[p * 6 + q] * A[p * 6 + q];
    if (off == 0.0) break;
    {  // converged to working precision (same rule as the oracle's 6x6 solve): off-diagonal mass below 1e-34 of the diagonal's
      double dg = 0.0;
      for (int p = 0; p < 6; p++) dg += A[p * 6 + p] * A[p * 6 + p];
      if (off <= 1e-34 * dg) break;
    }
    for (int p = 0; p < 6; p++)
      for (int q = p + 1; q < 6; q++) {
        double apq = A[p * 6 + q];
        if (apq == 0.0) continue;
        double app = A[p * 6 + p], aqq = A[q * 6 + q];
        double theta = (aqq - app) / (2.0 * apq);
        double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 6; k++) { double akp = A[k * 6 + p], akq = A[k * 6 + q]; A[k * 6 + p] = c * akp - s * akq; A[k * 6 + q] = s * akp + c * akq; }
        for (int k = 0; k < 6; k++) { double apk = A[p * 6 + k], aqk = A[q * 6 + k]; A[p * 6 + k] = c * apk - s * aqk; A[q * 6 + k] = s * apk + c * aqk; }
        for (int k = 0; k < 6; k++) { double vkp = V[k * 6 + p], vkq = V[k * 6 + q]; V[k * 6 + p] = c * vkp - s * vkq; V[k * 6 + q] = s * vkp + c * vkq; }
      }
  }
  for (int i = 0; i < 6; i++) w[i] = A[i * 6 + i];
  for (int i = 0; i < 6; i++) {
    int m = i;
    for (int j = i + 1; j < 6; j++) if (w[j] < w[m]) m = j;
    if (m != i) { std::swap(w[i], w[m]); for (int k = 0; k < 6; k++) std::swap(V[k * 6 + i], V[k * 6 + m]); }
  }
  double smax = 0;
  for (int i = 0; i < 6; i++) smax = std::max(smax, std::fabs(w[i]));
  double thr = std::max(smax * 6.0 * 2.220446049250313e-16, 2.2250738585072014e-308);
  for (int i = 0; i < 6; i++) x[i] = 0.0;
  for (int k = 0; k < 6; k++) {
    if (!(std::fabs(w[k]) > thr)) continue;
    double dot = 0;
    for (int i = 0; i < 6; i++) dot += V[i * 6 + k] * rhs[i];
    dot /= w[k];
    for (int i = 0; i < 6; i++) x[i] += V[i * 6 + k] * dot;
  }
}

struct NdtPass {
  double score, g[6], H[36];
  unsigned long long pairs;
};

// blocks of k_ndt_derivatives the device holds at once (occupancy x SM count), asked once per process
inline unsigned ndt_resident_blocks(bool hess) {
  static unsigned cached[2] = {0, 0};
  unsigned& c = cached[hess ? 1 : 0];
  if (c == 0) {
    int dev = 0, sms = 132, per = 4;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (hess) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_ndt_derivatives<true>, kNdtThreads, 0);
    else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_ndt_derivatives<false>, kNdtThreads, 0);
    if (const char* e = getenv("B2R_NDT_WAVES")) { const double w = atof(e); if (w > 0) per = std::max(1, (int)(per * w)); }
    c = (unsigned)std::max(1, sms * std::max(per, 1));
  }
  return c;
}

inline int ndt_run_pass(const b2r_config& cfg, Cloud& src, Cloud& tgt, NdtWork& W, cudaStream_t st, const NdtScalars& K, const float* Tf_row,
                        bool compute_hessian, bool hessian_only, NdtPass* out) {
  NdtVoxelMap& M = *tgt.ndt;
  NdtArgs A;
  A.src = src.sorted.p; A.n_sorted = src.nsup * 1024;
  A.geom = M.geom; A.table = M.table.p; A.mask = M.mask; A.cells = M.cells.p; A.vox = M.vox.p;
  for (int i = 0; i < 12; i++) A.Tf[i] = Tf_row[i];
  std::memcpy(A.jang, K.jang, sizeof(A.jang)); std::memcpy(A.hang, K.hang, sizeof(A.hang));
  std::memcpy(A.jang_d, K.jang_d, sizeof(A.jang_d)); std::memcpy(A.hang_d, K.hang_d, sizeof(A.hang_d));
  A.d1 = K.d1; A.d2 = K.d2;
  A.ncell_search = (cfg.ndt_search_method == 1) ? 1 : 7;
  A.compute_hessian = compute_hessian ? 1 : 0;
  const unsigned nb = (unsigned)((size_t)src.nsup * 1024 / kNdtThreads);  // 128-point chunks of the source
  B2R_CUDA(W.partials.reserve((size_t)(nb + 1) * kNdtAcc));  // derivative pass: [chunks][kNdtAcc]; Hessian pass: [blocks][36]
  const unsigned ngroups = (nb + 31) / 32;
  B2R_CUDA(W.grows.reserve((size_t)ngroups * kNdtAcc));
  if (ngroups > W.gcount.cap) {
    B2R_CUDA(W.gcount.reserve(ngroups));
    B2R_CUDA(cudaMemsetAsync(W.gcount.p, 0, W.gcount.cap * sizeof(unsigned int), st));  // every launch leaves the counters at zero
  }
  A.partials = W.partials.p; A.grows = W.grows.p; A.gcount = W.gcount.p; A.queue = W.d_queue; A.qbase = 0;
  A.out = W.h_out_dev; A.counter = W.d_counter; A.pairs = W.d_pairs;
  A.flag = W.h_flag_dev; A.seq = ++W.seq;
  if (hessian_only) {
    { TEL_BEGIN(W.tel, st);
      k_ndt_hessian<<<nb, kNdtThreads, 0, st>>>(A);
      TEL_END(W.tel, KC_NDT_HESS, 1, st); }
    if (W.tel) W.tel->d2h += 36 * sizeof(double);
    B2R_CUDA(cudaGetLastError());
    int rc = wait_host_result(W.h_flag, A.seq, W.h_out, 36, false, st);
    if (rc) return rc;
    std::memcpy(out->H, W.h_out, 36 * sizeof(double));
    return B2R_OK;
  }
  { TEL_BEGIN(W.tel, st);  // W.d_pairs is zero here: allocated zeroed, and the last block of every pass resets it after reading it
    const unsigned ng = std::min(nb, ndt_resident_blocks(compute_hessian));
    A.qbase = W.qnext;
    W.qnext += (unsigned long long)nb + ng;  // every block draws tickets until its first one past the last chunk: nb + ng draws per launch
    if (compute_hessian) k_ndt_derivatives<true><<<ng, kNdtThreads, 0, st>>>(A);
    else k_ndt_derivatives<false><<<ng, kNdtThreads, 0, st>>>(A);
    TEL_END(W.tel, KC_NDT_DERIV, 1, st);
    if (cudaPeekAtLastError() != cudaSuccess) W.qnext = A.qbase;  // nothing ran: no ticket was drawn
  }
  if (W.tel) W.tel->d2h += kNdtAcc * sizeof(double) + 8;
  B2R_CUDA(cudaGetLastError());
  int rc = wait_host_result(W.h_flag, A.seq, W.h_out, kNdtAcc, true, st);
  if (rc) return rc;
  out->score = W.h_out[0];
  std::memcpy(out->g, W.h_out + 1, 6 * sizeof(double));
  if (compute_hessian) {
    int k = 7;
    for (int r = 0; r < 6; r++)
      for (int c = r; c < 6; c++) out->H[r * 6 + c] = W.h_out[k++];     // first sweep: ii <= jj
    for (int r = 1; r < 6; r++)
      for (int c = 0; c < r; c++) out->H[r * 6 + c] = W.h_out[k++];     // second sweep: ii > jj
  }
  std::memcpy(&out->pairs, W.h_out + kNdtAcc, sizeof(unsigned long long));
  return B2R_OK;
}

inline int ndt_derivatives_at(const b2r_config& cfg, Cloud& src, Cloud& tgt, NdtWork& W, cudaStream_t st, const double* p, double* score,
                              double* g, double* H, uint64_t* n_pairs) {
  int rc = ndt_sync_geom(*tgt.ndt, W, st);
  if (rc) return rc;
  NdtScalars K;
  ndt_gauss(cfg, K);
  ndt_angle_derivs(p, K);
  float Tf[16];
  ndt_pose_to_matrix(p, Tf);
  NdtPass P;
  rc = ndt_run_pass(cfg, src, tgt, W, st, K, Tf, true, false, &P);
  if (rc) return rc;
  *score = P.score;
  std::memcpy(g, P.g, sizeof(P.g));
  std::memcpy(H, P.H, sizeof(P.H));
  if (n_pairs) *n_pairs = P.pairs;
  return B2R_OK;
}

// More-Thuente helpers (PCL ndt.hpp as copied by ndt_omp; SURVEY A.2)
inline double mt_psi(double a, double f_a, double f_0, double g_0, double mu) { return f_a - f_0 - mu * g_0 * a; }
inline double mt_dpsi(double g_a, double g_0, double mu) { return g_a - mu * g_0; }
inline double mt_trial(double a_l, double f_l, double g_l, double a_u, double f_u, double g_u, double a_t, double f_t, double g_t) {
  if (f_t > f_l) {
    double z = 3 * (f_t - f_l) / (a_t - a_l) - g_t - g_l;
    double w = std::sqrt(z * z - g_t * g_l);
    double a_c = a_l + (a_t - a_l) * (w - g_l - z) / (g_t - g_l + 2 * w);
    double a_q = a_l - 0.5 * (a_l - a_t) * g_l / (g_l - (f_l - f_t) / (a_l - a_t));
    return (std::fabs(a_c - a_l) < std::fabs(a_q - a_l)) ? a_c : 0.5 * (a_q + a_c);
  } else if (g_t * g_l < 0) {
    double z = 3 * (f_t - f_l) / (a_t - a_l) - g_t - g_l;
    double w = std::sqrt(z * z - g_t * g_l);
    double a_c = a_l + (a_t - a_l) * (w - g_l - z) / (g_t - g_l + 2 * w);
    double a_s = a_l - (a_l - a_t) / (g_l - g_t) * g_l;
    return (std::fabs(a_c - a_t) >= std::fabs(a_s - a_t)) ? a_c : a_s;
  } else if (std::fabs(g_t) <= std::fabs(g_l)) {
    double z = 3 * (f_t - f_l) / (a_t - a_l) - g_t - g_l;
    double w = std::sqrt(z * z - g_t * g_l);
    double a_c = a_l + (a_t - a_l) * (w - g_l - z) / (g_t - g_l + 2 * w);
    double a_s = a_l - (a_l - a_t) / (g_l - g_t) * g_l;
    double a_t_next = (std::fabs(a_c - a_t) < std::fabs(a_s - a_t)) ? a_c : a_s;
    return (a_t > a_l) ? std::min(a_t + 0.66 * (a_u - a_t), a_t_next) : std::max(a_t + 0.66 * (a_u - a_t), a_t_next);
  }
  double z = 3 * (f_t - f_u) / (a_t - a_u) - g_t - g_u;
  double w = std::sqrt(z * z - g_t * g_u);
  return a_u + (a_t - a_u) * (w - g_u - z) / (g_t - g_u + 2 * w);
}
inline bool mt_update(double& a_l, double& f_l, double& g_l, double& a_u, double& f_u, double& g_u, double a_t, double f_t, double g_t) {
  if (f_t > f_l) { a_u = a_t; f_u = f_t; g_u = g_t; return false; }
  if (g_t * (a_l - a_t) > 0) { a_l = a_t; f_l = f_t; g_l = g_t; return false; }
  if (g_t * (a_l - a_t) < 0) { a_u = a_l; f_u = f_l; g_u = g_l; a_l = a_t; f_l = f_t; g_l = g_t; return false; }
  return true;
}

// pclomp::NormalDistributionsTransform::computeTransformation (A.2).  guess: column-major float (ABI); Tfinal: row-major.
inline int ndt_align(const b2r_config& cfg, Cloud& src, Cloud& tgt, NdtWork& W, cudaStream_t st, const float* guess_col, float* Tfinal,
                     bool* converged_out, int* iters_out) {
  for (int i = 0; i < 16; i++) Tfinal[i] = (i % 5 == 0) ? 1.f : 0.f;
  *converged_out = false;
  *iters_out = 0;
  if (src.n == 0 || tgt.n == 0) return B2R_OK;  // initCompute fails silently
  int rc = ndt_ensure_map(cfg, tgt, W, st);
  if (rc) return rc;
  rc = ndt_sync_geom(*tgt.ndt, W, st);
  if (rc) return rc;
  if (tgt.ndt->h_geom.empty) return B2R_OK;
  NdtScalars K;
  ndt_gauss(cfg, K);
  float guess[16];
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) guess[r * 4 + c] = guess_col[c * 4 + r];
  bool is_identity = true;
  for (int i = 0; i < 16; i++) is_identity &= (guess[i] == ((i % 5 == 0) ? 1.f : 0.f));
  if (!is_identity) std::memcpy(Tfinal, guess, sizeof(guess));
  double p[6];
  {
    float e[3];
    ndt_euler_xyz(Tfinal, e);
    p[0] = Tfinal[3]; p[1] = Tfinal[7]; p[2] = Tfinal[11];
    p[3] = e[0]; p[4] = e[1]; p[5] = e[2];
  }
  ndt_angle_derivs(p, K);
  NdtPass P;
  rc = ndt_run_pass(cfg, src, tgt, W, st, K, Tfinal, true, false, &P);  // first pass: cloud transformed by the guess matrix itself
  if (rc) return rc;
  double score = P.score, g[6], H[36];
  std::memcpy(g, P.g, sizeof(g));
  std::memcpy(H, P.H, sizeof(H));
  int nr_iterations = 0;
  bool converged = false;
  const int max_it = cfg.max_iterations;
  while (!converged) {
    double ng[6], dp[6];
    for (int i = 0; i < 6; i++) ng[i] = -g[i];
    ndt_svd6_solve(H, ng, dp);
    double nrm = 0;
    for (int i = 0; i < 6; i++) nrm += dp[i] * dp[i];
    nrm = std::sqrt(nrm);
    if (nrm == 0 || nrm != nrm) { converged = (nrm == nrm); break; }
    for (int i = 0; i < 6; i++) dp[i] /= nrm;
    const double step_max = cfg.ndt_step_size, step_min = cfg.transformation_epsilon / 2;
    const double phi_0 = -score;
    double d_phi_0 = 0;
    for (int i = 0; i < 6; i++) d_phi_0 += g[i] * dp[i];
    d_phi_0 = -d_phi_0;
    double a_t = 0;
    bool skip = false;
    if (d_phi_0 >= 0) {
      if (d_phi_0 == 0) { skip = true; a_t = 0; }
      else { d_phi_0 *= -1; for (int i = 0; i < 6; i++) dp[i] *= -1; }
    }
    if (!skip) {
      const double mu = 1.e-4, nu = 0.9;
      double a_l = 0, a_u = 0;
      double f_l = mt_psi(a_l, phi_0, phi_0, d_phi_0, mu), g_l = mt_dpsi(d_phi_0, d_phi_0, mu);
      double f_u = mt_psi(a_u, phi_0, phi_0, d_phi_0, mu), g_u = mt_dpsi(d_phi_0, d_phi_0, mu);
      bool interval_converged = cfg.ndt_mt_interval_flag ? ((step_max - step_min) < 0) : ((step_max - step_min) > 0);
      bool open_interval = true;
      int step_iterations = 0;
      a_t = nrm;
      a_t = std::min(a_t, step_max);
      a_t = std::max(a_t, step_min);
      double x_t[6];
      for (int i = 0; i < 6; i++) x_t[i] = p[i] + dp[i] * a_t;
      ndt_pose_to_matrix(x_t, Tfinal);
      ndt_angle_derivs(x_t, K);
      rc = ndt_run_pass(cfg, src, tgt, W, st, K, Tfinal, true, false, &P);
      if (rc) return rc;
      score = P.score; std::memcpy(g, P.g, sizeof(g)); std::memcpy(H, P.H, sizeof(H));
      double phi_t = -score, d_phi_t = 0;
      for (int i = 0; i < 6; i++) d_phi_t += g[i] * dp[i];
      d_phi_t = -d_phi_t;
      double psi_t = mt_psi(a_t, phi_t, phi_0, d_phi_0, mu), d_psi_t = mt_dpsi(d_phi_t, d_phi_0, mu);
      while (!interval_converged && step_iterations < 10 && !(psi_t <= 0 && d_phi_t <= -nu * d_phi_0)) {
        if (open_interval) a_t = mt_trial(a_l, f_l, g_l, a_u, f_u, g_u, a_t, psi_t, d_psi_t);
        else a_t = mt_trial(a_l, f_l, g_l, a_u, f_u, g_u, a_t, phi_t, d_phi_t);
        a_t = std::min(a_t, step_max);
        a_t = std::max(a_t, step_min);
        for (int i = 0; i < 6; i++) x_t[i] = p[i] + dp[i] * a_t;
        ndt_pose_to_matrix(x_t, Tfinal);
        ndt_angle_derivs(x_t, K);
        rc = ndt_run_pass(cfg, src, tgt, W, st, K, Tfinal, false, false, &P);
        if (rc) return rc;
        score = P.score; std::memcpy(g, P.g, sizeof(g));
        phi_t = -score;
        d_phi_t = 0;
        for (int i = 0; i < 6; i++) d_phi_t += g[i] * dp[i];
        d_phi_t = -d_phi_t;
        psi_t = mt_psi(a_t, phi_t, phi_0, d_phi_0, mu);
        d_psi_t = mt_dpsi(d_phi_t, d_phi_0, mu);
        if (open_interval && (psi_t <= 0 && d_psi_t >= 0)) {
          open_interval = false;
          f_l = f_l + phi_0 - mu * d_phi_0 * a_l;
          g_l = g_l + mu * d_phi_0;
          f_u = f_u + phi_0 - mu * d_phi_0 * a_u;
          g_u = g_u + mu * d_phi_0;
        }
        if (open_interval) interval_converged = mt_update(a_l, f_l, g_l, a_u, f_u, g_u, a_t, psi_t, d_psi_t);
        else interval_converged = mt_update(a_l, f_l, g_l, a_u, f_u, g_u, a_t, phi_t, d_phi_t);
        step_iterations++;
      }
      if (step_iterations) {
        rc = ndt_run_pass(cfg, src, tgt, W, st, K, Tfinal, true, true, &P);
        if (rc) return rc;
        std::memcpy(H, P.H, sizeof(H));
      }
    }
    const double delta_p_norm = a_t;
    for (int i = 0; i < 6; i++) { dp[i] *= delta_p_norm; p[i] += dp[i]; }
    if (cfg.ndt_fixed_iterations > 0) {
      if (nr_iterations + 1 >= cfg.ndt_fixed_iterations) converged = true;
    } else if (nr_iterations > max_it || (nr_iterations && (std::fabs(delta_p_norm) < cfg.transformation_epsilon))) {
      converged = true;
    }
    nr_iterations++;
  }
  *converged_out = converged;
  *iters_out = nr_iterations;
  return B2R_OK;
}

}  // namespace b2r
