// voxelgrid.cuh — voxel-grid downsample, the companion kernel of the prefilter.
//
// Re-creates pcl::VoxelGrid<pcl::PointXYZI>::filter with setLeafSize(r,r,r), downsample_all_data = true (SURVEY.md A.5), as
// configured at /root/reference/apps/prefiltering_nodelet.cpp:54-58 and called at :138-149 (and, optionally, at
// apps/scan_matching_odometry_nodelet.cpp:86-90,147-157):
//   k_vg_params    <- getMinMax3D + min_b/div_b/divb_mul + the int32 overflow guard ("Leaf size is too small ...")
//   k_vg_keys      <- idx = (floor(p * inv_leaf) - min_b) . divb_mul          (float32 multiply, int32 index)
//   radix sort     <- std::sort of (idx, point index): stable LSD radix sort => ascending point index inside a voxel
//   k_vg_centroid  <- one thread per voxel, sequential float32 sums of x,y,z,intensity in that order, / count
// Output order = ascending voxel key (as PCL).  Keys, counts and ordering are bit-exact against the oracle; centroids too,
// because the within-voxel summation order is pinned (PCL leaves it implementation-defined).
// Clouds of up to 131 072 points (every scan of the BASELINE configs) take ONE kernel on a thread-block cluster
// (k_voxelgrid_cluster): bounding box, keys, the radix sort through distributed shared memory of bvh_build.cuh, head scan and
// centroids without leaving the cluster, output left in device memory.  Larger inputs fall back to the kernel chain below, whose
// sort and scan are the CUDA toolkit's cub::DeviceRadixSort / DeviceScan.
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <climits>
#include <vector>
#include "engine.cuh"
#include "bvh_build.cuh"

namespace b2r {

struct VgGeom {
  float inv_leaf;
  int min_b[3], div_b[3];
  int mul1, mul2;
  int overflow;  // dx*dy*dz > INT_MAX
  int empty;
};

struct VoxelWork {
  DevBuf<float> in, out;
  DevBuf<int> keys_a, keys_b, vals_a, vals_b, flags, slots, okeys, ocounts;
  DevBuf<int> buckets;  // approx_voxelgrid.cuh: per hash slot, occupied flag, then the output slot of its last run
  DevBuf<char> tmp;
  DevBuf<int> mm;            // 8 ints
  DevBuf<VgGeom> geom;
  PinnedBuf<VgGeom> h_geom;
  MappedBuf<int> h_total;    // [0] voxel count, [1] overflow flag
  Telemetry* tel = nullptr;
  bool wide_clusters = false;  // 16-CTA clusters may be launched on this device (set by the handle: cluster16_allowed())
};
static_assert(!std::is_copy_constructible<VoxelWork>::value, "a VoxelWork owns its buffers");

__global__ void k_vg_params(const int* mm, VgGeom* g, int n, float leaf) {
  VgGeom G;
  G.inv_leaf = 1.0f / leaf;
  G.overflow = 0;
  G.empty = 0;
  G.mul1 = G.mul2 = 1;
  for (int d = 0; d < 3; d++) { G.min_b[d] = 0; G.div_b[d] = 1; }
  if (n <= 0 || mm[0] == 0x7fffffff) { G.empty = 1; *g = G; return; }
  long long vol = 1;
  bool huge = false;
  for (int d = 0; d < 3; d++) {
    float mn = ord2f(mm[d]), mx = ord2f(mm[3 + d]);
    float ext = fmul(fsub(mx, mn), G.inv_leaf);
    if (!(ext < 4.0e9f)) { huge = true; continue; }
    long long dd = (long long)ext + 1;  // static_cast<int64>((max - min) * inv_leaf) + 1
    vol *= dd;
    if (vol > (long long)INT_MAX) huge = true;
  }
  if (huge) { G.overflow = 1; *g = G; return; }
  for (int d = 0; d < 3; d++) {
    float mn = ord2f(mm[d]), mx = ord2f(mm[3 + d]);
    G.min_b[d] = (int)floorf(fmul(mn, G.inv_leaf));
    int max_b = (int)floorf(fmul(mx, G.inv_leaf));
    G.div_b[d] = max_b - G.min_b[d] + 1;
  }
  G.mul1 = G.div_b[0];
  G.mul2 = G.div_b[0] * G.div_b[1];
  *g = G;
}

__global__ void k_vg_keys(const float* __restrict__ raw, int stride_f, int n, const VgGeom* __restrict__ gp, int* keys, int* vals) {
  const VgGeom G = *gp;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = raw + (size_t)i * stride_f;
  const float x = p[0], y = p[1], z = p[2];
  int key = INT_MAX;  // non-finite points sort last and are dropped
  if (finite3(x, y, z) && !G.overflow) {
    int i0 = (int)fsub(floorf(fmul(x, G.inv_leaf)), (float)G.min_b[0]);
    int i1 = (int)fsub(floorf(fmul(y, G.inv_leaf)), (float)G.min_b[1]);
    int i2 = (int)fsub(floorf(fmul(z, G.inv_leaf)), (float)G.min_b[2]);
    key = i0 + i1 * G.mul1 + i2 * G.mul2;
  }
  keys[i] = key;
  vals[i] = i;
}

__global__ void k_vg_heads(const int* __restrict__ keys, int n, int* flags) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int k = keys[s];
  flags[s] = (k != INT_MAX && (s == 0 || keys[s - 1] != k)) ? 1 : 0;
}

__global__ void k_vg_centroid(const float* __restrict__ raw, int stride_f, int n, const int* __restrict__ keys, const int* __restrict__ vals,
                              const int* __restrict__ flags, const int* __restrict__ slots, float* out, int out_stride_f, int* okeys,
                              int* ocounts, int* total) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  if (s == n - 1) *total = slots[s] + flags[s];
  if (!flags[s]) return;
  const int k = keys[s];
  const bool has_i = stride_f >= 5;
  float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
  int e = s;
  while (e < n && keys[e] == k) {
    const float* p = raw + (size_t)vals[e] * stride_f;
    sx = fadd(sx, p[0]); sy = fadd(sy, p[1]); sz = fadd(sz, p[2]);
    si = fadd(si, has_i ? p[4] : 0.f);
    e++;
  }
  const float cnt = (float)(e - s);
  const int slot = slots[s];
  float* o = out + (size_t)slot * out_stride_f;
  o[0] = __fdiv_rn(sx, cnt); o[1] = __fdiv_rn(sy, cnt); o[2] = __fdiv_rn(sz, cnt);
  if (out_stride_f >= 4) o[3] = 1.0f;
  if (out_stride_f >= 5) o[4] = __fdiv_rn(si, cnt);
  for (int j = 5; j < out_stride_f; j++) o[j] = 0.f;
  okeys[slot] = k;
  ocounts[slot] = e - s;
}

// ------------------------------------------------------------------------------------------------ one-kernel cluster path
struct VgArgs {
  const float* in;     // device records
  int stride_f;
  int n;
  float leaf;
  float* out;          // device, same record layout as the input
  int* okeys;          // device (may be null)
  int* ocounts;        // device (may be null)
  int* total;          // device: [0] voxel count, [1] overflow flag
  volatile int* h_total;  // host-mapped twin of `total` (or null): the count reaches the host without a copy
};

template <int CL, int PER>
__global__ void __launch_bounds__(kBuildThreads, 1) k_voxelgrid_cluster(const __grid_constant__ VgArgs A) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int kCap = BuildGeom<PER>::kCap;
  constexpr int kShift = BuildGeom<PER>::kShift;
  const ClusterSmem S = cluster_smem<PER>(smem_raw);
  uint2* buf = S.buf;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = A.n;
  const int g0 = rank * kCap;
  int mm[6];
  cluster_bbox<CL, PER>(cluster, S, A.in, A.stride_f, n, g0, mm);
  // ---- geometry (k_vg_params), computed redundantly by every thread from the cluster-wide bounding box
  const float inv_leaf = 1.0f / A.leaf;
  int min_b[3] = {0, 0, 0}, div_b[3] = {1, 1, 1};
  bool overflow = false, empty = (n <= 0 || mm[0] == 0x7fffffff);
  if (!empty) {
    long long vol = 1;
#pragma unroll
    for (int d = 0; d < 3; d++) {
      const float mn = ord2f(mm[d]), mx = ord2f(mm[3 + d]);
      const float ext = fmul(fsub(mx, mn), inv_leaf);
      if (!(ext < 4.0e9f)) { overflow = true; continue; }
      const long long dd = (long long)ext + 1;  // static_cast<int64>((max - min) * inv_leaf) + 1
      vol *= dd;
      if (vol > (long long)INT_MAX) overflow = true;
    }
    if (!overflow) {
#pragma unroll
      for (int d = 0; d < 3; d++) {
        min_b[d] = (int)floorf(fmul(ord2f(mm[d]), inv_leaf));
        div_b[d] = (int)floorf(fmul(ord2f(mm[3 + d]), inv_leaf)) - min_b[d] + 1;
      }
    }
  }
  if (overflow || empty) {  // uniform over the whole cluster: nobody has touched a peer's memory since the bbox barrier
    if (rank == 0 && tid == 0) {
      A.total[0] = 0; A.total[1] = overflow ? 1 : 0;
      if (A.h_total) { A.h_total[1] = overflow ? 1 : 0; A.h_total[0] = 0; }
    }
    cluster.sync();
    return;
  }
  const int mul1 = div_b[0], mul2 = div_b[0] * div_b[1];
  // ---- keys (k_vg_keys): int32 voxel index; non-finite points 0x7fffffff, padding 0xffffffff (both sort behind every voxel)
#pragma unroll 4
  for (int b = 0; b < PER; b++) {
    const int e = warp * (32 * PER) + b * 32 + lane;
    const int i = g0 + e;
    unsigned int key = 0xffffffffu;
    if (i < n) {
      const float* p = A.in + (size_t)i * A.stride_f;
      const float x = p[0], y = p[1], z = p[2];
      key = 0x7fffffffu;
      if (finite3(x, y, z)) {
        const int i0 = (int)fsub(floorf(fmul(x, inv_leaf)), (float)min_b[0]);
        const int i1 = (int)fsub(floorf(fmul(y, inv_leaf)), (float)min_b[1]);
        const int i2 = (int)fsub(floorf(fmul(z, inv_leaf)), (float)min_b[2]);
        key = (unsigned int)(i0 + i1 * mul1 + i2 * mul2);
      }
    }
    buf[e] = make_uint2(key, (unsigned int)i);
  }
  __syncthreads();
  cluster_radix_sort<CL, PER>(cluster, S, rank);  // ends with a cluster barrier: every slice is final and visible
  // ---- heads: thread t owns the PER consecutive positions t*PER .. t*PER+PER-1 of this CTA's slice
  const int e0 = tid * PER;
  unsigned int prev = 0xffffffffu;  // key before position e0 (none for the very first position of the cloud)
  if (e0 > 0) prev = buf[e0 - 1].x;
  else if (rank > 0) prev = cluster.map_shared_rank(buf, rank - 1)[kCap - 1].x;
  unsigned int headmask = 0;
  {
    unsigned int pk = prev;
    const bool first_of_cloud = (rank == 0 && e0 == 0);
#pragma unroll
    for (int j = 0; j < PER; j++) {
      const unsigned int k = buf[e0 + j].x;
      if (k < 0x7fffffffu && ((first_of_cloud && j == 0) || k != pk)) headmask |= 1u << j;
      pk = k;
    }
  }
  const int mine = __popc(headmask);
  // block exclusive scan of `mine`, then the cluster-wide offset of this CTA
  int* scr = S.base;  // [32] warp totals (the radix-sort scratch is free now)
  int inc = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) scr[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int w = scr[lane], winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += t; }
    scr[lane] = winc - w;
    if (lane == 31) S.cta_cnt[0] = winc;  // heads in this CTA's slice
  }
  cluster.sync();
  int slot = inc - mine + scr[warp];
  int total = 0;
  for (int c = 0; c < CL; c++) {
    const int v = cluster.map_shared_rank(S.cta_cnt, c)[0];
    total += v;
    if (c < rank) slot += v;
  }
  if (rank == 0 && tid == 0) {
    A.total[0] = total; A.total[1] = 0;
    if (A.h_total) { A.h_total[1] = 0; A.h_total[0] = total; }
  }
  // ---- centroids (k_vg_centroid): one thread per voxel, sequential float32 sums in ascending point index; a voxel's run may
  // continue into the next CTAs' slices (read through distributed shared memory)
  const bool has_i = A.stride_f >= 5;
  const int cap_all = CL * kCap;
  while (headmask) {
    const int j = __ffs(headmask) - 1;
    headmask &= headmask - 1;
    const unsigned int k = buf[e0 + j].x;
    float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
    int g = g0 + e0 + j, cnt = 0;
    for (;;) {
      const uint2 kv = (g >> kShift) == rank ? buf[g & (kCap - 1)] : cluster.map_shared_rank(buf, g >> kShift)[g & (kCap - 1)];
      if (kv.x != k) break;
      const float* p = A.in + (size_t)kv.y * A.stride_f;
      sx = fadd(sx, p[0]); sy = fadd(sy, p[1]); sz = fadd(sz, p[2]);
      si = fadd(si, has_i ? p[4] : 0.f);
      cnt++;
      if (++g >= cap_all) break;
    }
    const float fc = (float)cnt;
    float* o = A.out + (size_t)slot * A.stride_f;
    o[0] = __fdiv_rn(sx, fc); o[1] = __fdiv_rn(sy, fc); o[2] = __fdiv_rn(sz, fc);
    if (A.stride_f >= 4) o[3] = 1.0f;
    if (A.stride_f >= 5) o[4] = __fdiv_rn(si, fc);
    for (int q = 5; q < A.stride_f; q++) o[q] = 0.f;
    if (A.okeys) A.okeys[slot] = (int)k;
    if (A.ocounts) A.ocounts[slot] = cnt;
    slot++;
  }
  cluster.sync();  // no CTA may retire while a peer still walks a run that continues in its slice
}

template <int CL, int PER>
static cudaError_t launch_voxelgrid_cluster_t(const VgArgs& A, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_voxelgrid_cluster<CL, PER>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BuildGeom<PER>::kSmem);
    if (e != cudaSuccess) return e;
    if (CL > 8) {
      e = cudaFuncSetAttribute(k_voxelgrid_cluster<CL, PER>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
      if (e != cudaSuccess) return e;
    }
    attr_set = true;
  }
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3(CL); lc.blockDim = dim3(kBuildThreads); lc.dynamicSmemBytes = BuildGeom<PER>::kSmem; lc.stream = st;
  cudaLaunchAttribute la[1];
  la[0].id = cudaLaunchAttributeClusterDimension;
  la[0].val.clusterDim.x = CL; la[0].val.clusterDim.y = 1; la[0].val.clusterDim.z = 1;
  lc.attrs = la; lc.numAttrs = 1;
  return cudaLaunchKernelEx(&lc, k_voxelgrid_cluster<CL, PER>, A);
}
static cudaError_t launch_voxelgrid_cluster(int shape_index, const VgArgs& A, cudaStream_t st) {
  switch (shape_index) {  // build_shape_index(): (cluster size, pairs per thread)
    case 0: return launch_voxelgrid_cluster_t<1, 1>(A, st);
    case 1: return launch_voxelgrid_cluster_t<2, 1>(A, st);
    case 2: return launch_voxelgrid_cluster_t<4, 1>(A, st);
    case 3: return launch_voxelgrid_cluster_t<8, 1>(A, st);
    case 4: return launch_voxelgrid_cluster_t<8, 2>(A, st);
    case 5: return launch_voxelgrid_cluster_t<8, 4>(A, st);
    case 6: return launch_voxelgrid_cluster_t<8, 8>(A, st);
    case 7: return launch_voxelgrid_cluster_t<8, 16>(A, st);
    default: return launch_voxelgrid_cluster_t<16, 8>(A, st);
  }
}

// the small device / pinned words of the voxel-grid chains, allocated on first use
inline int vg_alloc_words(VoxelWork& W) {
  if (!W.mm.p) {
    B2R_CUDA(W.mm.alloc(8));
    B2R_CUDA(W.geom.alloc(1));
    B2R_CUDA(W.h_geom.alloc(1));
    B2R_CUDA(W.h_total.alloc(4));
  }
  return B2R_OK;
}

// device-resident voxel grid: d_in (device records) -> W.out / W.okeys / W.ocounts (device); *m = voxel count, *overflow = PCL's
// "leaf size too small" condition (output then undefined: the caller passes the input through)
inline int voxelgrid_device(VoxelWork& W, cudaStream_t st, const float* d_in, size_t n, size_t stride_bytes, float leaf, size_t* m, int* overflow) {
  const int sf = (int)(stride_bytes / 4);
  const int N = (int)n;
  int rc = vg_alloc_words(W);
  if (rc) return rc;
  B2R_CUDA(W.out.reserve(n * sf + 8));
  B2R_CUDA(W.okeys.reserve(n + 1)); B2R_CUDA(W.ocounts.reserve(n + 1));
  const BuildShape shape = build_shape_for(n, W.wide_clusters);
  static const bool cluster_ok = !getenv("B2R_CUB_SORT");
  if (shape.cl && cluster_ok) {
    VgArgs A;
    A.in = d_in; A.stride_f = sf; A.n = N; A.leaf = leaf; A.out = W.out.p; A.okeys = W.okeys.p; A.ocounts = W.ocounts.p;
    A.total = W.mm.p + 6; A.h_total = W.h_total.d;
    W.h_total.p[0] = -1;  // the kernel's count lands here (host-mapped); -1 = not yet
    TEL_BEGIN(W.tel, st);
    B2R_CUDA(launch_voxelgrid_cluster(build_shape_index(shape), A, st));
    TEL_END(W.tel, KC_VOXELGRID, 1, st);
    B2R_CUDA(cudaStreamSynchronize(st));
    *m = (size_t)(W.h_total.p[0] < 0 ? 0 : W.h_total.p[0]);
    *overflow = W.h_total.p[1];
    return B2R_OK;
  }
  // ---- inputs beyond 131 072 points: the kernel chain with the toolkit's radix sort / scan
  B2R_CUDA(W.keys_a.reserve(n)); B2R_CUDA(W.keys_b.reserve(n)); B2R_CUDA(W.vals_a.reserve(n)); B2R_CUDA(W.vals_b.reserve(n));
  B2R_CUDA(W.flags.reserve(n)); B2R_CUDA(W.slots.reserve(n));
  size_t tmp_sort = 0, tmp_scan = 0;
  B2R_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, W.keys_a.p, W.keys_b.p, W.vals_a.p, W.vals_b.p, N, 0, 32, st));
  B2R_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_scan, W.flags.p, W.slots.p, N, st));
  B2R_CUDA(W.tmp.reserve(std::max(tmp_sort, tmp_scan) + 256));
  const unsigned nb = (unsigned)((n + 255) / 256);
  TEL_BEGIN(W.tel, st);
  k_grid_reset<<<1, 32, 0, st>>>(W.mm.p);
  k_bbox<<<nb > 1184 ? 1184 : nb, 256, 0, st>>>(d_in, sf, N, W.mm.p);
  k_vg_params<<<1, 1, 0, st>>>(W.mm.p, W.geom.p, N, leaf);
  B2R_CUDA(cudaMemcpyAsync(W.h_geom.p, W.geom.p, sizeof(VgGeom), cudaMemcpyDeviceToHost, st));
  k_vg_keys<<<nb, 256, 0, st>>>(d_in, sf, N, W.geom.p, W.keys_a.p, W.vals_a.p);
  size_t tb = W.tmp.cap;
  B2R_CUDA(cub::DeviceRadixSort::SortPairs(W.tmp.p, tb, W.keys_a.p, W.keys_b.p, W.vals_a.p, W.vals_b.p, N, 0, 32, st));
  k_vg_heads<<<nb, 256, 0, st>>>(W.keys_b.p, N, W.flags.p);
  tb = W.tmp.cap;
  B2R_CUDA(cub::DeviceScan::ExclusiveSum(W.tmp.p, tb, W.flags.p, W.slots.p, N, st));
  k_vg_centroid<<<nb, 256, 0, st>>>(d_in, sf, N, W.keys_b.p, W.vals_b.p, W.flags.p, W.slots.p, W.out.p, sf, W.okeys.p, W.ocounts.p,
                                    (int*)(W.mm.p + 6));
  TEL_END(W.tel, KC_VOXELGRID, 14, st);
  B2R_CUDA(cudaGetLastError());
  B2R_CUDA(cudaMemcpyAsync(W.h_total.p, W.mm.p + 6, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaStreamSynchronize(st));
  *m = (size_t)W.h_total.p[0];
  *overflow = W.h_geom.p->overflow;
  return B2R_OK;
}

inline int voxelgrid_filter(VoxelWork& W, cudaStream_t st, const void* in, size_t n, size_t stride_bytes, float leaf, void* out,
                            size_t* n_out, int32_t* out_keys, int32_t* out_counts) {
  *n_out = 0;
  if (n == 0) return B2R_OK;
  if (n > (size_t)0x3fffffff) return fail(B2R_EINVAL, "too many points");
  const int sf = (int)(stride_bytes / 4);
  B2R_CUDA(W.in.reserve(n * sf));
  B2R_CUDA(cudaMemcpyAsync(W.in.p, in, n * stride_bytes, cudaMemcpyHostToDevice, st));
  if (W.tel) W.tel->h2d += n * stride_bytes;
  size_t m = 0;
  int overflow = 0;
  int rc = voxelgrid_device(W, st, W.in.p, n, stride_bytes, leaf, &m, &overflow);
  if (rc) return rc;
  if (overflow) {  // PCL: warn and pass the input through unchanged
    std::memcpy(out, in, n * stride_bytes);
    *n_out = n;
    if (out_keys) for (size_t i = 0; i < n; i++) out_keys[i] = -1;
    if (out_counts) for (size_t i = 0; i < n; i++) out_counts[i] = 1;
    return 1;
  }
  if (m) {
    B2R_CUDA(cudaMemcpyAsync(out, W.out.p, m * stride_bytes, cudaMemcpyDeviceToHost, st));
    if (out_keys) B2R_CUDA(cudaMemcpyAsync(out_keys, W.okeys.p, m * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (out_counts) B2R_CUDA(cudaMemcpyAsync(out_counts, W.ocounts.p, m * sizeof(int), cudaMemcpyDeviceToHost, st));
    B2R_CUDA(cudaStreamSynchronize(st));
  }
  if (W.tel) W.tel->d2h += m * stride_bytes;
  *n_out = m;
  return B2R_OK;
}

}  // namespace b2r
