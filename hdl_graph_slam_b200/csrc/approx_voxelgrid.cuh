// approx_voxelgrid.cuh — approximate voxel-grid downsample, the prefilter's APPROX_VOXELGRID option.
//
// Re-creates pcl::ApproximateVoxelGrid<pcl::PointXYZI>::applyFilter with setLeafSize(r,r,r) and every other setting at its default
// (SURVEY.md A.5), as configured at /root/reference/apps/prefiltering_nodelet.cpp:61-63 and called at :138-149.  PCL walks the
// input once in index order through a 512-slot hash table: a point whose slot holds another cell flushes that slot's centroid to
// the next output position and takes the slot over; after the last point the non-empty slots are flushed in slot order 0..511.
// The walk has an exact parallel form:
//   k_avg_keys      <- cell (ix, iy, iz) = x86 cvttss2si(floorf(p * inv_leaf)), bucket = (ix*7171 + iy*3079 + iz*4231) & 511
//   radix sort      <- stable 9-bit sort by bucket: inside a bucket the points stay in input order, which is the walk's order
//   k_avg_runs      <- a run (one output) starts where the bucket or the cell changes; a run followed by another run of the same
//                      bucket is flushed by that run's first point: a trigger flag at that point's input index
//   exclusive scan  <- triggers in input order: the output slot of every flushed run
//   k_avg_rank      <- a bucket's last run goes to T + rank of its bucket among the non-empty buckets (T = number of triggers)
//   k_avg_centroid  <- one thread per run, sequential float32 sums of x, y, z, intensity in the walk's order, / count
// Outputs, their order, counts and centroids are bit-exact against the sequential walk.  There is no finiteness check (PCL has
// none): a non-finite coordinate lands in cell INT_MIN along that axis, and the NaN / inf it carries reaches its run's centroid.
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <climits>
#include "engine.cuh"
#include "voxelgrid.cuh"

namespace b2r {

constexpr int kAvgSlots = 512;  // ApproximateVoxelGrid's histsize_ (no setter is called)
constexpr int kAvgBlock = 256;

// (int)f as x86's cvttss2si computes it: truncation in range; NaN, +-inf and values outside int32 give INT_MIN.  (The device's own
// conversion saturates instead and turns NaN into 0.)
__device__ __forceinline__ int x86_cvtt(float f) { return (f >= -2147483648.0f && f < 2147483648.0f) ? (int)f : INT_MIN; }

struct AvgCell {
  int i, j, k;
};
__device__ __forceinline__ AvgCell avg_cell(const float* p, float inv_leaf) {
  return {x86_cvtt(floorf(fmul(p[0], inv_leaf))), x86_cvtt(floorf(fmul(p[1], inv_leaf))), x86_cvtt(floorf(fmul(p[2], inv_leaf)))};
}
// PCL's int hash with wrapping (uint32) arithmetic, masked to the table size
__device__ __forceinline__ int avg_bucket(AvgCell c) {
  return (int)(((unsigned)c.i * 7171u + (unsigned)c.j * 3079u + (unsigned)c.k * 4231u) & (unsigned)(kAvgSlots - 1));
}

__global__ void k_avg_keys(const float* __restrict__ raw, int stride_f, int n, float inv_leaf, int* keys, int* vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  keys[i] = avg_bucket(avg_cell(raw + (size_t)i * stride_f, inv_leaf));
  vals[i] = i;
}

// sorted position s -> heads[s] (a run starts here), trig[input index] (this point flushes the run before it), occ[bucket] = 1
__global__ void k_avg_runs(const float* __restrict__ raw, int stride_f, int n, float inv_leaf, const int* __restrict__ keys,
                           const int* __restrict__ vals, int* heads, int* trig, int* occ) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int b = keys[s];
  int head = 1, t = 0;
  if (s > 0 && keys[s - 1] == b) {
    const AvgCell c0 = avg_cell(raw + (size_t)vals[s - 1] * stride_f, inv_leaf);
    const AvgCell c1 = avg_cell(raw + (size_t)vals[s] * stride_f, inv_leaf);
    head = t = (c0.i != c1.i || c0.j != c1.j || c0.k != c1.k) ? 1 : 0;
  } else {
    occ[b] = 1;
  }
  heads[s] = head;
  trig[vals[s]] = t;
}

// one block of kAvgSlots threads: occ[b] (1 = bucket b holds points) -> the output slot of bucket b's last run; total[0] = output
// count, total[1] = T
__global__ void __launch_bounds__(kAvgSlots) k_avg_rank(int* occ, const int* __restrict__ trig, const int* __restrict__ tslot, int n, int* total) {
  __shared__ int sc[kAvgSlots];
  const int t = threadIdx.x;
  const int v = occ[t];
  sc[t] = v;
  __syncthreads();
  for (int o = 1; o < kAvgSlots; o <<= 1) {
    const int a = t >= o ? sc[t - o] : 0;
    __syncthreads();
    sc[t] += a;
    __syncthreads();
  }
  const int T = tslot[n - 1] + trig[n - 1];
  occ[t] = T + sc[t] - v;
  if (t == kAvgSlots - 1) { total[0] = T + sc[t]; total[1] = T; }
}

__global__ void k_avg_centroid(const float* __restrict__ raw, int stride_f, int n, const int* __restrict__ keys, const int* __restrict__ vals,
                               const int* __restrict__ heads, const int* __restrict__ tslot, const int* __restrict__ last_slot, float* out,
                               int* ocounts) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n || !heads[s]) return;
  const bool has_i = stride_f >= 5;
  float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
  int e = s;
  do {
    const float* p = raw + (size_t)vals[e] * stride_f;
    sx = fadd(sx, p[0]); sy = fadd(sy, p[1]); sz = fadd(sz, p[2]);
    si = fadd(si, has_i ? p[4] : 0.f);
    e++;
  } while (e < n && !heads[e]);
  const int b = keys[s];
  const int slot = (e < n && keys[e] == b) ? tslot[vals[e]] : last_slot[b];
  const float cnt = (float)(e - s);
  float* o = out + (size_t)slot * stride_f;
  o[0] = __fdiv_rn(sx, cnt); o[1] = __fdiv_rn(sy, cnt); o[2] = __fdiv_rn(sz, cnt);
  if (stride_f >= 4) o[3] = 1.0f;
  if (stride_f >= 5) o[4] = __fdiv_rn(si, cnt);
  for (int j = 5; j < stride_f; j++) o[j] = 0.f;
  ocounts[slot] = e - s;
}

// device-resident approximate voxel grid: d_in (device records, 1 <= n <= 0x3fffffff) -> W.out / W.ocounts (device); *m = output
// count, the one value that comes back to the host
inline int approx_voxelgrid_device(VoxelWork& W, cudaStream_t st, const float* d_in, size_t n, size_t stride_bytes, float leaf, size_t* m) {
  const int sf = (int)(stride_bytes / 4);
  const int N = (int)n;
  const float inv_leaf = 1.0f / leaf;  // inverse_leaf_size_ = Array3f::Ones() / leaf_size_
  int rc = vg_alloc_words(W);
  if (rc) return rc;
  B2R_CUDA(W.out.reserve(n * sf + 8));
  B2R_CUDA(W.ocounts.reserve(n + 1));
  B2R_CUDA(W.keys_a.reserve(n)); B2R_CUDA(W.keys_b.reserve(n)); B2R_CUDA(W.vals_a.reserve(n)); B2R_CUDA(W.vals_b.reserve(n));
  B2R_CUDA(W.flags.reserve(n)); B2R_CUDA(W.slots.reserve(n)); B2R_CUDA(W.buckets.reserve(kAvgSlots));
  size_t tmp_sort = 0, tmp_scan = 0;
  B2R_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, W.keys_a.p, W.keys_b.p, W.vals_a.p, W.vals_b.p, N, 0, 9, st));
  B2R_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_scan, W.flags.p, W.slots.p, N, st));
  B2R_CUDA(W.tmp.reserve(std::max(tmp_sort, tmp_scan) + 256));
  const unsigned nb = (unsigned)((n + kAvgBlock - 1) / kAvgBlock);
  int* heads = W.keys_a.p;  // the sort's input keys are free once it has run
  TEL_BEGIN(W.tel, st);
  B2R_CUDA(cudaMemsetAsync(W.buckets.p, 0, kAvgSlots * sizeof(int), st));
  k_avg_keys<<<nb, kAvgBlock, 0, st>>>(d_in, sf, N, inv_leaf, W.keys_a.p, W.vals_a.p);
  size_t tb = W.tmp.cap;
  B2R_CUDA(cub::DeviceRadixSort::SortPairs(W.tmp.p, tb, W.keys_a.p, W.keys_b.p, W.vals_a.p, W.vals_b.p, N, 0, 9, st));
  k_avg_runs<<<nb, kAvgBlock, 0, st>>>(d_in, sf, N, inv_leaf, W.keys_b.p, W.vals_b.p, heads, W.flags.p, W.buckets.p);
  tb = W.tmp.cap;
  B2R_CUDA(cub::DeviceScan::ExclusiveSum(W.tmp.p, tb, W.flags.p, W.slots.p, N, st));
  k_avg_rank<<<1, kAvgSlots, 0, st>>>(W.buckets.p, W.flags.p, W.slots.p, N, W.mm.p + 6);
  k_avg_centroid<<<nb, kAvgBlock, 0, st>>>(d_in, sf, N, W.keys_b.p, W.vals_b.p, heads, W.slots.p, W.buckets.p, W.out.p, W.ocounts.p);
  TEL_END(W.tel, KC_VOXELGRID, 9, st);
  B2R_CUDA(cudaGetLastError());
  B2R_CUDA(cudaMemcpyAsync(W.h_total.p, W.mm.p + 6, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaStreamSynchronize(st));
  *m = (size_t)W.h_total.p[0];
  return B2R_OK;
}

inline int approx_voxelgrid_filter(VoxelWork& W, cudaStream_t st, const void* in, size_t n, size_t stride_bytes, float leaf, void* out,
                                   size_t* n_out, int32_t* out_counts) {
  *n_out = 0;
  if (n == 0) return B2R_OK;
  const int sf = (int)(stride_bytes / 4);
  B2R_CUDA(W.in.reserve(n * sf));
  B2R_CUDA(cudaMemcpyAsync(W.in.p, in, n * stride_bytes, cudaMemcpyHostToDevice, st));
  if (W.tel) W.tel->h2d += n * stride_bytes;
  size_t m = 0;
  int rc = approx_voxelgrid_device(W, st, W.in.p, n, stride_bytes, leaf, &m);
  if (rc) return rc;
  B2R_CUDA(cudaMemcpyAsync(out, W.out.p, m * stride_bytes, cudaMemcpyDeviceToHost, st));
  if (out_counts) B2R_CUDA(cudaMemcpyAsync(out_counts, W.ocounts.p, m * sizeof(int), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaStreamSynchronize(st));
  if (W.tel) W.tel->d2h += m * stride_bytes;
  *n_out = m;
  return B2R_OK;
}

}  // namespace b2r
