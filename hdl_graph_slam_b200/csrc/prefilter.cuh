// prefilter.cuh — the rest of the prefilter chain next to the voxel grid (SURVEY.md §8f-2, "next" rows):
//   k_distance_flags   <- PrefilteringNodelet::distance_filter          /root/reference/apps/prefiltering_nodelet.cpp:164-180
//   k_knn_stat         <- pcl::RadiusOutlierRemoval / pcl::StatisticalOutlierRemoval as configured at :72-93 and run at :151-162
// Both outlier filters are nearest-neighbour statistics of the cloud against itself, so they reuse the BVH k-NN traversal:
//   RADIUS      keep p  iff  its (min_neighbors+1)-th nearest neighbour (itself included) lies within the radius
//   STATISTICAL keep p  iff  mean distance to its mean_k nearest neighbours (itself excluded) <= mean + mul * stddev over the cloud
//   k_deskew           <- PrefilteringNodelet::deskewing                 /root/reference/apps/prefiltering_nodelet.cpp:182-243
// Decisions and compaction stay on the device: the per-point statistic, the cloud-wide mean / stddev of the statistical filter
// (PCL's index-order float64 sums), the keep flags, and an order-preserving stream compaction (count / scan / scatter) — so the
// chain deskew -> distance filter -> voxel grid -> outlier removal hands a device-resident cloud to the registration.
#pragma once
#include "common.cuh"
#include "bvh.cuh"
#include "gicp.cuh"

namespace b2r {

struct XfArgPF { float Tf[12]; };

__global__ void k_distance_flags(const float* __restrict__ raw, int stride_f, int n, double near_t, double far_t, unsigned char* flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = raw + (size_t)i * stride_f;
  const float x = p[0], y = p[1], z = p[2];
  // Eigen Vector3f::norm(): sqrt((x*x + y*y) + z*z) in float32, then promoted to double for the comparison
  const float sq = fadd(fadd(fmul(x, x), fmul(y, y)), fmul(z, z));
  const double d = (double)__fsqrt_rn(sq);
  flags[i] = (finite3(x, y, z) && d > near_t && d < far_t) ? 1 : 0;
}

// mode 0: out[orig idx] = squared distance of the k-th nearest neighbour (self included), +inf if fewer than k points
// mode 1: out[orig idx] = (float)( sum_{j=1..k-1} sqrtf(d2_j) / (k-1) )   (PCL StatisticalOutlierRemoval, k = mean_k + 1)
//         mean_k = 0 gives 0/0 = NaN, as in PCL: a NaN mean distance is a valid point's statistic, so a non-finite point (not in
//         the BVH, never written here) is marked by the caller's fill with a negative value no mean distance can take.
// Non-finite points keep the caller's fill: NaN in mode 0, kStatNonFinite in mode 1.
constexpr float kStatNonFinite = -1.0f;
constexpr unsigned kStatNonFiniteBits = 0xbf800000u;  // __float_as_uint(kStatNonFinite), usable by the host's fill
__global__ void __launch_bounds__(kKnnThreads, 4) k_knn_stat(Bvh b, int k, int mode, float* __restrict__ out) {
  extern __shared__ unsigned long long knn_keys[];
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int leaf = s >> 5;
  if (leaf >= b.nleaf) return;
  const float4 q = b.sp[s];
  const bool active = idx_bits(q.w) != kPadIdx;
  KnnList L;
  L.key = knn_keys + threadIdx.x;
  L.k = k;
  L.cnt = 0;
  L.stride = blockDim.x;
  L.wkey = kKeyInf;
  bvh_group_search(b, q.x, q.y, q.z, active, L, leaf);
  if (!active) return;
  float v;
  if (mode == 0) {
    v = (L.cnt == k) ? nn_key_d2(L.key[(k - 1) * L.stride]) : INFINITY;
  } else {
    double sum = 0.0;
    for (int j = 1; j < L.cnt; j++) sum += (double)__fsqrt_rn(nn_key_d2(L.key[j * L.stride]));
    v = (float)(sum / (double)(k - 1));
  }
  out[idx_bits(q.w)] = v;
}

// ---- deskew (prefiltering_nodelet.cpp:222-240): point i is rotated back by the gyro rate over its share of the scan period.
// Float32 in Eigen's evaluation order: delta_q = Quaternionf(1, dt/2 wx, dt/2 wy, dt/2 wz) (NOT normalised), inverse() =
// conjugate / squaredNorm, q * v = v + w (2 q.vec x v) + q.vec x (2 q.vec x v).  ang_v is the already negated rate (:217).
__global__ void k_deskew(const float* __restrict__ in, int stride_f, int n, double scan_period, float wx, float wy, float wz, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = in + (size_t)i * stride_f;
  float* o = out + (size_t)i * stride_f;
  for (int k = 3; k < stride_f; k++) o[k] = p[k];  // deskewed->at(i) = cloud->at(i)
  const double delta_t = scan_period * (double)i / (double)n;
  const double half = delta_t / 2.0;
  const float qw = 1.0f, qx = (float)(half * (double)wx), qy = (float)(half * (double)wy), qz = (float)(half * (double)wz);
  // inverse(): conjugate().coeffs() / squaredNorm()
  const float n2 = fadd(fadd(fadd(fmul(qx, qx), fmul(qy, qy)), fmul(qz, qz)), fmul(qw, qw));
  const float iw = __fdiv_rn(qw, n2), ix = __fdiv_rn(-qx, n2), iy = __fdiv_rn(-qy, n2), iz = __fdiv_rn(-qz, n2);
  const float vx = p[0], vy = p[1], vz = p[2];
  // uv = 2 * (q.vec x v)
  float ux = fsub(fmul(iy, vz), fmul(iz, vy)), uy = fsub(fmul(iz, vx), fmul(ix, vz)), uz = fsub(fmul(ix, vy), fmul(iy, vx));
  ux = fadd(ux, ux); uy = fadd(uy, uy); uz = fadd(uz, uz);
  // v + w * uv + q.vec x uv
  const float cx = fsub(fmul(iy, uz), fmul(iz, uy)), cy = fsub(fmul(iz, ux), fmul(ix, uz)), cz = fsub(fmul(ix, uy), fmul(iy, ux));
  o[0] = fadd(fadd(vx, fmul(iw, ux)), cx);
  o[1] = fadd(fadd(vy, fmul(iw, uy)), cy);
  o[2] = fadd(fadd(vz, fmul(iw, uz)), cz);
}

// pcl::transformPointCloud(cloud, out, Matrix4f): xyz by the affine part (float32, ((m0 x + m1 y) + m2 z) + m3), other fields copied
__global__ void k_transform_records(const float* __restrict__ in, int stride_f, int n, XfArgPF X, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = in + (size_t)i * stride_f;
  float* o = out + (size_t)i * stride_f;
  const float x = p[0], y = p[1], z = p[2];
  for (int k = 3; k < stride_f; k++) o[k] = p[k];
  o[0] = xform_row(X.Tf[0], X.Tf[1], X.Tf[2], X.Tf[3], x, y, z);
  o[1] = xform_row(X.Tf[4], X.Tf[5], X.Tf[6], X.Tf[7], x, y, z);
  o[2] = xform_row(X.Tf[8], X.Tf[9], X.Tf[10], X.Tf[11], x, y, z);
}

// ---- keep flags of the two outlier filters from the per-point statistic (original point order)
// RADIUS (pcl::RadiusOutlierRemoval, dense path): keep iff the (min_pts+1)-th neighbour exists and is not farther than the radius
__global__ void k_radius_flags(const float* __restrict__ kth_d2, int n, double r2, unsigned char* flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = kth_d2[i];
  flags[i] = (v == v && v != INFINITY && !((double)v > r2)) ? 1 : 0;
}

// STATISTICAL (pcl::StatisticalOutlierRemoval::applyFilterIndices): sum and sum of squares of the per-point mean distances over
// the VALID points (a non-finite point has distance 0 and is kept); squares are formed in float32 as PCL's `distance * distance`.
// The two float64 sums are PCL's: one running sum each, in index order.  A float64 sum of values spanning many binades depends on
// its order, and a mean distance that lands between two orders' thresholds is kept by one and removed by the other.
// Fast path: every term is a non-negative multiple of 2^e (e = the smallest ulp exponent among the nonzero float32 terms), so
// while a sum stays below 2^(e+53) every partial sum, in any order, is exact.  The block first sums in parallel (thread t adds
// t, t + 1024, ..., then two butterflies); if a computed sum is below that bound, no partial sum can have rounded (the first
// rounded one would be >= the bound, and adding non-negative terms never brings a rounded sum back below it), so it IS the
// sequential sum.  NaN / inf sums are the same in every order too.  Otherwise the block stages tiles of the distances in shared
// memory and thread 0 adds them up in index order (~16.5 ns per point on an H100: the _wide clouds of tools/sor_time.py).
constexpr int kSorThreads = 1024, kSorTile = 8192;
struct SorStats { double sum, sq_sum, thresh; unsigned long long valid; };
__device__ __forceinline__ int sor_ulp_exp(float v) { return max((__float_as_int(v) >> 23) & 0xff, 1) - 150; }  // v >= 0
__device__ __forceinline__ bool sor_order_free(double s, int e) { return !(s <= DBL_MAX) || e == INT_MAX || s < ldexp(1.0, e + 53); }
__global__ void __launch_bounds__(kSorThreads) k_sor_stats(const float* __restrict__ dist, int n, double stddev_mul, SorStats* out) {
  __shared__ float tile[kSorTile];
  __shared__ double s_sum[32], s_sq[32];
  __shared__ unsigned long long s_cnt[32];
  __shared__ int s_e[32], s_esq[32];
  __shared__ int sequential;
  double sum = 0.0, sq = 0.0;
  unsigned long long cnt = 0;
  int e = INT_MAX, esq = INT_MAX;
  for (int i = threadIdx.x; i < n; i += kSorThreads) {
    const float d = dist[i];
    if (d < 0.f) continue;  // kStatNonFinite
    const float dd = fmul(d, d);
    sum += (double)d;
    sq += (double)dd;
    cnt++;
    if (d > 0.f) e = min(e, sor_ulp_exp(d));
    if (dd > 0.f) esq = min(esq, sor_ulp_exp(dd));
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o); sq += __shfl_xor_sync(0xffffffffu, sq, o); cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  e = __reduce_min_sync(0xffffffffu, e);
  esq = __reduce_min_sync(0xffffffffu, esq);
  if (lane == 0) { s_sum[warp] = sum; s_sq[warp] = sq; s_cnt[warp] = cnt; s_e[warp] = e; s_esq[warp] = esq; }
  __syncthreads();
  if (warp == 0) {
    sum = s_sum[lane]; sq = s_sq[lane]; cnt = s_cnt[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sum += __shfl_xor_sync(0xffffffffu, sum, o); sq += __shfl_xor_sync(0xffffffffu, sq, o); cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    e = __reduce_min_sync(0xffffffffu, s_e[lane]);
    esq = __reduce_min_sync(0xffffffffu, s_esq[lane]);
    if (lane == 0) sequential = !(sor_order_free(sum, e) && sor_order_free(sq, esq));
  }
  __syncthreads();
  if (sequential) {
    sum = 0.0; sq = 0.0; cnt = 0;
    for (int base = 0; base < n; base += kSorTile) {
      const int m = min(kSorTile, n - base);
      for (int j = threadIdx.x; j < m; j += kSorThreads) tile[j] = dist[base + j];
      __syncthreads();
      if (threadIdx.x == 0) {
#pragma unroll 8
        for (int j = 0; j < m; j++) {
          const float d = tile[j];
          // a non-finite point (d == kStatNonFinite) is skipped: adding +0.0 leaves a sum of non-negative terms unchanged
          const bool valid = !(d < 0.f);
          sum += valid ? (double)d : 0.0;
          sq += valid ? (double)fmul(d, d) : 0.0;
          cnt += valid ? 1u : 0u;
        }
      }
      __syncthreads();
    }
  }
  if (threadIdx.x == 0) {  // thread 0 holds the block's sums on either path
    const double nv = (double)cnt;
    const double mean = sum / nv;
    const double variance = (sq - sum * sum / nv) / (nv - 1.0);
    out->sum = sum; out->sq_sum = sq; out->valid = cnt;
    out->thresh = __dadd_rn(mean, __dmul_rn(stddev_mul, sqrt(variance)));  // two roundings, as PCL: no fused multiply-add
  }
}
__global__ void k_sor_flags(const float* __restrict__ dist, int n, const SorStats* __restrict__ st, unsigned char* flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float d = dist[i];
  // non-finite point: distance 0.0 <= threshold -> kept, as PCL does; mean_k = 0 (every mean distance NaN, so the threshold is NaN):
  // !(d > NaN) keeps every point, as PCL does; no valid point at all: everything is removed
  const double dd = (d < 0.f) ? 0.0 : (double)d;
  flags[i] = (st->valid > 0 && !(dd > st->thresh)) ? 1 : 0;
}

// ---- order-preserving stream compaction of records by flags: block counts, one-block scan of the counts, scatter
constexpr int kCompactBlock = 1024;
__global__ void __launch_bounds__(kCompactBlock) k_compact_count(const unsigned char* __restrict__ flags, int n, int* block_cnt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = __syncthreads_count(i < n && flags[i]);
  if (threadIdx.x == 0) block_cnt[blockIdx.x] = c;
}
__global__ void __launch_bounds__(1024) k_compact_scan(int* block_cnt, int nblk, int* total, volatile int* h_total) {
  __shared__ int wsum[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < nblk; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < nblk ? block_cnt[i] : 0;
    int inc = v;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      int w = wsum[lane], winc = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += t; }
      wsum[lane] = winc - w;
    }
    __syncthreads();
    const int excl = inc - v + wsum[warp] + carry;
    if (i < nblk) block_cnt[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) { *total = carry; if (h_total) *h_total = carry; }
}
__global__ void __launch_bounds__(kCompactBlock) k_compact_scatter(const float* __restrict__ in, int stride_f, const unsigned char* __restrict__ flags, int n,
                                                                  const int* __restrict__ block_off, float* __restrict__ out) {
  __shared__ int wsum[32];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool keep = i < n && flags[i];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) wsum[warp] = __popc(m);
  __syncthreads();
  if (warp == 0) {
    int w = wsum[lane], winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += t; }
    wsum[lane] = winc - w;
  }
  __syncthreads();
  if (!keep) return;
  const int dst = block_off[blockIdx.x] + wsum[warp] + __popc(m & ((1u << lane) - 1u));
  const float* p = in + (size_t)i * stride_f;
  float* o = out + (size_t)dst * stride_f;
  for (int k = 0; k < stride_f; k++) o[k] = p[k];
}

}  // namespace b2r
