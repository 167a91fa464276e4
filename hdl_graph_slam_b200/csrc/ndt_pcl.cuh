// ndt_pcl.cuh — the factory's `NDT` branch: pcl::NormalDistributionsTransform (PCL 1.10) on the engine's voxel map.
//
// Re-creates, GPU-first, what pcl::NormalDistributionsTransform adds to the voxel Gaussians ndt.cuh already builds
// (registrations.cpp:93-100; semantics pinned by tests/ndt_pcl_ref.cpp, see its header):
//   k_pcl_centroids / k_pcl_buckets  <- VoxelGridCovariance::filter(true): the float32 centroid of every leaf with >= 6 points,
//                                       searchable (here: bucketed by its own cell, CSR over a hash table)
//   pcl_collect                      <- target_cells_.radiusSearch(x_trans_pt, resolution_): FLANN L2_Simple<float>, d2 < (float)r^2
//   k_ndt_pcl_derivatives            <- computeDerivatives / computePointDerivatives / updateDerivatives, float64, unfused
//                                       (the Hessian-only pass of computeHessian / updateHessian is the same term: the same kernel
//                                       with the Hessian, read for H alone)
// The Newton / More-Thuente driver (NdtPairState), the chunk-ticket queue and the fixed reduction tree are ndt.cuh's.
#pragma once

namespace b2r {

constexpr unsigned long long kPclNoBucket = 1ull << 40;  // sorts after every bucket key (keys < 27 * 2^31 < 2^36)
constexpr int kPclBucketBits = 41;
constexpr int kPclNb = 32;  // neighbours held per selection round of one point (more are taken in further rounds)

struct NdtPclArgs {
  NdtArgs A;                          // source, pose, angle derivatives, voxel records and the reduction workspace of the pass
  const float4* cent;                 // per sorted position s of the voxel map: the centroid of the voxel whose record is at s
  const int* bpos;                    // centroid positions s grouped by bucket, ascending s inside a bucket
  const unsigned long long* btab_key; // bucket key -> slot (kNdtEmpty = free)
  const uint2* btab_val;              // slot -> (first index into bpos, count)
  unsigned int bmask;
  int blo[3], bhi[3];                 // bucket cells min_b - 1 .. max_b + 1 per axis (every cell outside is clamped onto them)
  unsigned long long bdim0, bdim01;
  float r2;                           // (float)(resolution * resolution), as KdTreeFLANN::radiusSearch passes it
  double r_margin;                    // 1.0001 * resolution: the box searched around a query (see pcl_collect)
};

// the bucket cell of a coordinate: floor(c * inv_leaf) in float32 (the voxel keys' product), clamped onto [lo, hi] in float64 so
// that no coordinate, however far out or infinite, overflows the integer conversion.  Monotone non-decreasing in c.
__device__ __forceinline__ int pcl_cell_axis(float c, float inv_leaf, int lo, int hi) {
  const double f = (double)floorf(fmul(c, inv_leaf));
  return f < (double)lo ? lo : (f > (double)hi ? hi : (int)f);
}

__device__ __forceinline__ unsigned long long pcl_bucket_key(const NdtPclArgs& P, int i, int j, int k) {
  return (unsigned long long)(i - P.blo[0]) + (unsigned long long)(j - P.blo[1]) * P.bdim0 + (unsigned long long)(k - P.blo[2]) * P.bdim01;
}

__device__ __forceinline__ unsigned int pcl_hash64(unsigned long long k) { return ndt_hash((unsigned int)k ^ ndt_hash((unsigned int)(k >> 32))); }

// VoxelGridCovariance::applyFilter's centroid: one thread per voxel (at the sorted position of its first point): the float32 sum of
// x, y, z in ascending point index, divided by (float)nr_points, for every leaf of >= 6 points (counted before invalidation).
// bkey[s] = the centroid's bucket key (kPclNoBucket at every other position), bpos[s] = s: the sort input of the bucket CSR.
__global__ void k_pcl_centroids(const unsigned int* __restrict__ keys_sorted, const float4* __restrict__ sorted, const VoxGeom* __restrict__ vg,
                                float4* cent, unsigned long long* bkey, int* bpos, int n) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  bpos[s] = s;
  unsigned long long bk = kPclNoBucket;
  const unsigned int key = keys_sorted[s];
  if (key != 0xffffffffu && (s == 0 || keys_sorted[s - 1] != key)) {
    float sx = 0.f, sy = 0.f, sz = 0.f;
    int cnt = 0;
    for (int j = s; j < n && keys_sorted[j] == key; j++) {
      const float4 p = sorted[j];
      sx = fadd(sx, p.x); sy = fadd(sy, p.y); sz = fadd(sz, p.z);
      cnt++;
    }
    if (cnt >= 6) {
      const VoxGeom V = *vg;
      const float fc = (float)cnt;
      const float cx = __fdiv_rn(sx, fc), cy = __fdiv_rn(sy, fc), cz = __fdiv_rn(sz, fc);
      cent[s] = make_float4(cx, cy, cz, bits_idx(s));
      const int b0 = V.min_b[0] - 1, b1 = V.min_b[1] - 1, b2 = V.min_b[2] - 1;
      const unsigned long long d0 = (unsigned long long)(V.div_b[0] + 2), d01 = d0 * (unsigned long long)(V.div_b[1] + 2);
      const int i = pcl_cell_axis(cx, V.inv_leaf, b0, V.max_b[0] + 1);
      const int jj = pcl_cell_axis(cy, V.inv_leaf, b1, V.max_b[1] + 1);
      const int k = pcl_cell_axis(cz, V.inv_leaf, b2, V.max_b[2] + 1);
      bk = (unsigned long long)(i - b0) + (unsigned long long)(jj - b1) * d0 + (unsigned long long)(k - b2) * d01;
    }
  }
  bkey[s] = bk;
}

// one thread per position of the bucket-sorted centroids: the first of each bucket inserts (key -> (position, count))
__global__ void k_pcl_buckets(const unsigned long long* __restrict__ bkey_sorted, unsigned long long* tab_key, uint2* tab_val, unsigned int mask, int n) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const unsigned long long k = bkey_sorted[t];
  if (k == kPclNoBucket || (t > 0 && bkey_sorted[t - 1] == k)) return;
  int cnt = 0;
  for (int j = t; j < n && bkey_sorted[j] == k; j++) cnt++;
  unsigned int h = pcl_hash64(k) & mask;
  while (atomicCAS(tab_key + h, kNdtEmpty, k) != kNdtEmpty) h = (h + 1) & mask;  // every key is inserted once
  tab_val[h] = make_uint2((unsigned int)t, (unsigned int)cnt);
}

// radiusSearch(q, r): every centroid c with float32 d2 = ((dx*dx + dy*dy) + dz*dz) < r2, d = q - c.  Keeps the kPclNb smallest
// (d2, s) keys above `after` in buf, ascending, and returns how many keys lie above `after` in all.
//
// Completeness: d2 < r2 in float32 implies |q - c| < r (1 + 3 u) < 1.0001 r per axis in real numbers (u = 2^-24: dx, dx*dx and
// the sums each round by at most a factor 1 -+ u, and r2 = (float)(r*r) <= r*r (1 + u)).  So c lies strictly inside the real
// interval (q - 1.0001 r, q + 1.0001 r); lo / hi are that interval's ends rounded outwards to float32, so lo <= c <= hi.  The
// bucket cell is a monotone function of the coordinate (float32 product with the positive inv_leaf, floor, clamp), so
// cell(lo) <= cell(c) <= cell(hi): the buckets of the box [cell(lo), cell(hi)]^3 hold every neighbour, whichever way the float
// sums put a centroid relative to its own voxel, and a query exactly at distance r fails the strict test like any other.  A far
// query clamps onto the outermost buckets and is decided by the same exact test.
__device__ __forceinline__ int pcl_collect(const NdtPclArgs& P, const VoxGeom& V, float qx, float qy, float qz, long long after,
                                           unsigned long long* buf) {
  const float q[3] = {qx, qy, qz};
  int lo[3], hi[3];
#pragma unroll
  for (int d = 0; d < 3; d++) {
    lo[d] = pcl_cell_axis(__double2float_rd((double)q[d] - P.r_margin), V.inv_leaf, P.blo[d], P.bhi[d]);
    hi[d] = pcl_cell_axis(__double2float_ru((double)q[d] + P.r_margin), V.inv_leaf, P.blo[d], P.bhi[d]);
  }
  int total = 0, held = 0;
  for (int k = lo[2]; k <= hi[2]; k++)
    for (int j = lo[1]; j <= hi[1]; j++)
      for (int i = lo[0]; i <= hi[0]; i++) {
        const unsigned long long key = pcl_bucket_key(P, i, j, k);
        unsigned int h = pcl_hash64(key) & P.bmask;
        unsigned long long e;
        while ((e = __ldg(P.btab_key + h)) != key && e != kNdtEmpty) h = (h + 1) & P.bmask;
        if (e == kNdtEmpty) continue;
        const uint2 span = __ldg(P.btab_val + h);
        for (unsigned int t = span.x; t < span.x + span.y; t++) {
          const int s = __ldg(P.bpos + t);
          const float4 c = __ldg(P.cent + s);
          const float d2 = dist2_f32(qx, qy, qz, c.x, c.y, c.z);
          if (!(d2 < P.r2)) continue;
          const unsigned long long kk = ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned int)s;  // d2 >= 0: bits order as values
          if ((long long)kk <= after) continue;
          total++;
          if (held == kPclNb && kk >= buf[kPclNb - 1]) continue;
          int pos = held < kPclNb ? held++ : kPclNb - 1;
          while (pos > 0 && buf[pos - 1] > kk) { buf[pos] = buf[pos - 1]; pos--; }
          buf[pos] = kk;
        }
      }
  return total;
}

// updateDerivatives (and, the same expression, updateHessian) for one (point, leaf), float64 in PCL's written order, unfused.
// x_trans = (double)x_trans_pt - mean; J = point_gradient_ (columns 0..2 the identity), jx / hx = the original point's dot products
// with j_ang_* / h_ang_*.  acc: score, g[6], the upper triangle of H; low: this thread's column of the strict lower triangle.
template <bool HESS>
__device__ __forceinline__ void ndt_pcl_term(const NdtArgs& A, const NdtVoxel* __restrict__ L, double xt, double yt, double zt, const double* jx,
                                             const double* hx, double* acc, double* low) {
  const double q0 = dsub(xt, L->mean[0]), q1 = dsub(yt, L->mean[1]), q2 = dsub(zt, L->mean[2]);
  double C[9];
#pragma unroll
  for (int k = 0; k < 9; k++) C[k] = L->icov[k];
  double Cq[3];
#pragma unroll
  for (int r = 0; r < 3; r++) Cq[r] = dadd(dadd(dmul(C[r * 3 + 0], q0), dmul(C[r * 3 + 1], q1)), dmul(C[r * 3 + 2], q2));
  const double qCq = dadd(dadd(dmul(q0, Cq[0]), dmul(q1, Cq[1])), dmul(q2, Cq[2]));
  double e = exp(dmul(-A.d2, qCq) / 2.0);
  const double score_inc = dmul(-A.d1, e);
  e = dmul(A.d2, e);
  if (e > 1.0 || e < 0.0 || e != e) return;  // updateDerivatives returns 0: the term adds nothing, not even its score
  e = dmul(e, A.d1);
  acc[0] = dadd(acc[0], score_inc);
  const double J[3][6] = {{1.0, 0.0, 0.0, 0.0, jx[2], jx[5]}, {0.0, 1.0, 0.0, jx[0], jx[3], jx[6]}, {0.0, 0.0, 1.0, jx[1], jx[4], jx[7]}};
  double CJ[3][6], gq[6];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int i = 0; i < 6; i++) CJ[r][i] = dadd(dadd(dmul(C[r * 3 + 0], J[0][i]), dmul(C[r * 3 + 1], J[1][i])), dmul(C[r * 3 + 2], J[2][i]));
#pragma unroll
  for (int i = 0; i < 6; i++) {
    gq[i] = dadd(dadd(dmul(q0, CJ[0][i]), dmul(q1, CJ[1][i])), dmul(q2, CJ[2][i]));
    acc[1 + i] = dadd(acc[1 + i], dmul(gq[i], e));
  }
  if (HESS) {
    // point_hessian_ blocks (i, j >= 3): a = (0, hx0, hx1), b = (0, hx2, hx3), c = (0, hx4, hx5), d, e, f = hx[6..8], [9..11], [12..14]
    const double Z = 0.0;
    const double PH[6][3] = {{Z, hx[0], hx[1]}, {Z, hx[2], hx[3]}, {Z, hx[4], hx[5]}, {hx[6], hx[7], hx[8]}, {hx[9], hx[10], hx[11]}, {hx[12], hx[13], hx[14]}};
    const int blk[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
    int hk = 7, lk = 0;
#pragma unroll
    for (int ii = 0; ii < 6; ii++)
#pragma unroll
      for (int jj = 0; jj < 6; jj++) {
        double xh = 0.0;  // x_trans . (C * 0) outside the angular block
        if (ii >= 3 && jj >= 3) {
          const double* v = PH[blk[ii - 3][jj - 3]];
          double Cv[3];
#pragma unroll
          for (int r = 0; r < 3; r++) Cv[r] = dadd(dadd(dmul(C[r * 3 + 0], v[0]), dmul(C[r * 3 + 1], v[1])), dmul(C[r * 3 + 2], v[2]));
          xh = dadd(dadd(dmul(q0, Cv[0]), dmul(q1, Cv[1])), dmul(q2, Cv[2]));
        }
        const double jcj = dadd(dadd(dmul(J[0][jj], CJ[0][ii]), dmul(J[1][jj], CJ[1][ii])), dmul(J[2][jj], CJ[2][ii]));
        const double w = dmul(e, dadd(dadd(dmul(dmul(-A.d2, gq[ii]), gq[jj]), xh), jcj));
        if (jj >= ii) { acc[hk] = dadd(acc[hk], w); hk++; }
        else { low[lk * kNdtRow] = dadd(low[lk * kNdtRow], w); lk++; }
      }
  }
}

// The end of a chunk of a derivative pass: the pair count, the chunk's row of kNdtAcc sums (tile: shared rows of kNdtRow
// doubles, free once the pair loop is over; low: the kNdtAccB shared columns of the strict lower triangle of H), and the fixed
// two-level tree over the chunk rows, whose last block publishes the result: the same sequence as the end of ndt.cuh's
// ndt_derivatives_body (which keeps its own inline copy: calling this helper there moves that kernel's register assignment).
template <bool HESS>
__device__ __forceinline__ void ndt_chunk_finish(const NdtArgs& A, int chunk, int nchunks, unsigned int npairs, const double* acc, double* tile,
                                                 const double* low, double* s_fin, int& s_role) {
  constexpr int NV = HESS ? kNdtAcc : 7;  // values that carry information (score + gradient without the Hessian)
  const int lane = threadIdx.x & 31;
  __syncthreads();  // the pair loop is over: the staging area becomes the reduction rows
  // pair count (integer, exact) through a warp reduction + one atomic per warp
  npairs = __reduce_add_sync(0xffffffffu, npairs);
  if (lane == 0 && npairs) atomicAdd(A.pairs, (unsigned long long)npairs);
  // ---- this chunk's row of sums
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
    ndt_rows_sum(low, kNdtAccB, my_row + kNdtAccA);
  }
  __syncthreads();  // the row is written (by several threads); the shared arrays are free for the next chunk
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
        publish_flag(A.flag, A.seq, A.round, A.round_n);
      }
    }
  }
}

// The term rule of pcl::NormalDistributionsTransform (B2R_METHOD_NDT_PCL): computePointDerivatives of the original point promoted
// to double, and ndt_pcl_term over the voxel's float64 record at the neighbour's sorted position s.
struct NdtPclTermRule {
  template <bool HESS>
  struct Point { double jx[8], hx[15]; };
  template <bool HESS>
  static __device__ __forceinline__ void point(const NdtArgs& A, float x, float y, float z, Point<HESS>& pd) {
    const double xd = x, yd = y, zd = z;
#pragma unroll
    for (int r = 0; r < 8; r++) pd.jx[r] = dadd(dadd(dmul(xd, A.jang_d[r][0]), dmul(yd, A.jang_d[r][1])), dmul(zd, A.jang_d[r][2]));
    if (HESS) {
#pragma unroll
      for (int r = 0; r < 15; r++) pd.hx[r] = dadd(dadd(dmul(xd, A.hang_d[r][0]), dmul(yd, A.hang_d[r][1])), dmul(zd, A.hang_d[r][2]));
    }
  }
  template <bool HESS>
  static __device__ __forceinline__ void term(const NdtArgs& A, unsigned int s, float xt, float yt, float zt, const Point<HESS>& pd, double* acc,
                                              double* low) {
    ndt_pcl_term<HESS>(A, A.vox + s, (double)xt, (double)yt, (double)zt, pd.jx, pd.hx, acc, low);
  }
};

// computeDerivatives over the Hilbert-sorted source: one thread per point, its radius neighbours in ascending (d2, leaf) order,
// then the chunk row and the fixed two-level tree (ndt_chunk_finish), so the sums are bitwise reproducible.  Rule: the per-point
// derivatives and the per-(point, neighbour) term (NdtPclTermRule here; ndt_kdtree.cuh's NdtKdtreeTermRule for NDT_OMP's KDTREE).
template <class Rule, bool HESS>
__device__ __forceinline__ void ndt_pcl_derivatives_body(const NdtPclArgs& P) {
  const NdtArgs& A = P.A;
  __shared__ __align__(16) double s_tile[14 * kNdtRow];
  __shared__ double s_low[kNdtAccB][kNdtRow];
  __shared__ double s_fin[kNdtAcc];
  __shared__ int s_chunk, s_role;
  const VoxGeom V = *A.geom;
  const int nchunks = A.n_sorted / kNdtThreads;
  for (;;) {
    if (threadIdx.x == 0) s_chunk = (int)(atomicAdd(A.queue, 1ull) - A.qbase);
    __syncthreads();
    const int chunk = s_chunk;
    if (chunk >= nchunks) break;  // block-uniform
    double acc[kNdtAccA];
#pragma unroll
    for (int k = 0; k < kNdtAccA; k++) acc[k] = 0.0;
    if (HESS) {
#pragma unroll
      for (int q = 0; q < kNdtAccB; q++) s_low[q][threadIdx.x] = 0.0;
    }
    unsigned int npairs = 0;
    const float4 pt = A.src[chunk * kNdtThreads + threadIdx.x];
    if (idx_bits(pt.w) != kPadIdx && !V.empty && V.ok) {
      const float x = pt.x, y = pt.y, z = pt.z;
      const float xt = xform_row(A.Tf[0], A.Tf[1], A.Tf[2], A.Tf[3], x, y, z);
      const float yt = xform_row(A.Tf[4], A.Tf[5], A.Tf[6], A.Tf[7], x, y, z);
      const float zt = xform_row(A.Tf[8], A.Tf[9], A.Tf[10], A.Tf[11], x, y, z);
      if (finite3(xt, yt, zt)) {
        // computePointDerivatives(x): the original point
        typename Rule::template Point<HESS> pd;
        Rule::template point<HESS>(A, x, y, z, pd);
        unsigned long long buf[kPclNb];
        long long after = -1;
        for (;;) {
          const int total = pcl_collect(P, V, xt, yt, zt, after, buf);
          const int m = min(total, kPclNb);
          for (int t = 0; t < m; t++) Rule::template term<HESS>(A, (unsigned int)buf[t], xt, yt, zt, pd, acc, &s_low[0][threadIdx.x]);
          npairs += (unsigned int)m;
          if (total <= kPclNb) break;
          after = (long long)buf[kPclNb - 1];
        }
      }
    }
    ndt_chunk_finish<HESS>(A, chunk, nchunks, npairs, acc, s_tile, &s_low[0][0], s_fin, s_role);
  }
}

template <bool HESS>
__global__ void __launch_bounds__(kNdtThreads) k_ndt_pcl_derivatives(const __grid_constant__ NdtPclArgs P) {
  ndt_pcl_derivatives_body<NdtPclTermRule, HESS>(P);
}

// many pairs: blockIdx.y = the pair's record, each pair with its own tickets, rows and counters (as k_ndt_derivatives_batch)
template <bool HESS>
__global__ void __launch_bounds__(kNdtThreads) k_ndt_pcl_derivatives_batch(const NdtPclArgs* __restrict__ recs) {
  ndt_pcl_derivatives_body<NdtPclTermRule, HESS>(recs[blockIdx.y]);
}

// b2r_ndt_neighbors_at: the radius neighbours of each point of the source in the caller's order (counts, then positions)
__global__ void k_ndt_pcl_neighbors(const __grid_constant__ NdtPclArgs P, const float* __restrict__ raw, int stride_f, int n, unsigned int* counts,
                                    const unsigned long long* __restrict__ offsets, int* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const NdtArgs& A = P.A;
  const VoxGeom V = *A.geom;
  const float* p = raw + (size_t)i * stride_f;
  unsigned int cnt = 0;
  if (!V.empty && V.ok) {
    const float xt = xform_row(A.Tf[0], A.Tf[1], A.Tf[2], A.Tf[3], p[0], p[1], p[2]);
    const float yt = xform_row(A.Tf[4], A.Tf[5], A.Tf[6], A.Tf[7], p[0], p[1], p[2]);
    const float zt = xform_row(A.Tf[8], A.Tf[9], A.Tf[10], A.Tf[11], p[0], p[1], p[2]);
    if (finite3(xt, yt, zt)) {
      unsigned long long buf[kPclNb];
      long long after = -1;
      for (;;) {
        const int total = pcl_collect(P, V, xt, yt, zt, after, buf);
        const int m = min(total, kPclNb);
        if (offsets)
          for (int t = 0; t < m; t++) out[offsets[i] + cnt + t] = (int)(unsigned int)buf[t];
        cnt += (unsigned int)m;
        if (total <= kPclNb) break;
        after = (long long)buf[kPclNb - 1];
      }
    }
  }
  if (!offsets) counts[i] = cnt;
}

// ------------------------------------------------------------------------------------------------ host side
inline int ndt_sync_geom(NdtVoxelMap& M, NdtWork& W, cudaStream_t st);

// blocks of k_ndt_pcl_derivatives the device holds at once, asked once per process
inline unsigned ndt_pcl_resident_blocks(bool hess) {
  static unsigned cached[2] = {0, 0};
  unsigned& c = cached[hess ? 1 : 0];
  if (c == 0) {
    int dev = 0, sms = 132, per = 4;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (hess) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_ndt_pcl_derivatives<true>, kNdtThreads, 0);
    else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_ndt_pcl_derivatives<false>, kNdtThreads, 0);
    if (const char* e = getenv("B2R_NDT_WAVES")) { const double w = atof(e); if (w > 0) per = std::max(1, (int)(per * w)); }
    c = (unsigned)std::max(1, sms * std::max(per, 1));
  }
  return c;
}

// after k_vox_finalize, for a B2R_METHOD_NDT_PCL target only: centroids, their bucket CSR and its hash table
inline int ndt_pcl_build(NdtVoxelMap& M, BuildCtx* B, int n, cudaStream_t st) {
  size_t tsize = 1024;
  while (tsize < 2 * (size_t)n) tsize <<= 1;
  M.bmask = (unsigned int)(tsize - 1);
  B2R_CUDA(M.cent.reserve((size_t)n + 1));
  B2R_CUDA(M.bkey.reserve((size_t)n + 1)); B2R_CUDA(M.bkey_sorted.reserve((size_t)n + 1));
  B2R_CUDA(M.bpos_in.reserve((size_t)n + 1)); B2R_CUDA(M.bpos.reserve((size_t)n + 1));
  B2R_CUDA(M.btab_key.reserve(tsize)); B2R_CUDA(M.btab_val.reserve(tsize));
  B2R_CUDA(cudaMemsetAsync(M.btab_key.p, 0xff, tsize * sizeof(unsigned long long), st));
  if (n <= 0) return B2R_OK;
  size_t tmp_bytes = 0;
  B2R_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, M.bkey.p, M.bkey_sorted.p, M.bpos_in.p, M.bpos.p, n, 0, kPclBucketBits, st));
  B2R_CUDA(B->sort_tmp.reserve(tmp_bytes + 256));
  k_pcl_centroids<<<(n + 127) / 128, 128, 0, st>>>(M.keys.p, M.sorted.p, M.geom.p, M.cent.p, M.bkey.p, M.bpos_in.p, n);
  size_t tb = B->sort_tmp.cap;
  B2R_CUDA(cub::DeviceRadixSort::SortPairs(B->sort_tmp.p, tb, M.bkey.p, M.bkey_sorted.p, M.bpos_in.p, M.bpos.p, n, 0, kPclBucketBits, st));
  k_pcl_buckets<<<(n + 127) / 128, 128, 0, st>>>(M.bkey_sorted.p, M.btab_key.p, M.btab_val.p, M.bmask, n);
  return B2R_OK;
}

// the pass's inputs for a PCL target (M's geometry must be on the host: ndt_sync_geom)
inline void ndt_pcl_fill_args(const b2r_config& cfg, const Cloud& tgt, const NdtArgs& A, NdtPclArgs& P) {
  const NdtVoxelMap& M = *tgt.ndt;
  const VoxGeom& V = M.h_geom;
  P.A = A;
  P.cent = M.cent.p; P.bpos = M.bpos.p; P.btab_key = M.btab_key.p; P.btab_val = M.btab_val.p; P.bmask = M.bmask;
  for (int d = 0; d < 3; d++) { P.blo[d] = V.min_b[d] - 1; P.bhi[d] = V.max_b[d] + 1; }
  P.bdim0 = (unsigned long long)(V.div_b[0] + 2);
  P.bdim01 = P.bdim0 * (unsigned long long)(V.div_b[1] + 2);
  P.r2 = (float)(cfg.ndt_resolution * cfg.ndt_resolution);
  P.r_margin = 1.0001 * cfg.ndt_resolution;
}

// b2r_ndt_get_centroids: (leaf key, centroid) of every emitted leaf, keys ascending
inline int ndt_pcl_dump_centroids(Cloud& c, NdtWork& W, cudaStream_t st, size_t capacity, size_t* n_out, int64_t* keys, float* xyz) {
  NdtVoxelMap& M = *c.ndt;
  int rc = ndt_sync_geom(M, W, st);
  if (rc) return rc;
  std::vector<unsigned int> ks(M.n + 1);
  std::vector<unsigned long long> bk(M.n + 1);
  std::vector<float4> ce(M.n + 1);
  if (M.n) {
    B2R_CUDA(cudaMemcpyAsync(ks.data(), M.keys.p, M.n * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    B2R_CUDA(cudaMemcpyAsync(bk.data(), M.bkey.p, M.n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    B2R_CUDA(cudaMemcpyAsync(ce.data(), M.cent.p, M.n * sizeof(float4), cudaMemcpyDeviceToHost, st));
  }
  B2R_CUDA(cudaStreamSynchronize(st));
  size_t k = 0;
  for (size_t s = 0; s < M.n; s++) {
    if (bk[s] == kPclNoBucket) continue;
    if (k < capacity) {
      if (keys) keys[k] = (int64_t)ks[s];
      if (xyz) { xyz[3 * k] = ce[s].x; xyz[3 * k + 1] = ce[s].y; xyz[3 * k + 2] = ce[s].z; }
    }
    k++;
  }
  *n_out = k;
  return B2R_OK;
}

}  // namespace b2r
