// gicp.cuh — GICP kernels: k-NN covariances, and the block / grid reductions shared by every reducing kernel.
//
// Re-creates, GPU-first, the arithmetic of fast_gicp::FastGICP (SURVEY.md A.4) that the reference selects at
// /root/reference/src/hdl_graph_slam/registrations.cpp:27-36 and runs from apps/scan_matching_odometry_nodelet.cpp:177,210
// and include/hdl_graph_slam/loop_detector.hpp:136,143:
//   k_knn_cov_reg<20>  <- FastGICP::calculate_covariances (k = 20 exact NN in registers, PLANE regularisation); k_knn_cov: any k
//   (update_correspondences / linearize / compute_error and the LM loop live in pair_engine.cuh: k_pair_search, k_pair_accumulate)
// All per-cloud arrays live in the BVH's sorted order (Hilbert key, then original index), so consecutive threads hold spatial
// neighbours; block partials are combined in a fixed order => bitwise reproducible results.
#pragma once
#include "common.cuh"
#include "bvh.cuh"
#include "linalg.cuh"

namespace b2r {

constexpr int kKnnThreads = 128;
// resident blocks per SM: the single-cloud kernel is bound by its slowest warp (4 blocks, 104 registers, no spills); the batched one by
// throughput (5 blocks, 96 registers: faster on the k-NN share of the loop batch; the same setting slows the odometry chain)
#ifndef B2R_KNN_MINBLOCKS
#define B2R_KNN_MINBLOCKS 4
#endif
#ifndef B2R_KNN_BATCH_MINBLOCKS
#define B2R_KNN_BATCH_MINBLOCKS 5
#endif
constexpr int kLinThreads = 128;
#ifndef B2R_ACC_THREADS
#define B2R_ACC_THREADS 256
#endif
constexpr int kAccThreads = B2R_ACC_THREADS;  // k_gicp_accumulate: ~126 registers per thread; 256 rows of partials for the final reduction
constexpr int kAcc = 29;  // 21 (upper H) + 6 (b) + 1 (cost) + 1 (trial cost at this pose with the PREVIOUS correspondences)

// ---------------------------------------------------------------- k-NN covariance
// per-lane sorted top-k of packed 64-bit keys in shared memory, slot-major ([k][blockDim]); the k-th key is cached in a
// register so the all-pairs tile loop costs one 64-bit compare per candidate.
struct KnnList {
  static constexpr int kTileLanes = 3;   // coop mode only when 1-2 lanes want the leaf (each pick costs an insertion)
  static constexpr int kTileUnroll = 2;  // the insertion loop is big: keep the instruction footprint small (i-cache)
  static constexpr bool kTwoPhase = true;
  unsigned long long* key;
  int k, cnt, stride;
  unsigned long long wkey;  // key[k-1] once the list is full, else kKeyInf
#ifdef B2R_KNN_PROFILE
  int n_test = 0, n_ins = 0, n_shift = 0, n_tile = 0, n_coop = 0, n_try = 0;
#endif
  __device__ __forceinline__ float worst() const { return nn_key_d2(wkey); }
  __device__ __forceinline__ float limit() const { return INFINITY; }
  __device__ __forceinline__ void visit(float d2, int idx, int) {
    const unsigned long long kq = nn_key(d2, idx);
#ifdef B2R_KNN_PROFILE
    n_test++;
#endif
    if (kq >= wkey) return;
#ifdef B2R_KNN_PROFILE
    n_ins++;
#endif
    int j = (cnt < k) ? cnt++ : k - 1;
    while (j > 0) {
      const unsigned long long prev = key[(j - 1) * stride];
      if (prev <= kq) break;
      key[j * stride] = prev;
      j--;
#ifdef B2R_KNN_PROFILE
      n_shift++;
#endif
    }
    key[j * stride] = kq;
    if (cnt == k) wkey = key[(k - 1) * stride];
  }
};

// mean / covariance over the neighbours in ascending (d2, index) order (float64), PLANE regularisation, store 6 doubles.
// pt_at(j) returns the j-th neighbour's coordinates.
template <class PtAt>
__device__ __forceinline__ void knn_cov_store(int kk, PtAt pt_at, double* __restrict__ o) {
  double mx = 0, my = 0, mz = 0;
  for (int j = 0; j < kk; j++) {
    const float3 p = pt_at(j);
    mx += (double)p.x; my += (double)p.y; mz += (double)p.z;
  }
  const double inv = 1.0 / (double)kk;
  mx *= inv; my *= inv; mz *= inv;
  double c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int j = 0; j < kk; j++) {
    const float3 p = pt_at(j);
    double vx = (double)p.x - mx, vy = (double)p.y - my, vz = (double)p.z - mz;
    c[0] += vx * vx; c[1] += vx * vy; c[2] += vx * vz;
    c[4] += vy * vy; c[5] += vy * vz; c[8] += vz * vz;
  }
  c[0] *= inv; c[1] *= inv; c[2] *= inv; c[4] *= inv; c[5] *= inv; c[8] *= inv;
  c[3] = c[1]; c[6] = c[2]; c[7] = c[5];
  // PLANE regularisation: singular values (descending) replaced by (1, 1, 1e-3).  With orthonormal eigenvectors
  // v0 (smallest), v1, v2:  1*v2 v2^T + 1*v1 v1^T + 1e-3*v0 v0^T  ==  I - (1 - 1e-3) v0 v0^T : only the normal is needed.
  double n[3];
  sym_min_eigvec3(c, n);
  const double w = 1.0 - 1e-3;
  o[0] = 1.0 - w * n[0] * n[0];
  o[1] = -w * n[0] * n[1];
  o[2] = -w * n[0] * n[2];
  o[3] = 1.0 - w * n[1] * n[1];
  o[4] = -w * n[1] * n[2];
  o[5] = 1.0 - w * n[2] * n[2];
}

// one warp per leaf (4 leaves per block): its 32 points are the queries; per-lane top-k lists in shared memory
__global__ void __launch_bounds__(kKnnThreads, 4) k_knn_cov(Bvh b, int k, const float* __restrict__ raw, int stride_f, double* __restrict__ cov,
                                                            long long* prof) {
  extern __shared__ unsigned long long knn_keys[];  // [k][blockDim]
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int leaf = s >> 5;
  if (leaf >= b.nleaf) return;  // whole warps only (blockDim is a multiple of 32)
  const float4 q = b.sp[s];
  const bool active = idx_bits(q.w) != kPadIdx;
  KnnList L;
  L.key = knn_keys + threadIdx.x;
  L.k = k;
  L.cnt = 0;
  L.stride = blockDim.x;
  L.wkey = kKeyInf;
#ifdef B2R_KNN_PROFILE
  const long long t0 = clock64();
#endif
  bvh_group_search(b, q.x, q.y, q.z, active, L, leaf);
#ifdef B2R_KNN_PROFILE
  {
    const long long t1 = clock64();
    const unsigned F = 0xffffffffu;
    int v[6] = {L.n_test, L.n_ins, L.n_shift, L.n_ins, L.n_shift, 0};
    for (int o = 16; o > 0; o >>= 1) {
      v[0] += __shfl_xor_sync(F, v[0], o); v[1] += __shfl_xor_sync(F, v[1], o); v[2] += __shfl_xor_sync(F, v[2], o);
      v[3] = max(v[3], __shfl_xor_sync(F, v[3], o)); v[4] = max(v[4], __shfl_xor_sync(F, v[4], o));
    }
    const int ntile = __shfl_sync(F, L.n_tile, 0), ncoop = __shfl_sync(F, L.n_coop, 0);
    if ((threadIdx.x & 31) == 0) {
      long long* o = prof + (size_t)leaf * 8;
      o[0] = t1 - t0; o[1] = ntile; o[2] = ncoop; o[3] = v[0]; o[4] = v[1]; o[5] = v[2]; o[6] = v[3]; o[7] = v[4];
    }
  }
#endif
  if (!active) return;
  const int stride = L.stride;
  const unsigned long long* keyp = L.key;
  knn_cov_store(L.cnt, [=](int j) {
    const int idx = (int)(unsigned int)(keyp[j * stride] & 0xffffffffull);
    const float* p = raw + (size_t)idx * stride_f;
    return make_float3(p[0], p[1], p[2]);
  }, cov + (size_t)s * 6);
}

// ---- register-resident lists (K fixed at compile time).  With the lists in shared memory a warp spends hundreds of
// cycles per candidate step, the latency of a data-dependent LDS -> compare -> STS chain (max over lanes of the shift count);
// in registers every slot is recomputed branch-free from the OLD neighbours (new[j] = old[j-1] > q ? old[j-1] : old[j] > q ? q :
// old[j]), so the K slot updates are independent instructions.  Same candidates, same (d2, idx) order => identical lists.
template <int K>
struct KnnRegs {
  static constexpr int kTileLanes = 3;
  static constexpr int kTileUnroll = 1;
  static constexpr bool kTwoPhase = true;
  unsigned long long key[K];
#ifdef B2R_KNN_PROFILE
  int n_test = 0, n_ins = 0, n_shift = 0, n_tile = 0, n_coop = 0, n_try = 0;
#endif
  __device__ __forceinline__ void reset() {
#pragma unroll
    for (int j = 0; j < K; j++) key[j] = kKeyInf;
  }
  __device__ __forceinline__ float worst() const { return nn_key_d2(key[K - 1]); }
  __device__ __forceinline__ float limit() const { return INFINITY; }
  __device__ __forceinline__ void visit(float d2, int idx, int) {
    const unsigned long long kq = nn_key(d2, idx);
#ifdef B2R_KNN_PROFILE
    n_test++;
#endif
    if (kq >= key[K - 1]) return;  // also rejects padding (kq == kKeyInf)
#ifdef B2R_KNN_PROFILE
    n_ins++;
#endif
    if constexpr (K == 20) {
      insert20(kq);
    } else {
      bool pj = true;  // p_j = old key[j] > kq, monotone in j; p_{K-1} holds (tested above)
#pragma unroll
      for (int j = K - 1; j > 0; j--) {  // descending: key[j-1] is still the old value when slot j is rewritten
        const unsigned long long lo = key[j - 1];
        const bool pl = lo > kq;
        if (pj) key[j] = pl ? lo : kq;   // slot j changes only if p_j: takes its left neighbour, or the new key at the boundary
        pj = pl;
      }
      if (pj) key[0] = kq;
    }
  }
  // The same network for K = 20 written out in PTX.  From the C++ loop above ptxas evaluates every 64-bit compare TWICE (once as
  // the guard of slot j, once as the selector of slot j + 1: 4 ISETP + 2 SEL per slot, 118 instructions per insertion); here each
  // compare is one setp.u64 whose predicate serves both uses: 2 ISETP + 2 SEL per slot, 80 instructions.  Same decisions, same list.
  __device__ __forceinline__ void insert20(unsigned long long kq) {
#ifdef __CUDA_ARCH__
    asm("{\n\t.reg .pred pa, pb;\n\t"
        "setp.gt.u64 pa, %18, %20;\n\t selp.b64 %19, %18, %20, pa;\n\t"
        "setp.gt.u64 pb, %17, %20;\n\t @pa selp.b64 %18, %17, %20, pb;\n\t"
        "setp.gt.u64 pa, %16, %20;\n\t @pb selp.b64 %17, %16, %20, pa;\n\t"
        "setp.gt.u64 pb, %15, %20;\n\t @pa selp.b64 %16, %15, %20, pb;\n\t"
        "setp.gt.u64 pa, %14, %20;\n\t @pb selp.b64 %15, %14, %20, pa;\n\t"
        "setp.gt.u64 pb, %13, %20;\n\t @pa selp.b64 %14, %13, %20, pb;\n\t"
        "setp.gt.u64 pa, %12, %20;\n\t @pb selp.b64 %13, %12, %20, pa;\n\t"
        "setp.gt.u64 pb, %11, %20;\n\t @pa selp.b64 %12, %11, %20, pb;\n\t"
        "setp.gt.u64 pa, %10, %20;\n\t @pb selp.b64 %11, %10, %20, pa;\n\t"
        "setp.gt.u64 pb, %9, %20;\n\t @pa selp.b64 %10, %9, %20, pb;\n\t"
        "setp.gt.u64 pa, %8, %20;\n\t @pb selp.b64 %9, %8, %20, pa;\n\t"
        "setp.gt.u64 pb, %7, %20;\n\t @pa selp.b64 %8, %7, %20, pb;\n\t"
        "setp.gt.u64 pa, %6, %20;\n\t @pb selp.b64 %7, %6, %20, pa;\n\t"
        "setp.gt.u64 pb, %5, %20;\n\t @pa selp.b64 %6, %5, %20, pb;\n\t"
        "setp.gt.u64 pa, %4, %20;\n\t @pb selp.b64 %5, %4, %20, pa;\n\t"
        "setp.gt.u64 pb, %3, %20;\n\t @pa selp.b64 %4, %3, %20, pb;\n\t"
        "setp.gt.u64 pa, %2, %20;\n\t @pb selp.b64 %3, %2, %20, pa;\n\t"
        "setp.gt.u64 pb, %1, %20;\n\t @pa selp.b64 %2, %1, %20, pb;\n\t"
        "setp.gt.u64 pa, %0, %20;\n\t @pb selp.b64 %1, %0, %20, pa;\n\t"
        "@pa mov.b64 %0, %20;\n\t}"
        : "+l"(key[0]), "+l"(key[1]), "+l"(key[2]), "+l"(key[3]), "+l"(key[4]), "+l"(key[5]), "+l"(key[6]), "+l"(key[7]), "+l"(key[8]),
          "+l"(key[9]), "+l"(key[10]), "+l"(key[11]), "+l"(key[12]), "+l"(key[13]), "+l"(key[14]), "+l"(key[15]), "+l"(key[16]),
          "+l"(key[17]), "+l"(key[18]), "+l"(key[19])
        : "l"(kq));
#endif
  }
  __device__ __forceinline__ int count() const {
    int c = 0;
#pragma unroll
    for (int j = 0; j < K; j++) c += key[j] != kKeyInf;
    return c;
  }
};

constexpr int kKnnRegK = 20;

template <int K>
__device__ __forceinline__ void knn_cov_reg_body(const Bvh& b, const float* __restrict__ raw, int stride_f, double* __restrict__ cov, int block_x, int (*nbr)[kKnnThreads],
                                                 long long* prof) {
  const int s = block_x * blockDim.x + threadIdx.x;
  const int leaf = s >> 5;
  if (leaf >= b.nleaf) return;  // whole warps only
  const float4 q = b.sp[s];
  const bool active = idx_bits(q.w) != kPadIdx;
  KnnRegs<K> L;
  L.reset();
#ifdef B2R_KNN_PROFILE
  const long long t0 = clock64();
#endif
  bvh_group_search(b, q.x, q.y, q.z, active, L, leaf);
#ifdef B2R_KNN_PROFILE
  {
    const long long t1 = clock64();
    const unsigned F = 0xffffffffu;
    int v[4] = {L.n_test, L.n_ins, L.n_ins, 0};
    for (int o = 16; o > 0; o >>= 1) {
      v[0] += __shfl_xor_sync(F, v[0], o); v[1] += __shfl_xor_sync(F, v[1], o);
      v[2] = max(v[2], __shfl_xor_sync(F, v[2], o));
    }
    const int ntile = __shfl_sync(F, L.n_tile, 0), ncoop = __shfl_sync(F, L.n_coop, 0);
    if ((threadIdx.x & 31) == 0 && prof) {
      long long* o = prof + (size_t)leaf * 8;
      o[0] = t1 - t0; o[1] = ntile; o[2] = ncoop; o[3] = v[0]; o[4] = v[1]; o[5] = 0; o[6] = v[2]; o[7] = 0;
    }
  }
#endif
  if (!active) return;
#pragma unroll
  for (int j = 0; j < K; j++) nbr[j][threadIdx.x] = (int)(unsigned int)(L.key[j] & 0xffffffffull);
  const int tx = threadIdx.x;
  knn_cov_store(L.count(), [&](int j) {
    const float* p = raw + (size_t)nbr[j][tx] * stride_f;
    return make_float3(p[0], p[1], p[2]);
  }, cov + (size_t)s * 6);
}

template <int K>
__global__ void __launch_bounds__(kKnnThreads, B2R_KNN_MINBLOCKS) k_knn_cov_reg(Bvh b, const float* __restrict__ raw, int stride_f, double* __restrict__ cov,
                                                                long long* prof) {
  __shared__ int nbr[K][kKnnThreads];  // neighbour indices, ascending (d2, idx), for the covariance pass
  knn_cov_reg_body<K>(b, raw, stride_f, cov, blockIdx.x, nbr, prof);
}

// the same for MANY clouds in one launch (blockIdx.y = cloud): the batched path registers a whole set of keyframe clouds at once,
// and one cloud alone fills less than a wave (0.86) with a 3x tail — together the clouds keep every SM busy
struct KnnBatchItem {
  Bvh b;
  const float* raw;
  double* cov;
  int stride_f;
  int pad;
};
template <int K>
__global__ void __launch_bounds__(kKnnThreads, B2R_KNN_BATCH_MINBLOCKS) k_knn_cov_reg_batch(const KnnBatchItem* __restrict__ items) {
  __shared__ int nbr[K][kKnnThreads];
  const KnnBatchItem it = items[blockIdx.y];
  knn_cov_reg_body<K>(it.b, it.raw, it.stride_f, it.cov, blockIdx.x, nbr, nullptr);
}

// deterministic block reduction of NV doubles per thread; result valid in thread 0
template <int NV>
__device__ __forceinline__ void block_reduce(double* v, double* smem /* NV * 32 */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; i++) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; i++) smem[i * 32 + warp] = v[i];
  }
  __syncthreads();
  if (threadIdx.x < 32) {
#pragma unroll
    for (int i = 0; i < NV; i++) {
      double x = (lane < nw) ? smem[i * 32 + lane] : 0.0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
      v[i] = x;
    }
  }
}

// last-block-done final reduction: partials [gridDim][NV] -> out[NV], summed in a fixed order.
// `out` may live in host-mapped pinned memory: the result then lands in host memory straight from the kernel together with a
// checksum word (out[NV+1]; out[NV] carries `extra` or is unused) and `flag` = `seq`, so the host can spin on it instead of paying a
// memcpy + stream sync.
// finish_stored: thread 0 of every block has already written the block's NV sums to partials[blockIdx.x][0..NV)
template <int NV>
__device__ __forceinline__ void finish_stored(double* partials, double* out, unsigned int* counter, unsigned long long* flag = nullptr,
                                              unsigned long long seq = 0, unsigned long long* extra = nullptr);

template <int NV>
__device__ __forceinline__ void finish_partials(const double* v, double* partials, double* out, unsigned int* counter,
                                                unsigned long long* flag = nullptr, unsigned long long seq = 0,
                                                unsigned long long* extra = nullptr) {
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < NV; i++) partials[(size_t)blockIdx.x * NV + i] = v[i];
  }
  finish_stored<NV>(partials, out, counter, flag, seq, extra);
}

template <int NV>
__device__ __forceinline__ void finish_stored(double* partials, double* out, unsigned int* counter, unsigned long long* flag,
                                              unsigned long long seq, unsigned long long* extra) {
  __shared__ bool is_last;
  if (threadIdx.x == 0) {
    __threadfence();
    unsigned int t = atomicAdd(counter, 1u);
    is_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    // fixed-order parallel sum: warp w adds rows w, w+nw, ... (lane = value: one coalesced row per load, 8 loads in flight,
    // ld.cg: the rows were written by other SMs during this launch), then thread i adds the per-warp sums in warp order.
    // The order depends only on the launch geometry => run-to-run bitwise reproducible.
    __shared__ double fin[8 * NV];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nw = (blockDim.x >> 5) < 8 ? (int)(blockDim.x >> 5) : 8;
    const unsigned int nrow = gridDim.x;
    if (warp < nw) {
      for (int i = lane; i < NV; i += 32) {
        double s = 0.0;
        unsigned int r = warp;
        for (; r + 7 * nw < nrow; r += 8 * nw) {
          double t[8];
#pragma unroll
          for (int u = 0; u < 8; u++) t[u] = __ldcg(partials + (size_t)(r + u * nw) * NV + i);
#pragma unroll
          for (int u = 0; u < 8; u++) s += t[u];
        }
        for (; r < nrow; r += nw) s += __ldcg(partials + (size_t)r * NV + i);
        fin[warp * NV + i] = s;
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < NV; i += blockDim.x) {
      double s = 0.0;
      for (int w = 0; w < nw; w++) s += fin[w * NV + i];
      out[i] = s;
      fin[i] = s;  // column i of `fin` is read by this thread only: slot [0][i] is free again and carries the value to thread 0
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      *counter = 0;
      unsigned long long x = seq;
      if (extra) {
        const unsigned long long e = *reinterpret_cast<volatile unsigned long long*>(extra);
        *extra = 0;  // device-side counter accumulated with atomics during this launch: read once, re-armed for the next launch
        reinterpret_cast<unsigned long long*>(out)[NV] = e;
        x ^= msg_mix(e, NV);
      }
      if (flag) {
        // Publication without system-scope fences (each costs a PCIe round trip): the host accepts the result words only when
        // flag == seq AND the checksum word equals seq ^ xor(result words), so the order in which these stores land in host memory
        // does not matter (wait_host_result re-reads until the message is self-consistent).
        for (int i = 0; i < NV; i++) x ^= msg_mix((unsigned long long)__double_as_longlong(fin[i]), i);
        reinterpret_cast<unsigned long long*>(out)[NV + 1] = x;
        *reinterpret_cast<volatile unsigned long long*>(flag) = seq;
      }
    }
  }
}

}  // namespace b2r
