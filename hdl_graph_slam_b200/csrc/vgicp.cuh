// vgicp.cuh — fast_gicp::FastVGICP on the device (B2R_METHOD_VGICP): the target's Gaussian voxel map and the VGICP round.
//
// Semantics (tests/vgicp_ref.cpp is the sequential statement the tests hold this file to):
//   * voxel map (GaussianVoxelMap::create_voxelmap, voxel mode ADDITIVE) of the TARGET: cell = (int)floor((double)p / resolution) per
//     axis (a float64 division); points appended in ascending point index: num_points++, mean += (x, y, z), cov += C_i (the point's
//     PLANE covariance, k_knn_cov*); finalize: mean /= num_points, cov /= num_points.  A one-point voxel is valid.
//     A point with a non-finite coordinate is dropped (it has no covariance either).  Keys hold 21 bits per axis: a finite point
//     whose cell lies outside [-2^20, 2^20) fails the build with B2R_EUNSUPPORTED (never a silently wrong map).
//   * update_correspondences (DIRECT1): t = T (x, y, z, 1) in float64 as ((r0 x + r1 y) + r2 z) + t0, unfused; the correspondence is
//     the voxel of cell floor(t / resolution), or none; M = (cov_B + R cov_A R^T)^-1 in GICP's operation order.
//   * linearize / compute_error: w = sqrt(num_points), e = mean_B - T mean_A, cost += w e^T M e, H += w J^T M J, b += w J^T M e,
//     J = [skew(T mean_A) | -I].  compute_error reuses the correspondences and M of the linearisation point.
//
// Device layout: the map is built from the cloud's BVH arrays (sorted points + pos_of) and its covariances, so it needs neither the
// caller's records nor a copy of them: a promoted source (odometry keyframe) gets its map from what it already holds.  The build is
// templated on the cell and accumulation rule: FastVGICP's VgicpMapRule below, FastVGICPCuda's float32 VcudaMapRule (vgicp_cuda.cuh).
// One VGICP round = k_vgicp_round (probe, M, trial cost of the previous set, weighted linearisation; the 29 block partials of
// k_pair_accumulate's layout) + the unchanged k_pair_lm.  Pair records (PairDev) are the GICP engine's; the map travels beside them.
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>
#include "engine.cuh"
#include "pair_engine.cuh"
#include "fitness.cuh"

namespace b2r {

constexpr int kVgicpAxisBits = 21;
constexpr long long kVgicpBias = 1ll << (kVgicpAxisBits - 1);  // cells in [-2^20, 2^20) per axis
constexpr unsigned long long kVgicpNone = ~0ull;                // dropped point / empty table slot

// what a VGICP round reads of a target's voxel map
struct VgicpMapDev {
  const unsigned long long* tkeys;  // open-addressing table: cell key or kVgicpNone
  const int* tvals;                 // voxel index of the slot
  const double* mean;               // 3 per voxel
  const double* cov;                // 6 per voxel: xx xy xz yy yz zz
  const int* count;                 // num_points per voxel
  double res;
  unsigned int mask;                // table capacity - 1
  int nvox;
};

struct VgicpMap {
  DevBuf<unsigned long long> keys_a, keys_b, ukeys, tkeys;
  DevBuf<int> vals_a, vals_b, counts, offs, tvals, misc;  // misc: [0] extent violations, [1] dropped points, [2] runs
  DevBuf<double> mean, cov;
  DevBuf<int> count;
  DevBuf<char> tmp;
  PinnedBuf<int> h_misc;
  DevBuf<VgicpMapDev> d_desc;  // the descriptor below, on the device (single-pair rounds read it from here)
  VgicpMapDev desc{};
  int nvox = 0;
};

// the key of the cell (fx, fy, fz) (whole numbers), false outside the 21-bit range per axis or for a NaN
__device__ __forceinline__ bool vgicp_key(double fx, double fy, double fz, unsigned long long* key) {
  const double lo = -(double)kVgicpBias, hi = (double)kVgicpBias;
  if (!(fx >= lo && fx < hi && fy >= lo && fy < hi && fz >= lo && fz < hi)) return false;  // also every NaN
  *key = ((unsigned long long)((long long)fx + kVgicpBias) << (2 * kVgicpAxisBits)) |
         ((unsigned long long)((long long)fy + kVgicpBias) << kVgicpAxisBits) | (unsigned long long)((long long)fz + kVgicpBias);
  return true;
}

__device__ __forceinline__ bool vgicp_cell(double x, double y, double z, double res, unsigned long long* key) {
  return vgicp_key(floor(x / res), floor(y / res), floor(z / res), key);
}

// The map's cell and accumulation rule.  This one is FastVGICP's: float64 cells floor(p / res) and float64 sums; FastVGICPCuda's
// float32 rule is VcudaMapRule (vgicp_cuda.cuh).  Both store the finalised means and covariances as doubles.
struct VgicpMapRule {
  using Acc = double;
  __device__ __forceinline__ static bool cell(float x, float y, float z, double res, unsigned long long* key) {
    return vgicp_cell((double)x, (double)y, (double)z, res, key);
  }
  __device__ __forceinline__ static double add(double a, double b) { return dadd(a, b); }
  __device__ __forceinline__ static double div(double a, int n) { return __ddiv_rn(a, (double)n); }
};

__device__ __forceinline__ unsigned int vgicp_hash(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (unsigned int)k;
}

// one key per point in ascending point index (the radix sort below is stable, so a voxel's points stay in index order)
template <class Rule>
__global__ void k_vgicp_keys(const float4* __restrict__ sorted, const int* __restrict__ pos_of, int n, double res, unsigned long long* keys,
                             int* vals, int* misc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  vals[i] = i;
  unsigned long long key = kVgicpNone;
  const int j = pos_of[i];
  if (j >= 0) {  // in the search structure = a finite point
    const float4 p = sorted[j];
    if (!Rule::cell(p.x, p.y, p.z, res, &key)) { key = kVgicpNone; atomicAdd(misc + 0, 1); }
  } else {
    atomicAdd(misc + 1, 1);
  }
  keys[i] = key;
}

// one thread per voxel: sums in point-index order, finalize, table insert
template <class Rule>
__global__ void k_vgicp_voxels(const float4* __restrict__ sorted, const int* __restrict__ pos_of, const double* __restrict__ pcov,
                               const unsigned long long* __restrict__ ukeys, const int* __restrict__ counts, const int* __restrict__ offs,
                               const int* __restrict__ idx, int nvox, double* mean, double* cov, int* count, unsigned long long* tkeys,
                               int* tvals, unsigned int mask) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nvox) return;
  const int c = counts[v], o = offs[v];
  using Acc = typename Rule::Acc;
  Acc m[3] = {0, 0, 0}, s[6] = {0, 0, 0, 0, 0, 0};
  for (int k = 0; k < c; k++) {
    const int j = pos_of[idx[o + k]];
    const float4 p = sorted[j];
    m[0] = Rule::add(m[0], (Acc)p.x); m[1] = Rule::add(m[1], (Acc)p.y); m[2] = Rule::add(m[2], (Acc)p.z);
    const double* ci = pcov + (size_t)j * 6;
#pragma unroll
    for (int q = 0; q < 6; q++) s[q] = Rule::add(s[q], (Acc)ci[q]);
  }
#pragma unroll
  for (int q = 0; q < 3; q++) mean[(size_t)v * 3 + q] = (double)Rule::div(m[q], c);
#pragma unroll
  for (int q = 0; q < 6; q++) cov[(size_t)v * 6 + q] = (double)Rule::div(s[q], c);
  count[v] = c;
  const unsigned long long key = ukeys[v];
  unsigned int h = vgicp_hash(key) & mask;
  for (;;) {
    const unsigned long long old = atomicCAS(tkeys + h, kVgicpNone, key);
    if (old == kVgicpNone) { tvals[h] = v; break; }
    h = (h + 1) & mask;
  }
}

__device__ __forceinline__ int vgicp_probe(const VgicpMapDev& M, unsigned long long key) {
  unsigned int h = vgicp_hash(key) & M.mask;
  for (;;) {
    const unsigned long long k = __ldg(M.tkeys + h);
    if (k == key) return __ldg(M.tvals + h);
    if (k == kVgicpNone) return -1;
    h = (h + 1) & M.mask;
  }
}

// Builds (or keeps) the voxel map of cloud `c` at `res` under `Rule`: needs c's BVH and covariances.  Synchronises `st` once (extent
// check, voxel count).  B2R_EUNSUPPORTED when a finite point lies beyond the 21-bit key range.
template <class Rule>
inline int vgicp_build_map(Cloud& c, double res, Telemetry* tel, cudaStream_t st) {
  if (!c.vgicp) c.vgicp.reset(new VgicpMap());
  VgicpMap& M = *c.vgicp;
  const int n = (int)c.n;
  B2R_CUDA(M.misc.reserve(4));
  if (!M.h_misc.p) B2R_CUDA(M.h_misc.alloc(4));
  B2R_CUDA(M.d_desc.reserve(1));
  B2R_CUDA(cudaMemsetAsync(M.misc.p, 0, 4 * sizeof(int), st));
  M.nvox = 0;
  if (n > 0) {
    B2R_CUDA(M.keys_a.reserve(n)); B2R_CUDA(M.keys_b.reserve(n)); B2R_CUDA(M.ukeys.reserve(n));
    B2R_CUDA(M.vals_a.reserve(n)); B2R_CUDA(M.vals_b.reserve(n)); B2R_CUDA(M.counts.reserve(n)); B2R_CUDA(M.offs.reserve(n));
    size_t b_sort = 0, b_rle = 0, b_scan = 0;
    B2R_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b_sort, M.keys_a.p, M.keys_b.p, M.vals_a.p, M.vals_b.p, n, 0, 64, st));
    B2R_CUDA(cub::DeviceRunLengthEncode::Encode(nullptr, b_rle, M.keys_b.p, M.ukeys.p, M.counts.p, M.misc.p + 2, n, st));
    B2R_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b_scan, M.counts.p, M.offs.p, n, st));
    B2R_CUDA(M.tmp.reserve(std::max(b_sort, std::max(b_rle, b_scan)) + 256));
    TEL_BEGIN(tel, st);
    k_vgicp_keys<Rule><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c.sorted.p, c.pos_of.p, n, res, M.keys_a.p, M.vals_a.p, M.misc.p);
    size_t tb = M.tmp.cap;
    B2R_CUDA(cub::DeviceRadixSort::SortPairs(M.tmp.p, tb, M.keys_a.p, M.keys_b.p, M.vals_a.p, M.vals_b.p, n, 0, 64, st));
    tb = M.tmp.cap;
    B2R_CUDA(cub::DeviceRunLengthEncode::Encode(M.tmp.p, tb, M.keys_b.p, M.ukeys.p, M.counts.p, M.misc.p + 2, n, st));
    tb = M.tmp.cap;
    B2R_CUDA(cub::DeviceScan::ExclusiveSum(M.tmp.p, tb, M.counts.p, M.offs.p, n, st));
    TEL_END(tel, KC_VGICP_MAP, 4, st);
    B2R_CUDA(cudaGetLastError());
    B2R_CUDA(cudaMemcpyAsync(M.h_misc.p, M.misc.p, 3 * sizeof(int), cudaMemcpyDeviceToHost, st));
    B2R_CUDA(cudaStreamSynchronize(st));
    if (tel) tel->d2h += 3 * sizeof(int);
    if (M.h_misc.p[0] > 0)
      return fail(B2R_EUNSUPPORTED, "VGICP voxel map: " + std::to_string(M.h_misc.p[0]) +
                                        " point(s) lie beyond the 21-bit cell range per axis (|p| / resolution >= 2^20)");
    // dropped points sort behind every cell under the key kVgicpNone: their run is not a voxel
    M.nvox = M.h_misc.p[2] - (M.h_misc.p[1] > 0 ? 1 : 0);
  }
  unsigned int cap = 16;
  while (cap < 2u * (unsigned)M.nvox) cap <<= 1;
  B2R_CUDA(M.tkeys.reserve(cap)); B2R_CUDA(M.tvals.reserve(cap));
  B2R_CUDA(M.mean.reserve((size_t)M.nvox * 3 + 3)); B2R_CUDA(M.cov.reserve((size_t)M.nvox * 6 + 6)); B2R_CUDA(M.count.reserve(M.nvox + 1));
  B2R_CUDA(cudaMemsetAsync(M.tkeys.p, 0xff, cap * sizeof(unsigned long long), st));
  if (M.nvox > 0) {
    TEL_BEGIN(tel, st);
    k_vgicp_voxels<Rule><<<(unsigned)((M.nvox + 127) / 128), 128, 0, st>>>(c.sorted.p, c.pos_of.p, c.cov.p, M.ukeys.p, M.counts.p, M.offs.p, M.vals_b.p,
                                                                     M.nvox, M.mean.p, M.cov.p, M.count.p, M.tkeys.p, M.tvals.p, cap - 1);
    TEL_END(tel, KC_VGICP_MAP, 1, st);
    B2R_CUDA(cudaGetLastError());
  }
  M.desc.tkeys = M.tkeys.p; M.desc.tvals = M.tvals.p; M.desc.mean = M.mean.p; M.desc.cov = M.cov.p; M.desc.count = M.count.p;
  M.desc.res = res; M.desc.mask = cap - 1; M.desc.nvox = M.nvox;
  B2R_CUDA(cudaMemcpyAsync(M.d_desc.p, &M.desc, sizeof(VgicpMapDev), cudaMemcpyHostToDevice, st));
  B2R_CUDA(cudaStreamSynchronize(st));  // M.desc is the source of the copy above
  c.vgicp_ready = true;
  return B2R_OK;
}

// voxels of a built map, cells ascending (keys unpacked to cells): arrays may be NULL
inline int vgicp_dump(Cloud& c, cudaStream_t st, size_t capacity, size_t* n_vox, int32_t* cells, int32_t* counts, double* mean, double* cov) {
  VgicpMap& M = *c.vgicp;
  *n_vox = (size_t)M.nvox;
  const size_t k = std::min(capacity, (size_t)M.nvox);
  if (k == 0) return B2R_OK;
  std::vector<unsigned long long> keys(k);
  std::vector<int> cnt(k);
  std::vector<double> mu(k * 3), cv(k * 6);
  B2R_CUDA(cudaMemcpyAsync(keys.data(), M.ukeys.p, k * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaMemcpyAsync(cnt.data(), M.count.p, k * sizeof(int), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaMemcpyAsync(mu.data(), M.mean.p, k * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaMemcpyAsync(cv.data(), M.cov.p, k * 6 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2R_CUDA(cudaStreamSynchronize(st));
  const unsigned long long am = (1ull << kVgicpAxisBits) - 1;
  for (size_t v = 0; v < k; v++) {
    if (cells) {
      cells[v * 3 + 0] = (int32_t)((long long)((keys[v] >> (2 * kVgicpAxisBits)) & am) - kVgicpBias);
      cells[v * 3 + 1] = (int32_t)((long long)((keys[v] >> kVgicpAxisBits) & am) - kVgicpBias);
      cells[v * 3 + 2] = (int32_t)((long long)(keys[v] & am) - kVgicpBias);
    }
    if (counts) counts[v] = cnt[v];
    if (mean) for (int q = 0; q < 3; q++) mean[v * 3 + q] = mu[v * 3 + q];
    if (cov) {
      const double* s = &cv[v * 6];
      double* o = cov + v * 9;
      o[0] = s[0]; o[1] = s[1]; o[2] = s[2]; o[3] = s[1]; o[4] = s[3]; o[5] = s[4]; o[6] = s[2]; o[7] = s[4]; o[8] = s[5];
    }
  }
  return B2R_OK;
}

#ifdef __CUDACC__
// The VGICP round of every active pair: correspondence probe at xe (PM_FIRST / PM_FUSED) into the write set, M and the weighted
// linearisation, and compute_error at xe with the previous set (PM_FUSED / PM_ERR).  maps[k] belongs to pairs[k].  Block partials as
// k_pair_accumulate leaves them (29 values, transposed), so k_pair_lm takes the LM step unchanged.  The stored mahalanobis matrix is
// w M, so the trial cost is e^T (w M) e.  VGICP rounds never carry fitness sums: a caller that wants getFitnessScore runs k_fitness
// at the final pose (the kernel and reduction of b2r_fitness).
__global__ void __launch_bounds__(kAccThreads, B2R_ACC_MINBLOCKS) k_vgicp_round(PairDev* pairs, const int* __restrict__ active,
                                                                                const VgicpMapDev* __restrict__ maps) {
  __shared__ double red[kAcc * 8];
  __shared__ double tiles[(kAccThreads / 32) * 8 * kRedRow];
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (!active) asm volatile("griddepcontrol.launch_dependents;");
  if (active && (int)blockIdx.y >= active[0]) return;
  const int pi = active ? active[1 + blockIdx.y] : blockIdx.y;
  PairDev& p = pairs[pi];
  const int mode = p.mode;
  if (mode < PM_FIRST || mode > PM_ERR) return;
  const int nblk = p.nblk_acc;
  if ((int)blockIdx.x >= nblk) return;
  const VgicpMapDev M = maps[pi];
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* tile = tiles + warp * 8 * kRedRow;
  const int cur = p.cur;
  const int wset = (mode == PM_FIRST) ? cur : (cur ^ 1);
  float4 pt = make_float4(0.f, 0.f, 0.f, bits_idx(kPadIdx));
  if (s < p.src.nleaf * kLeaf) pt = p.src.sp[s];
  const bool is_point = idx_bits(pt.w) != kPadIdx;
  if (!is_point) { pt.x = 0.f; pt.y = 0.f; pt.z = 0.f; }
  const bool do_trial = (mode == PM_FUSED || mode == PM_ERR) && is_point;
  const bool do_lin = (mode == PM_FIRST || mode == PM_FUSED) && is_point;
  double T[12];
#pragma unroll
  for (int i = 0; i < 12; i++) T[i] = p.xe[i];
  const double ax = (double)pt.x, ay = (double)pt.y, az = (double)pt.z;
  const double tx = dadd(dadd(dadd(dmul(T[0], ax), dmul(T[1], ay)), dmul(T[2], az)), T[3]);
  const double ty = dadd(dadd(dadd(dmul(T[4], ax), dmul(T[5], ay)), dmul(T[6], az)), T[7]);
  const double tz = dadd(dadd(dadd(dmul(T[8], ax), dmul(T[9], ay)), dmul(T[10], az)), T[11]);
  // ---- compute_error at xe with the previous correspondences
  double trial = 0.0;
  if (do_trial) {
    const int v = p.cpos[cur][s];
    if (v >= 0) {
      const double* m = p.mahal[cur] + (size_t)s * 6;
      const double* mb = M.mean + (size_t)v * 3;
      const double ex = mb[0] - tx, ey = mb[1] - ty, ez = mb[2] - tz;
      const double Mex = m[0] * ex + m[1] * ey + m[2] * ez;
      const double Mey = m[1] * ex + m[3] * ey + m[4] * ez;
      const double Mez = m[2] * ex + m[4] * ey + m[5] * ez;
      trial = ex * Mex + ey * Mey + ez * Mez;
    }
  }
  // ---- update_correspondences (DIRECT1) + linearize
  double m00 = 0, m01 = 0, m02 = 0, m11 = 0, m12 = 0, m22 = 0, ex = 0, ey = 0, ez = 0;
  if (do_lin) {
    unsigned long long key;
    const int v = vgicp_cell(tx, ty, tz, M.res, &key) ? vgicp_probe(M, key) : -1;
    p.cpos[wset][s] = v;
    p.corr[wset][idx_bits(pt.w)] = v;
    if (v >= 0) {
      const double* ca = p.scov + (size_t)s * 6;
      const double* cb = M.cov + (size_t)v * 6;
      const double* mb = M.mean + (size_t)v * 3;
      const double CA[9] = {ca[0], ca[1], ca[2], ca[1], ca[3], ca[4], ca[2], ca[4], ca[5]};
      const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
      double tmp[9], rcr[9], Mi[9];
      mul3(R, CA, tmp);
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
      inv3(rcr, Mi);
      const double w = sqrt((double)M.count[v]);
      m00 = w * Mi[0]; m01 = w * Mi[1]; m02 = w * Mi[2]; m11 = w * Mi[4]; m12 = w * Mi[5]; m22 = w * Mi[8];
      double* mo = p.mahal[wset] + (size_t)s * 6;
      mo[0] = m00; mo[1] = m01; mo[2] = m02; mo[3] = m11; mo[4] = m12; mo[5] = m22;
      ex = mb[0] - tx; ey = mb[1] - ty; ez = mb[2] - tz;
    }
  }
  // a point without correspondence has M = 0, e = 0: every term below is an exact zero
  const double Mex = m00 * ex + m01 * ey + m02 * ez;
  const double Mey = m01 * ex + m11 * ey + m12 * ez;
  const double Mez = m02 * ex + m12 * ey + m22 * ez;
  const double ms00 = m01 * tz - m02 * ty, ms01 = -m00 * tz + m02 * tx, ms02 = m00 * ty - m01 * tx;
  const double ms10 = m11 * tz - m12 * ty, ms11 = -m01 * tz + m12 * tx, ms12 = m01 * ty - m11 * tx;
  const double ms20 = m12 * tz - m22 * ty, ms21 = -m02 * tz + m22 * tx, ms22 = m02 * ty - m12 * tx;
  red_emit<0, 28>(tz * ms10 - ty * ms20, tile, red, lane, warp);
  red_emit<1, 28>(tz * ms11 - ty * ms21, tile, red, lane, warp);
  red_emit<2, 28>(tz * ms12 - ty * ms22, tile, red, lane, warp);
  red_emit<3, 28>(-ms00, tile, red, lane, warp);
  red_emit<4, 28>(-ms10, tile, red, lane, warp);
  red_emit<5, 28>(-ms20, tile, red, lane, warp);
  red_emit<6, 28>(-tz * ms01 + tx * ms21, tile, red, lane, warp);
  red_emit<7, 28>(-tz * ms02 + tx * ms22, tile, red, lane, warp);
  red_emit<8, 28>(-ms01, tile, red, lane, warp);
  red_emit<9, 28>(-ms11, tile, red, lane, warp);
  red_emit<10, 28>(-ms21, tile, red, lane, warp);
  red_emit<11, 28>(ty * ms02 - tx * ms12, tile, red, lane, warp);
  red_emit<12, 28>(-ms02, tile, red, lane, warp);
  red_emit<13, 28>(-ms12, tile, red, lane, warp);
  red_emit<14, 28>(-ms22, tile, red, lane, warp);
  red_emit<15, 28>(m00, tile, red, lane, warp); red_emit<16, 28>(m01, tile, red, lane, warp); red_emit<17, 28>(m02, tile, red, lane, warp);
  red_emit<18, 28>(m11, tile, red, lane, warp); red_emit<19, 28>(m12, tile, red, lane, warp);
  red_emit<20, 28>(m22, tile, red, lane, warp);
  red_emit<21, 28>(tz * Mey - ty * Mez, tile, red, lane, warp);
  red_emit<22, 28>(-tz * Mex + tx * Mez, tile, red, lane, warp);
  red_emit<23, 28>(ty * Mex - tx * Mey, tile, red, lane, warp);
  red_emit<24, 28>(-Mex, tile, red, lane, warp); red_emit<25, 28>(-Mey, tile, red, lane, warp); red_emit<26, 28>(-Mez, tile, red, lane, warp);
  red_emit<27, 28>(ex * Mex + ey * Mey + ez * Mez, tile, red, lane, warp);
  red_emit<28, 28>(trial, tile, red, lane, warp);
  __syncthreads();
  if (threadIdx.x < kAcc) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < kAccThreads / 32; w++) v += red[threadIdx.x * 8 + w];
    p.partials[(size_t)threadIdx.x * (((unsigned)nblk + 31u) & ~31u) + blockIdx.x] = v;
  }
}

#endif  // __CUDACC__

}  // namespace b2r
