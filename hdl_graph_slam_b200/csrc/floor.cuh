// floor.cuh — FloorDetectionNodelet::detect (apps/floor_detection_nodelet.cpp:110-180) on the device (SURVEY.md §8f row 5).
//
// Semantics are pinned by tests/floor_ref.cpp (its header marks every rule UPSTREAM-RECALL or ENGINE):
//   k_floor_band          <- transformPointCloud(tilt) (:117) and the two PlaneClipper3D clips (:118-119, plane_clip :189-204): keep
//                            iff ((0 x' + 0 y') + 1 z') >= -(h + r) and NOT >= -(h - r), in float32; tilted records written whole
//   k_floor_normal_flags  <- normal_filtering (:211-238): k = 10 neighbours (itself included) in ascending (d2, index) order over the
//                            band's BVH, pcl::computeMeanAndCovarianceMatrix (raw_moment_cov_f32), pcl::eigen33 (linalg.cuh),
//                            keep iff |normalized(n).z| > cos(normal_filter_thresh) in float64; fewer than 3 neighbours -> NaN -> drop
//   k_ransac_samples      <- SampleConsensusModelPlane + RandomSampleConsensus (PCL 1.10, sequential): the model's boost::mt19937
//                            seeded 12345, drawIndexSample over the persistent shuffled_indices_, isSampleGood, computeModelCoefficients.
//                            One thread: the stream is sequential by construction (each draw swaps the permutation the next one reads)
//   k_ransac_count        <- countWithinDistance for B hypotheses over all n points (integer counts: independent of the order)
//   k_ransac_inlier_flags <- selectWithinDistance of the best model, then the order-preserving compaction (prefilter.cuh)
// The sample stream depends on the cloud and the seed only, never on the inlier counts; the counts only decide where the loop stops.
// So the device draws and counts B hypotheses at a time and the host replays computeModel's loop (RansacReplay, with the host's libm
// for log / pow) over them, asking for the next B only when the loop has not stopped inside the batch.
#pragma once
#include <algorithm>
#include <climits>
#include <cmath>
#include <cfloat>
#include <limits>
#include "engine.cuh"
#include "linalg.cuh"
#include "bvh.cuh"
#include "gicp.cuh"
#include "vgicp_cuda.cuh"

namespace b2r {

constexpr int kFloorK = 10;                 // ne.setKSearch(10) (:219)
constexpr unsigned kRansacSeed = 12345u;    // SampleConsensusModel(cloud, random = false)
constexpr int kRansacMaxSampleChecks = 1000;
constexpr int kRansacMaxIterations = 10000;
constexpr double kRansacProbability = 0.99;
constexpr double kRansacThreshold = 0.1;    // ransac.setDistanceThreshold(0.1) (:140)

// ---- boost::mt19937 (== std::mt19937: MT19937 with the reference initialisation) as __host__ __device__ code
struct Mt19937 {
  unsigned int mt[624];
  int mti;
  B2R_HD void seed(unsigned int s) {
    mt[0] = s;
    for (int i = 1; i < 624; i++) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (unsigned int)i;
    mti = 624;
  }
  B2R_HD unsigned int next() {
    if (mti >= 624) {
      for (int i = 0; i < 624; i++) {
        const unsigned int y = (mt[i] & 0x80000000u) | (mt[(i + 1) % 624] & 0x7fffffffu);
        mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
      }
      mti = 0;
    }
    unsigned int y = mt[mti++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
  }
  // SampleConsensusModel::rnd(): boost::uniform_int<>(0, INT_MAX) over mt19937's [0, 2^32 - 1] draws one word and divides it by the
  // bucket size 2 (brange = 2^32 - 1 is the type's maximum and brange % 2^31 == range, so bucket_size = 2^32 / 2^31 ... + 1 = 2);
  // every quotient is <= INT_MAX, so nothing is rejected: rnd() == mt() >> 1
  B2R_HD unsigned int rnd() { return next() >> 1; }
};

// one RANSAC hypothesis: the three sample indices (into the filtered cloud), the plane, ok = 0 when getSamples found no good sample
struct FloorHyp {
  int idx[3];
  float c[4];
  int ok;
};

// drawIndexSample + isSampleGood (at most 1000 checks) + computeModelCoefficients.  pt(i) returns point i's xyz; shuffled is the
// model's shuffled_indices_ (0..n-1 initially), which persists across draws within one computeModel.
template <class PtAt>
B2R_HD void ransac_draw(Mt19937& g, int* shuffled, int n, PtAt pt, FloorHyp& h) {
  h.ok = 0;
  if (n < 3) return;  // getSamples: fewer indices than the sample size -> empty selection
  for (int check = 0; check < kRansacMaxSampleChecks; check++) {
    for (int i = 0; i < 3; i++) {
      const int j = i + (int)(g.rnd() % (unsigned int)(n - i));
      const int t = shuffled[i]; shuffled[i] = shuffled[j]; shuffled[j] = t;
    }
    const float3 p0 = pt(shuffled[0]), p1 = pt(shuffled[1]), p2 = pt(shuffled[2]);
    const float ax = fsub(p1.x, p0.x), ay = fsub(p1.y, p0.y), az = fsub(p1.z, p0.z);
    const float bx = fsub(p2.x, p0.x), by = fsub(p2.y, p0.y), bz = fsub(p2.z, p0.z);
    const float d0 = fdiv_rn(ax, bx), d1 = fdiv_rn(ay, by), d2 = fdiv_rn(az, bz);
    if (!(d0 != d1 || d2 != d1)) continue;  // collinear (a NaN quotient counts as good)
    h.idx[0] = shuffled[0]; h.idx[1] = shuffled[1]; h.idx[2] = shuffled[2];
    float c0 = fsub(fmul(ay, bz), fmul(az, by)), c1 = fsub(fmul(az, bx), fmul(ax, bz)), c2 = fsub(fmul(ax, by), fmul(ay, bx)), c3 = 0.0f;
    // VectorXf::normalize(): squaredNorm as one SSE packet reduction (a0 + a2) + (a1 + a3); a zero vector is left unchanged
    const float sq = fadd(fadd(fmul(c0, c0), fmul(c2, c2)), fadd(fmul(c1, c1), fmul(c3, c3)));
    if (sq > 0.0f) {
      const float r = fsqrt_rn(sq);
      c0 = fdiv_rn(c0, r); c1 = fdiv_rn(c1, r); c2 = fdiv_rn(c2, r); c3 = fdiv_rn(c3, r);
    }
    // d = -(c . p0) with p0's fourth float, which is 1 in every pcl::PointXYZI
    const float dot = fadd(fadd(fmul(c0, p0.x), fmul(c2, p0.z)), fadd(fmul(c1, p0.y), fmul(c3, 1.0f)));
    h.c[0] = c0; h.c[1] = c1; h.c[2] = c2; h.c[3] = fmul(-1.0f, dot);
    h.ok = 1;
    return;
  }
}

// |c . (x, y, z, 1)| < threshold (countWithinDistance / selectWithinDistance), the float dot associated as above
B2R_HD bool ransac_inlier(const float* c, float x, float y, float z) {
  const float d = fadd(fadd(fmul(c[0], x), fmul(c[2], z)), fadd(fmul(c[1], y), fmul(c[3], 1.0f)));
  return (double)fabsf(d) < kRansacThreshold;
}

// RandomSampleConsensus::computeModel's loop, fed one hypothesis (the iterations_-th sample) and its inlier count at a time.
// No hypothesis is ever skipped: computeModelCoefficients repeats isSampleGood's test, so it cannot fail after it.
struct RansacReplay {
  int iterations = 0;
  int best_count = -INT_MAX;
  int best = -1;        // index of the best hypothesis in the stream
  double k = 1.0;
  double log_probability = 0.0, one_over_indices = 0.0;
  bool stopped = false;
  void init(size_t n) {
    log_probability = std::log(1.0 - kRansacProbability);
    one_over_indices = 1.0 / static_cast<double>(n);
  }
  bool wants_more() const { return !stopped && iterations < k; }
  // returns false once the loop has stopped.  A hypothesis rejected up front (the loop had already stopped, or no sample) is not
  // consumed; the one that reaches the iteration cap is: it may have become the best before the loop breaks, as in computeModel
  bool step(const FloorHyp& h, int count) {
    if (!wants_more() || !h.ok) { stopped = true; return false; }
    if (count > best_count) {
      best_count = count;
      best = iterations;
      const double w = static_cast<double>(best_count) * one_over_indices;
      double p_no_outliers = 1.0 - std::pow(w, 3.0);
      p_no_outliers = std::max(std::numeric_limits<double>::epsilon(), p_no_outliers);
      p_no_outliers = std::min(1.0 - std::numeric_limits<double>::epsilon(), p_no_outliers);
      k = log_probability / std::log(p_no_outliers);
    }
    ++iterations;
    if (iterations > kRansacMaxIterations) { stopped = true; return false; }
    return true;
  }
};

// ---- device kernels
// tilt + both clips: tilted records to `out`, keep flags
struct FloorBandArg { float Tf[12]; float d_hi, d_lo; };  // d = (float)(sensor_height +- height_clip_range)
__global__ void k_floor_band(const float* __restrict__ in, int stride_f, int n, FloorBandArg A, float* __restrict__ out, unsigned char* flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = in + (size_t)i * stride_f;
  float* o = out + (size_t)i * stride_f;
  const float x = p[0], y = p[1], z = p[2];
  for (int k = 3; k < stride_f; k++) o[k] = p[k];
  const float tx = xform_row(A.Tf[0], A.Tf[1], A.Tf[2], A.Tf[3], x, y, z);
  const float ty = xform_row(A.Tf[4], A.Tf[5], A.Tf[6], A.Tf[7], x, y, z);
  const float tz = xform_row(A.Tf[8], A.Tf[9], A.Tf[10], A.Tf[11], x, y, z);
  o[0] = tx; o[1] = ty; o[2] = tz;
  // PlaneClipper3D::clipPoint3D with plane (0, 0, 1, d): ((a x + b y) + c z) >= -d
  const float s = fadd(fadd(fmul(0.0f, tx), fmul(0.0f, ty)), fmul(1.0f, tz));
  flags[i] = (s >= -A.d_hi && !(s >= -A.d_lo)) ? 1 : 0;
}

// one warp per leaf of the band's BVH: k = 10 neighbours, PCL's moments, eigen33, the keep flag at the point's band index
__global__ void __launch_bounds__(kKnnThreads, 4) k_floor_normal_flags(Bvh b, const float* __restrict__ raw, int stride_f, double cos_thresh,
                                                                       unsigned char* __restrict__ flags) {
  __shared__ int nbr[kFloorK][kKnnThreads];
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int leaf = s >> 5;
  if (leaf >= b.nleaf) return;  // whole warps only
  const float4 q = b.sp[s];
  const bool active = idx_bits(q.w) != kPadIdx;
  KnnRegs<kFloorK> L;
  L.reset();
  bvh_group_search(b, q.x, q.y, q.z, active, L, leaf);
  if (!active) return;
  const int tx = threadIdx.x;
#pragma unroll
  for (int j = 0; j < kFloorK; j++) nbr[j][tx] = (int)(unsigned int)(L.key[j] & 0xffffffffull);
  const int kk = L.count();
  bool keep = false;
  if (kk >= 3) {  // computePointNormal: fewer than 3 neighbours -> NaN normal, which no threshold keeps
    float C[9], v[3];
    raw_moment_cov_f32(kk, [&](int j) {
      const float* p = raw + (size_t)nbr[j][tx] * stride_f;
      return make_float3(p[0], p[1], p[2]);
    }, C);
    pcl_eigen33(C, v);
    // getNormalVector3fMap().normalized().dot(UnitZ()): n.z / |n| (the flip towards the viewpoint only changes the sign)
    const float sq = fadd(fmul(v[0], v[0]), fadd(fmul(v[1], v[1]), fmul(v[2], v[2])));
    const float nz = sq > 0.0f ? __fdiv_rn(v[2], __fsqrt_rn(sq)) : v[2];
    keep = fabs((double)nz) > cos_thresh;
  }
  flags[idx_bits(q.w)] = keep ? 1 : 0;
}

// the RANSAC stream: hypotheses [t0, t0 + B) of one computeModel.  The generator and the permutation live in device memory
// between batches; `init` starts a fresh model (seed 12345, shuffled_indices_ = 0..n-1, filled by k_floor_iota before).
__global__ void k_ransac_samples(const float* __restrict__ rec, int stride_f, int n, Mt19937* __restrict__ g, int* __restrict__ shuffled,
                                 int B, int init, FloorHyp* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (init) g->seed(kRansacSeed);
  bool exhausted = false;
  for (int t = 0; t < B; t++) {
    FloorHyp h;
    h.ok = 0;
    if (!exhausted) {
      ransac_draw(*g, shuffled, n, [&](int i) {
        const float* p = rec + (size_t)i * stride_f;
        return make_float3(p[0], p[1], p[2]);
      }, h);
      exhausted = !h.ok;  // the loop stops at the first empty selection
    }
    out[t] = h;
  }
}

__global__ void k_floor_iota(int* a, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = i;
}

// B hypotheses (blockIdx.y) x n points: exact integer inlier counts (counts[] zeroed before)
constexpr int kRansacCountThreads = 256;
__global__ void __launch_bounds__(kRansacCountThreads) k_ransac_count(const float* __restrict__ rec, int stride_f, int n,
                                                                      const FloorHyp* __restrict__ hyp, int* __restrict__ counts) {
  const FloorHyp h = hyp[blockIdx.y];
  if (!h.ok) return;
  int c = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float* p = rec + (size_t)i * stride_f;
    c += ransac_inlier(h.c, p[0], p[1], p[2]) ? 1 : 0;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(counts + blockIdx.y, c);
}

__global__ void k_ransac_inlier_flags(const float* __restrict__ rec, int stride_f, int n, FloorHyp h, unsigned char* __restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = rec + (size_t)i * stride_f;
  flags[i] = ransac_inlier(h.c, p[0], p[1], p[2]) ? 1 : 0;
}

// ---- host side
// tilt_matrix (:112-113): AngleAxisf(tilt_deg * M_PI / 180.0f, UnitY).toRotationMatrix() in Eigen's float32 statement order
// (sinf / cosf are glibc's here, as upstream's), row-major 4x4
inline void floor_tilt_matrix(double tilt_deg, float* T) {
  const float angle = (float)(tilt_deg * M_PI / 180.0f);
  const float s = std::sin(angle), c = std::cos(angle);
  const float ax[3] = {0.0f, 1.0f, 0.0f};
  const float sa[3] = {s * ax[0], s * ax[1], s * ax[2]};
  const float ca[3] = {(1.0f - c) * ax[0], (1.0f - c) * ax[1], (1.0f - c) * ax[2]};
  float R[9];
  float t = ca[0] * ax[1];
  R[1] = t - sa[2]; R[3] = t + sa[2];
  t = ca[0] * ax[2];
  R[2] = t + sa[1]; R[6] = t - sa[1];
  t = ca[1] * ax[2];
  R[5] = t - sa[0]; R[7] = t + sa[0];
  R[0] = ca[0] * ax[0] + c; R[4] = ca[1] * ax[1] + c; R[8] = ca[2] * ax[2] + c;
  for (int r = 0; r < 4; r++)
    for (int k = 0; k < 4; k++) T[r * 4 + k] = (r < 3 && k < 3) ? R[r * 3 + k] : (r == k ? 1.0f : 0.0f);
}

// one handle's floor-detection state: its own clouds and scratch, never shared with the registration or prefilter buffers
struct FloorWork {
  DevBuf<float> in, tilted, band, kept, filtered, inliers;  // records (stride of the call)
  DevBuf<unsigned char> flags;
  DevBuf<int> blocks, total, shuffled, counts;
  MappedBuf<int> h_total;
  DevBuf<Mt19937> rng;
  DevBuf<FloorHyp> hyp;
  PinnedBuf<FloorHyp> h_hyp;
  PinnedBuf<int> h_counts;
  Cloud band_cloud;  // the band's BVH (normal filter)
};

}  // namespace b2r
