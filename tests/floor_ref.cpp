// tests/floor_ref.cpp — sequential restatement of FloorDetectionNodelet::detect (apps/floor_detection_nodelet.cpp:110-180, PCL 1.10,
// Eigen 3.3) that the device call b2r_floor_detect is held to bit for bit.  Test infrastructure, built by tests/floor_ref.py with
// -ffp-contract=off (the reference is built without FMA); PCL and Eigen are not available here, so every rule is restated:
//
//   UPSTREAM-RECALL  read from the upstream sources as remembered; DOUBT marks the ones not certain
//   ENGINE           a choice of this project where upstream cannot be reproduced or is unspecified
//
// 1. tilt (:112-113, :117)  UPSTREAM-RECALL  AngleAxisf(float(tilt_deg * M_PI / 180.0f), UnitY).toRotationMatrix() in Eigen's
//    statement order (sin_axis = sinf(a) axis, cos1_axis = (1 - cosf(a)) axis; off-diagonals tmp -+ sin_axis, diagonal
//    cos1_axis.*axis + c); glibc's sinf / cosf.  transformPointCloud: x' = ((m0 x + m1 y) + m2 z) + m3 in float32  ENGINE (the
//    project's rule for every pcl::transformPointCloud); the other fields are copied.
// 2. band (:118-119, :189-204)  UPSTREAM-RECALL  PlaneClipper3D::clipPoint3D keeps p iff ((a x + b y) + c z) >= -d in float32 with
//    plane (0, 0, 1, (float)(sensor_height +- height_clip_range)); clipPointCloud3D lists the passing indices in order, and
//    ExtractIndices keeps them (first clip) or everything else (second clip, setNegative(true)).  So a NaN z or an infinite x / y
//    (0 * inf = NaN) fails the first clip, and a point on a plane follows >=.
// 3. normal filter (:121-123, :211-238)
//    neighbours  ENGINE  k = 10 (itself included, min(10, m) when the band is smaller) in ascending (d2, index) order with
//                d2 = ((dx dx + dy dy) + dz dz) in float32 (FLANN's own order and distance are not reproduced).
//    moments     UPSTREAM-RECALL  computeMeanAndCovarianceMatrix, dense path: float32 sums of xx xy xz yy yz zz x y z in neighbour
//                order, each / k (float32), cov = E[ab] - E[a] E[b].  Fewer than 3 neighbours: NaN normal (computePointNormal).
//    eigen33     UPSTREAM-RECALL  pcl::eigen33's smallest-eigenvalue form: scale = max |entry| (1 if <= FLT_MIN), computeRoots in
//                float32 in its written order (c0 < FLT_EPSILON -> computeRoots2; sort; roots(0) <= 0 -> computeRoots2), the three
//                row cross products of (A/scale - roots(0) I), the first largest squared norm, divided by its sqrt.
//                computeRoots2's d = Scalar(b * b - 4.0 * c): b * b in float32, the rest in float64.
//    trig        ENGINE  atan2f / cosf / sinf of computeRoots as (float)f((double)x): glibc's float routines cannot be reproduced on
//                the device.  atan2 is the engine's atan2_rn (csrc/atan2_rn.cuh), shared with the device: CUDA's and glibc's float64
//                atan2 round some float32 results differently; cos and sin agree on every |t| <= 1.1.
//    squares     UPSTREAM-RECALL  Vector3f squaredNorm as x x + (y y + z z): Eigen 3.3 reduces a fixed-size 3-vector with
//                redux_novec_unroller, which splits at Length / 2 = 1 (first element, then the sum of the other two).
//    keep        UPSTREAM-RECALL  |normalized(n).dot(UnitZ)| > cos(normal_filter_thresh * M_PI / 180.0) in float64, where the dot
//                is n.z / sqrt(squaredNorm) (the zeros of UnitZ add nothing); the viewpoint flip only changes the sign.
// 4. back-transform (:125)  ENGINE (unpinned against Eigen's general 4x4 inverse)  the inverse of odometry_gate.cuh: the 3x3 block
//    by cofactors in float64, -A^-1 t in float64, each entry rounded to float32 once.  At tilt 0 it is the identity.
// 5. size gate (:133)  UPSTREAM-RECALL  size_t < int: a negative threshold converts to a huge value and rejects every cloud.
// 6. RANSAC (:138-144), SampleConsensusModelPlane + RandomSampleConsensus, sequential PCL 1.10  UPSTREAM-RECALL
//    rng         boost::mt19937 seeded 12345 (random = false) == std::mt19937(12345).  rnd() = uniform_int<>(0, INT_MAX) over
//                [0, 2^32 - 1]: boost's generate_uniform_int takes brange = 2^32 - 1 (the type's max), bucket_size = brange / 2^31 = 1,
//                +1 because brange % 2^31 == range, so 2, and result = mt() / 2 <= INT_MAX is never rejected: rnd() = mt() >> 1.
//    samples     shuffled_indices_ starts 0..n-1 and persists within the call; drawIndexSample swaps shuffled[i] with
//                shuffled[i + rnd() % (n - i)] for i = 0, 1, 2 and takes shuffled[0..2]; isSampleGood: dy1dy2 = (p1 - p0) / (p2 - p0)
//                is good iff [0] != [1] || [2] != [1] (NaN counts as good); at most 1000 checks, then the selection is empty and
//                the loop breaks.  Fewer than 3 points: empty selection at once, and getSamples sets iterations_ = INT_MAX - 1
//                (its "one of these will make it stop"), which is what computeModel leaves in iterations_.
//    model       computeModelCoefficients: float32 cross product of p1 - p0 and p2 - p0, w = 0, VectorXf::normalize() (a zero vector
//                is left unchanged), d = -1 * (c . p0) with p0's fourth float, 1 in every pcl::PointXYZI.
//    dots        (DOUBT) a 4-float dot / squared norm as Eigen's SSE packet reduction: (a0 b0 + a2 b2) + (a1 b1 + a3 b3).
//    count       countWithinDistance / selectWithinDistance: |c . (x, y, z, 1)| < 0.1, the float widened to double.
//    loop        max_iterations_ 10000, probability_ 0.99, best count starts at -INT_MAX, a new best needs a strictly larger count,
//                k = log(1 - p) / log(clamp(1 - w^3, eps, 1 - eps)) in float64; while (iterations_ < k), ++iterations_ after each
//                hypothesis, break once iterations_ > max_iterations_.  Duplicate points give the zero model (0, 0, 0, -0), which
//                counts every point as an inlier.
//    no model    ENGINE  computeModel found none: the inlier list is empty.  With floor_pts_thresh <= 0 the reference would go on
//                to read an empty coefficient vector (undefined); reported as none here.
// 7. gates (:147-166)  UPSTREAM-RECALL  inliers < floor_pts_thresh (size_t against int) -> none; ref = tilt^-1 UnitZ (float32 rows
//    ((r0 0 + r1 0) + r2 1) + r3 0); |(double)(c0 r0 + (c1 r1 + c2 r2))| < cos(floor_normal_thresh * M_PI / 180.0) -> none (the
//    3-float dot of head<3>() associated as the squares above); c . UnitZ < 0 -> all four coefficients * -1.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <random>
#include <unordered_map>
#include <utility>
#include <vector>
#include "../hdl_graph_slam_b200/csrc/atan2_rn.cuh"

namespace {

struct Params {  // == b2r_floor_params
  double tilt_deg, sensor_height, height_clip_range;
  int32_t floor_pts_thresh, use_normal_filtering;
  double floor_normal_thresh, normal_filter_thresh;
};
struct Result {  // == b2r_floor_result
  int32_t detected, reason;
  float coeffs[4];
  uint64_t n_filtered, n_inliers;
  int32_t ransac_iterations, model_indices[3], ransac_batches, ransac_hypotheses, readbacks, reserved;
};
static_assert(sizeof(Params) == 48 && sizeof(Result) == 72, "mirrors of the ABI structs");

void tilt_matrix(double tilt_deg, float* T) {
  const float angle = (float)(tilt_deg * M_PI / 180.0f);
  const float s = std::sin(angle), c = std::cos(angle);
  const float axis[3] = {0.f, 1.f, 0.f};
  float sin_axis[3], cos1_axis[3];
  for (int i = 0; i < 3; i++) { sin_axis[i] = s * axis[i]; cos1_axis[i] = (1.0f - c) * axis[i]; }
  float R[3][3];
  float tmp = cos1_axis[0] * axis[1];
  R[0][1] = tmp - sin_axis[2];
  R[1][0] = tmp + sin_axis[2];
  tmp = cos1_axis[0] * axis[2];
  R[0][2] = tmp + sin_axis[1];
  R[2][0] = tmp - sin_axis[1];
  tmp = cos1_axis[1] * axis[2];
  R[1][2] = tmp - sin_axis[0];
  R[2][1] = tmp + sin_axis[0];
  for (int i = 0; i < 3; i++) R[i][i] = cos1_axis[i] * axis[i] + c;
  for (int r = 0; r < 4; r++)
    for (int k = 0; k < 4; k++) T[r * 4 + k] = (r < 3 && k < 3) ? R[r][k] : (r == k ? 1.f : 0.f);
}

void inverse_rigid(const float* m, float* o) {
  const double a[9] = {m[0], m[1], m[2], m[4], m[5], m[6], m[8], m[9], m[10]};
  const double c00 = a[4] * a[8] - a[5] * a[7], c01 = a[5] * a[6] - a[3] * a[8], c02 = a[3] * a[7] - a[4] * a[6];
  const double id = 1.0 / (a[0] * c00 + a[1] * c01 + a[2] * c02);
  const double Ai[9] = {c00 * id, (a[2] * a[7] - a[1] * a[8]) * id, (a[1] * a[5] - a[2] * a[4]) * id,
                        c01 * id, (a[0] * a[8] - a[2] * a[6]) * id, (a[2] * a[3] - a[0] * a[5]) * id,
                        c02 * id, (a[1] * a[6] - a[0] * a[7]) * id, (a[0] * a[4] - a[1] * a[3]) * id};
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) o[r * 4 + c] = (float)Ai[r * 3 + c];
    o[r * 4 + 3] = (float)(-(Ai[r * 3 + 0] * m[3] + Ai[r * 3 + 1] * m[7] + Ai[r * 3 + 2] * m[11]));
  }
  o[12] = o[13] = o[14] = 0.f;
  o[15] = 1.f;
}

void transform(const float* in, size_t n, size_t sf, const float* T, float* out) {
  for (size_t i = 0; i < n; i++) {
    const float* p = in + i * sf;
    float* o = out + i * sf;
    const float x = p[0], y = p[1], z = p[2];
    for (size_t k = 3; k < sf; k++) o[k] = p[k];
    for (int r = 0; r < 3; r++) o[r] = ((T[r * 4] * x + T[r * 4 + 1] * y) + T[r * 4 + 2] * z) + T[r * 4 + 3];
  }
}

bool clip(const float* p, float d) { return ((0.0f * p[0] + 0.0f * p[1]) + 1.0f * p[2]) >= -d; }

// ---- pcl::eigen33 (smallest eigenvalue's eigenvector)
void roots2(float b, float c, float* r) {
  r[0] = 0.f;
  float d = (float)((double)(b * b) - 4.0 * (double)c);
  if (d < 0.f) d = 0.f;
  const float sd = std::sqrt(d);
  r[2] = 0.5f * (b + sd);
  r[1] = 0.5f * (b - sd);
}
void roots(const float m[3][3], float* r) {
  const float c0 = m[0][0] * m[1][1] * m[2][2] + 2.0f * m[0][1] * m[0][2] * m[1][2] - m[0][0] * m[1][2] * m[1][2] -
                   m[1][1] * m[0][2] * m[0][2] - m[2][2] * m[0][1] * m[0][1];
  const float c1 = m[0][0] * m[1][1] - m[0][1] * m[0][1] + m[0][0] * m[2][2] - m[0][2] * m[0][2] + m[1][1] * m[2][2] - m[1][2] * m[1][2];
  const float c2 = m[0][0] + m[1][1] + m[2][2];
  if (std::fabs(c0) < std::numeric_limits<float>::epsilon()) {
    roots2(c2, c1, r);
    return;
  }
  const float s_inv3 = (float)(1.0 / 3.0);
  const float s_sqrt3 = std::sqrt(3.0f);
  const float c2_over_3 = c2 * s_inv3;
  float a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
  if (a_over_3 > 0.f) a_over_3 = 0.f;
  const float half_b = 0.5f * (c0 + c2_over_3 * (2.0f * c2_over_3 * c2_over_3 - c1));
  float q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
  if (q > 0.f) q = 0.f;
  const float rho = std::sqrt(-a_over_3);
  const float theta = (float)b2r::atan2_rn((double)std::sqrt(-q), (double)half_b) * s_inv3;
  const float cos_theta = (float)std::cos((double)theta), sin_theta = (float)std::sin((double)theta);
  r[0] = c2_over_3 + 2.0f * rho * cos_theta;
  r[1] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
  r[2] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
  if (r[0] >= r[1]) std::swap(r[0], r[1]);
  if (r[1] >= r[2]) {
    std::swap(r[1], r[2]);
    if (r[0] >= r[1]) std::swap(r[0], r[1]);
  }
  if (r[0] <= 0.f) roots2(c2, c1, r);
}
float sqnorm3(const float* v) { return v[0] * v[0] + (v[1] * v[1] + v[2] * v[2]); }
void eigen33(const float* A, float* v) {
  float scale = std::fabs(A[0]);
  for (int i = 1; i < 9; i++) scale = std::fabs(A[i]) > scale ? std::fabs(A[i]) : scale;
  if (scale <= std::numeric_limits<float>::min()) scale = 1.0f;
  float m[3][3];
  for (int i = 0; i < 9; i++) m[i / 3][i % 3] = A[i] / scale;
  float r[3];
  roots(m, r);
  for (int i = 0; i < 3; i++) m[i][i] -= r[0];
  auto cross = [](const float* a, const float* b, float* o) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
  };
  float v1[3], v2[3], v3[3];
  cross(m[0], m[1], v1);
  cross(m[0], m[2], v2);
  cross(m[1], m[2], v3);
  const float l1 = sqnorm3(v1), l2 = sqnorm3(v2), l3 = sqnorm3(v3);
  const float* s;
  float l;
  if (l1 >= l2 && l1 >= l3) { s = v1; l = l1; }
  else if (l2 >= l1 && l2 >= l3) { s = v2; l = l2; }
  else { s = v3; l = l3; }
  const float sl = std::sqrt(l);
  for (int i = 0; i < 3; i++) v[i] = s[i] / sl;
}

// ---- exact k-NN in ascending (d2, index) order over a hashed grid
struct Knn {
  const float* pts;
  size_t n, sf;
  double cell;
  bool brute = false;
  std::unordered_map<uint64_t, std::vector<int>> grid;
  float lo[3];
  static uint64_t key(long long a, long long b, long long c) { return ((uint64_t)(a & 0x1fffff) << 42) | ((uint64_t)(b & 0x1fffff) << 21) | (uint64_t)(c & 0x1fffff); }
  long long ci(float v, int a) const { return (long long)std::floor(((double)v - lo[a]) / cell); }
  Knn(const float* p, size_t n_, size_t sf_, double cell_) : pts(p), n(n_), sf(sf_), cell(cell_) {
    float hi[3];
    for (int a = 0; a < 3; a++) { lo[a] = INFINITY; hi[a] = -INFINITY; }
    for (size_t i = 0; i < n; i++)
      for (int a = 0; a < 3; a++) { lo[a] = std::min(lo[a], p[i * sf + a]); hi[a] = std::max(hi[a], p[i * sf + a]); }
    for (int a = 0; a < 3; a++)
      if (n && !(((double)hi[a] - lo[a]) / cell < 1e6)) brute = true;
    if (brute) return;
    for (size_t i = 0; i < n; i++) grid[key(ci(p[i * sf], 0), ci(p[i * sf + 1], 1), ci(p[i * sf + 2], 2))].push_back((int)i);
  }
  float d2(size_t q, int j) const {
    const float dx = pts[q * sf] - pts[j * sf], dy = pts[q * sf + 1] - pts[j * sf + 1], dz = pts[q * sf + 2] - pts[j * sf + 2];
    return (dx * dx + dy * dy) + dz * dz;
  }
  void query(size_t q, int k, std::vector<std::pair<float, int>>& out) const {
    out.clear();
    auto consider = [&](int j) {
      const std::pair<float, int> e(d2(q, j), j);
      if ((int)out.size() == k && !(e < out.back())) return;
      out.insert(std::upper_bound(out.begin(), out.end(), e), e);
      if ((int)out.size() > k) out.pop_back();
    };
    if (brute) {
      for (size_t j = 0; j < n; j++) consider((int)j);
      return;
    }
    const long long c[3] = {ci(pts[q * sf], 0), ci(pts[q * sf + 1], 1), ci(pts[q * sf + 2], 2)};
    for (long long R = 0;; R++) {
      for (long long a = -R; a <= R; a++)
        for (long long b = -R; b <= R; b++)
          for (long long d = -R; d <= R; d++) {
            if (std::max({std::llabs(a), std::llabs(b), std::llabs(d)}) != R) continue;
            auto it = grid.find(key(c[0] + a, c[1] + b, c[2] + d));
            if (it == grid.end()) continue;
            for (int j : it->second) consider(j);
          }
      // every unvisited point is at least R cells away on some axis
      const double reach = (double)R * cell;
      if (out.size() == std::min<size_t>(k, n) && (out.size() == n || (double)out.back().first * (1.0 + 1e-5) + 1e-30 < reach * reach)) return;
      if (R > 2000000) return;
    }
  }
};

// ---- RANSAC
struct Hyp { int idx[3]; float c[4]; int ok; };
struct Sampler {
  std::mt19937 mt{12345u};
  std::vector<int> shuffled;
  const float* pts;
  size_t sf;
  Sampler(const float* p, size_t n, size_t sf_) : shuffled(n), pts(p), sf(sf_) {
    for (size_t i = 0; i < n; i++) shuffled[i] = (int)i;
  }
  unsigned rnd() { return (unsigned)(mt() >> 1); }
  Hyp next() {
    Hyp h{};
    const size_t n = shuffled.size();
    if (n < 3) return h;
    for (int check = 0; check < 1000; check++) {
      for (size_t i = 0; i < 3; i++) std::swap(shuffled[i], shuffled[i + (size_t)rnd() % (n - i)]);
      const float* p0 = pts + shuffled[0] * sf;
      const float* p1 = pts + shuffled[1] * sf;
      const float* p2 = pts + shuffled[2] * sf;
      float a[3], b[3], q[3];
      for (int k = 0; k < 3; k++) { a[k] = p1[k] - p0[k]; b[k] = p2[k] - p0[k]; q[k] = a[k] / b[k]; }
      if (!((q[0] != q[1]) || (q[2] != q[1]))) continue;
      for (int k = 0; k < 3; k++) h.idx[k] = shuffled[k];
      float c[4] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0], 0.f};
      const float z = (c[0] * c[0] + c[2] * c[2]) + (c[1] * c[1] + c[3] * c[3]);
      if (z > 0.f) {
        const float s = std::sqrt(z);
        for (int k = 0; k < 4; k++) c[k] = c[k] / s;
      }
      const float dot = (c[0] * p0[0] + c[2] * p0[2]) + (c[1] * p0[1] + c[3] * 1.0f);
      for (int k = 0; k < 3; k++) h.c[k] = c[k];
      h.c[3] = -1 * dot;
      h.ok = 1;
      return h;
    }
    return h;
  }
};
bool inlier(const float* c, const float* p) {
  const float d = (c[0] * p[0] + c[2] * p[2]) + (c[1] * p[1] + c[3] * 1.0f);
  return (double)std::fabs(d) < 0.1;
}

}  // namespace

extern "C" {

void ref_mt19937(uint32_t seed, size_t n, uint32_t* out) {
  std::mt19937 mt(seed);
  for (size_t i = 0; i < n; i++) out[i] = (uint32_t)mt();
}

void ref_eigen33(const float* A, float* v) { eigen33(A, v); }
void ref_eigen33_many(const float* A, size_t count, float* v) {
  for (size_t i = 0; i < count; i++) eigen33(A + 9 * i, v + 3 * i);
}

// the first `count` hypotheses of a fresh model: idx[3], c[4], ok per record (8 x 4 bytes)
void ref_ransac_hypotheses(const float* pts, size_t n, size_t sf, size_t count, Hyp* out) {
  Sampler S(pts, n, sf);
  for (size_t t = 0; t < count; t++) out[t] = S.next();
}

// detect(); band_mask[i] (capacity n): input point i lies in the height band; normal_keep[j] (capacity n): band point j passed the
// normal filter (all 1 when it is off)
int ref_floor_detect(const float* pts, size_t n, size_t sf, const Params* p, Result* r, float* filtered, float* inliers_out,
                     unsigned char* band_mask, unsigned char* normal_keep) {
  std::memset(r, 0, sizeof(*r));
  r->model_indices[0] = r->model_indices[1] = r->model_indices[2] = -1;
  if (n == 0) { r->reason = 1; return 0; }
  float T[16], Ti[16];
  tilt_matrix(p->tilt_deg, T);
  inverse_rigid(T, Ti);
  std::vector<float> tilted(n * sf), band;
  transform(pts, n, sf, T, tilted.data());
  const float d_hi = (float)(p->sensor_height + p->height_clip_range), d_lo = (float)(p->sensor_height - p->height_clip_range);
  for (size_t i = 0; i < n; i++) {
    const float* q = tilted.data() + i * sf;
    const bool keep = clip(q, d_hi) && !clip(q, d_lo);
    band_mask[i] = keep;
    if (keep) band.insert(band.end(), q, q + sf);
  }
  const size_t m = band.size() / sf;
  std::vector<float> kept;
  if (p->use_normal_filtering) {
    const double cos_t = std::cos(p->normal_filter_thresh * M_PI / 180.0);
    Knn knn(band.data(), m, sf, 0.5);
    std::vector<std::pair<float, int>> nb;
    for (size_t i = 0; i < m; i++) {
      knn.query(i, 10, nb);
      bool keep = false;
      if (nb.size() >= 3) {
        float acc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        for (auto& e : nb) {
          const float* q = band.data() + (size_t)e.second * sf;
          acc[0] += q[0] * q[0]; acc[1] += q[0] * q[1]; acc[2] += q[0] * q[2];
          acc[3] += q[1] * q[1]; acc[4] += q[1] * q[2]; acc[5] += q[2] * q[2];
          acc[6] += q[0]; acc[7] += q[1]; acc[8] += q[2];
        }
        const float kf = (float)nb.size();
        for (int a = 0; a < 9; a++) acc[a] /= kf;
        const float C[9] = {acc[0] - acc[6] * acc[6], acc[1] - acc[6] * acc[7], acc[2] - acc[6] * acc[8],
                            acc[1] - acc[6] * acc[7], acc[3] - acc[7] * acc[7], acc[4] - acc[7] * acc[8],
                            acc[2] - acc[6] * acc[8], acc[4] - acc[7] * acc[8], acc[5] - acc[8] * acc[8]};
        float v[3];
        eigen33(C, v);
        const float z = sqnorm3(v);
        const float nz = z > 0.f ? v[2] / std::sqrt(z) : v[2];
        keep = std::fabs((double)nz) > cos_t;
      }
      normal_keep[i] = keep;
      if (keep) kept.insert(kept.end(), band.begin() + i * sf, band.begin() + (i + 1) * sf);
    }
  } else {
    for (size_t i = 0; i < m; i++) normal_keep[i] = 1;
    kept = band;
  }
  const size_t nf = kept.size() / sf;
  transform(kept.data(), nf, sf, Ti, filtered);
  r->n_filtered = nf;
  if (nf < static_cast<size_t>(p->floor_pts_thresh)) { r->reason = 2; return 0; }
  // RandomSampleConsensus::computeModel
  Sampler S(filtered, nf, sf);
  int iterations = 0, best_count = -INT_MAX;
  double k = 1.0;
  Hyp best{};
  const double log_probability = std::log(1.0 - 0.99), one_over_indices = 1.0 / static_cast<double>(nf);
  while (iterations < k) {
    const Hyp h = S.next();
    if (!h.ok) break;
    int count = 0;
    for (size_t i = 0; i < nf; i++) count += inlier(h.c, filtered + i * sf);
    if (count > best_count) {
      best_count = count;
      best = h;
      const double w = static_cast<double>(best_count) * one_over_indices;
      double p_no_outliers = 1.0 - std::pow(w, 3.0);
      p_no_outliers = std::max(std::numeric_limits<double>::epsilon(), p_no_outliers);
      p_no_outliers = std::min(1.0 - std::numeric_limits<double>::epsilon(), p_no_outliers);
      k = log_probability / std::log(p_no_outliers);
    }
    ++iterations;
    if (iterations > 10000) break;
  }
  r->ransac_iterations = nf < 3 ? INT_MAX - 1 : iterations;
  if (!best.ok) { r->reason = 3; return 0; }
  for (int i = 0; i < 3; i++) r->model_indices[i] = best.idx[i];
  for (int i = 0; i < 4; i++) r->coeffs[i] = best.c[i];
  size_t ni = 0;
  for (size_t i = 0; i < nf; i++)
    if (inlier(best.c, filtered + i * sf)) { std::memcpy(inliers_out + ni * sf, filtered + i * sf, sf * 4); ni++; }
  r->n_inliers = ni;
  if (ni < static_cast<size_t>(p->floor_pts_thresh)) { r->reason = 4; return 0; }
  float ref[3];
  for (int i = 0; i < 3; i++) ref[i] = ((Ti[i * 4] * 0.f + Ti[i * 4 + 1] * 0.f) + Ti[i * 4 + 2] * 1.f) + Ti[i * 4 + 3] * 0.f;
  const double dot = r->coeffs[0] * ref[0] + (r->coeffs[1] * ref[1] + r->coeffs[2] * ref[2]);
  if (std::abs(dot) < std::cos(p->floor_normal_thresh * M_PI / 180.0)) { r->reason = 5; return 0; }
  if (r->coeffs[0] * 0.f + (r->coeffs[1] * 0.f + r->coeffs[2] * 1.f) < 0.0f)
    for (int i = 0; i < 4; i++) r->coeffs[i] *= -1.0f;
  r->detected = 1;
  r->reason = 0;
  return 0;
}

}  // extern "C"
