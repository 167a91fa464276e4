// tests/icp_pcl_ref.cpp — sequential CPU reference of pcl::IterativeClosestPoint<PointXYZI, PointXYZI> (PCL 1.10 + Eigen 3.3.7, the
// `noetic` image of the reference's docker/) as the factory's ICP branch builds it (registrations.cpp:57-65).  It is the parity target of
// B2R_METHOD_ICP_PCL (csrc/icp_pcl.cuh, csrc/linalg.cuh).  Built by tests/icp_pcl_ref.py with -O2 -ffp-contract=off (no FMA anywhere).
//
// Every choice, tagged UPSTREAM-RECALL (what PCL / Eigen do, restated from memory of their sources) or ENGINE RULE (where this engine
// fixes what upstream leaves open or cannot be reproduced on a device):
//
// computeTransformation
//   UPSTREAM-RECALL  final_transformation_ = guess; input_transformed = transformPointCloud(input, guess) (float32, x' = ((m0 x + m1 y) +
//                    m2 z) + m3), skipped (a plain copy) when guess == Identity exactly; transformation_ = Identity.
//   UPSTREAM-RECALL  loop: correspondences (forward or reciprocal); cnt < min_number_correspondences_ (3) -> converged_ = false, break;
//                    transformation_ = estimateRigidTransformation; input_transformed = transformation_ input_transformed (float32, in
//                    place: the rounding accumulates); final_transformation_ = transformation_ * final_transformation_ (Matrix4f product,
//                    ((a0 b0 + a1 b1) + a2 b2) + a3 b3); ++nr_iterations_; converged_ = hasConverged(); repeat while the criteria's
//                    state is NOT_CONVERGED.
//   UPSTREAM-RECALL  euclidean_fitness_epsilon_ = -DBL_MAX (the relative MSE test never fires), transformation_rotation_epsilon_ = 0
//                    (rotation threshold = 1 - transformation_epsilon).
// determineCorrespondences
//   UPSTREAM-RECALL  float d2 of the 1-NN, d2 = ((dx dx + dy dy) + dz dz), float32; rejected only if (double)d2 > max_dist^2 (INCLUSIVE).
//                    distance = the forward d2.
//   UPSTREAM-RECALL  reciprocal: forward 1-NN i -> j; then the 1-NN of target point j among the CURRENT input_transformed (its tree is
//                    rebuilt every iteration); kept only if that d2' <= max_dist^2 and its index is i.
//   ENGINE RULE      1-NN ties go to the smallest (d2, original index), forward and reverse (bvh.cuh's rule; FLANN leaves it open).
//   ENGINE RULE      points with a non-finite coordinate (source or target, and a source point whose transform overflows) take no part.
// TransformationEstimationSVD -> pcl::umeyama(src, tgt, false), Scalar = float
//   UPSTREAM-RECALL  means, demeaned clouds, sigma = (1/n) dst_demean src_demean^T; JacobiSVD<Matrix3f>(sigma, FullU | FullV);
//                    S = diag(1, 1, det(sigma) < 0 ? -1 : 1); rank = #{i : !isMuchSmallerThan(d_i, d_0)} (|d_i| <= |d_0| 1e-5f);
//                    rank == 2: R = U V^T when det U det V > 0, else U diag(1, 1, -1) V^T; otherwise R = U S V^T; t = dst_mean - R src_mean.
//   RECORDED DOUBT   PCL 1.10 ships its own pcl::umeyama (common/eigen.h, "patched version until Eigen is released") and this reference
//                    takes it to carry the Eigen 3.2 rank branch above, not only Eigen 3.3's det U det V < 0 rule.  The two differ only
//                    when sigma has rank 2 (all correspondences on one plane, as ground-only scans are); test_icp_pcl_oracle's planar
//                    case pins the choice so that a correction shows up.
//   UPSTREAM-RECALL  JacobiSVD (Eigen 3.3.7, square: no QR preconditioner): scale = max |a_ij| (1 if 0); W = A / scale; sweeps over
//                    (p, q) = (1, 0), (2, 0), (2, 1) while |W_pq| or |W_qp| > max(FLT_MIN, 2 FLT_EPSILON maxDiagEntry);
//                    real_2x2_jacobi_svd (rot1 from t = m00 + m11, d = m10 - m01; makeJacobi; j_left = rot1 j_right^T);
//                    apply_rotation_in_the_plane returns early for (c, s) == (1, 0); singular values |W_ii| (U's column negated for a
//                    negative one) times scale, then a selection sort (first maximum wins, stop at a zero).  No isfinite check of the
//                    scale (sigma is finite here).
//   UPSTREAM-RECALL  a 3-term coefficient of a small fixed-size product (U S V^T, R src_mean) is x0 + (x1 + x2) (redux_novec_unroller).
//   ENGINE RULE      the sums (count, sum d2, sum src, sum tgt) and the demeaned cross products are accumulated in float64, products
//                    of the float32 demeaned coordinates exact; means = (float)(S / n); demeaning in float32 per point as Eigen does it;
//                    sigma = (float)(C / n) before the float32 SVD.  PCL sums in float in an order a device cannot reproduce (a strided
//                    sequential redux and Eigen's blocked GEMM).  Here the sums are sequential; the device reduces through its fixed tree.
// DefaultConvergenceCriteria::hasConverged
//   UPSTREAM-RECALL  iterations >= max -> true (failure_after_max_iter_ = false).
//   UPSTREAM-RECALL  cos = 0.5 (double)(((t00 + t11) + t22) - 1.0f) (float sum, double product); tsq = (double)((t03 t03 + t13 t13) + t23 t23)
//                    (float32); cos >= 1 - eps && tsq <= eps -> true.  eps is compared with the SQUARED translation.
//   UPSTREAM-RECALL  mse = sum distance / n in double over this iteration's correspondences (measured before the step);
//                    |mse - prev| < 1e-12 -> true; prev starts at DBL_MAX; max_iterations_similar_transforms_ = 0.
// Empty clouds: initCompute fails, the guess, not converged, no iteration (as every other method).
#include <cfloat>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <unordered_map>
#include <vector>

namespace {

struct P3 { float x, y, z; };

bool finite3(float x, float y, float z) { return std::isfinite(x) && std::isfinite(y) && std::isfinite(z); }
float dist2(const P3& a, const P3& b) {
  const float dx = a.x - b.x, dy = a.y - b.y, dz = a.z - b.z;
  return (dx * dx + dy * dy) + dz * dz;
}
P3 xform(const float* M, const P3& p) {  // row-major 4x4
  return {((M[0] * p.x + M[1] * p.y) + M[2] * p.z) + M[3], ((M[4] * p.x + M[5] * p.y) + M[6] * p.z) + M[7],
          ((M[8] * p.x + M[9] * p.y) + M[10] * p.z) + M[11]};
}

// exact 1-NN restricted to candidates within max_dist: a uniform grid of cells a little wider than max_dist, the 27 cells around the
// query.  Any point within max_dist lies in them, so the smallest (d2, index) found is the global 1-NN whenever that one is accepted.
struct Grid {
  double cell;
  const std::vector<P3>* pts;
  const std::vector<char>* valid;
  std::unordered_map<long long, std::vector<int>> cells;
  static long long key(long long x, long long y, long long z) { return ((x + (1ll << 20)) << 42) | ((y + (1ll << 20)) << 21) | (z + (1ll << 20)); }
  void build(const std::vector<P3>& p, const std::vector<char>& v, double max_dist) {
    cell = max_dist * 1.01 + 1e-30;
    pts = &p; valid = &v;
    cells.clear();
    for (size_t i = 0; i < p.size(); i++)
      if (v[i]) cells[key((long long)std::floor(p[i].x / cell), (long long)std::floor(p[i].y / cell), (long long)std::floor(p[i].z / cell))].push_back((int)i);
  }
  // index of the 1-NN within the cells (-1 if none), its d2
  int nearest(const P3& q, float* d2) const {
    const long long cx = (long long)std::floor(q.x / cell), cy = (long long)std::floor(q.y / cell), cz = (long long)std::floor(q.z / cell);
    int best = -1;
    float bd = INFINITY;
    for (long long a = -1; a <= 1; a++)
      for (long long b = -1; b <= 1; b++)
        for (long long c = -1; c <= 1; c++) {
          auto it = cells.find(key(cx + a, cy + b, cz + c));
          if (it == cells.end()) continue;
          for (int j : it->second) {
            const float d = dist2(q, (*pts)[j]);
            if (d < bd || (d == bd && j < best)) { bd = d; best = j; }
          }
        }
    *d2 = bd;
    return best;
  }
};

// ---- Eigen 3.3.7 JacobiSVD<Matrix3f>, restated with its JacobiRotation objects (matrices row-major)
struct Rot { float c, s; };
Rot mul(const Rot& a, const Rot& b) { return {a.c * b.c - a.s * b.s, a.c * b.s + a.s * b.c}; }  // operator*, real
Rot transpose(const Rot& j) { return {j.c, -j.s}; }
void apply_plane(float* x0, float* x1, float* x2, float* y0, float* y1, float* y2, const Rot& j) {
  if (j.c == 1.0f && j.s == 0.0f) return;
  float* xs[3] = {x0, x1, x2};
  float* ys[3] = {y0, y1, y2};
  for (int i = 0; i < 3; i++) {
    const float xi = *xs[i], yi = *ys[i];
    *xs[i] = j.c * xi + j.s * yi;
    *ys[i] = -j.s * xi + j.c * yi;
  }
}
void on_left(float* M, int p, int q, const Rot& j) { apply_plane(&M[p * 3], &M[p * 3 + 1], &M[p * 3 + 2], &M[q * 3], &M[q * 3 + 1], &M[q * 3 + 2], j); }
void on_right(float* M, int p, int q, const Rot& j) { apply_plane(&M[p], &M[3 + p], &M[6 + p], &M[q], &M[3 + q], &M[6 + q], transpose(j)); }
Rot make_jacobi(float x, float y, float z) {
  const float deno = 2.0f * std::fabs(y);
  if (deno < FLT_MIN) return {1.0f, 0.0f};
  const float tau = (x - z) / deno;
  const float w = std::sqrt(tau * tau + 1.0f);
  const float t = tau > 0.0f ? 1.0f / (tau + w) : 1.0f / (tau - w);
  const float sign_t = t > 0.0f ? 1.0f : -1.0f;
  const float n = 1.0f / std::sqrt(t * t + 1.0f);
  return {n, -sign_t * (y / std::fabs(y)) * std::fabs(t) * n};
}
void real_2x2_jacobi_svd(const float* W, int p, int q, Rot* jl, Rot* jr) {
  float m[4] = {W[p * 3 + p], W[p * 3 + q], W[q * 3 + p], W[q * 3 + q]};
  const float t = m[0] + m[3], d = m[2] - m[1];
  Rot rot1;
  if (std::fabs(d) < FLT_MIN) rot1 = {1.0f, 0.0f};
  else {
    const float u = t / d;
    const float tmp = std::sqrt(1.0f + u * u);
    rot1 = {u / tmp, 1.0f / tmp};
  }
  if (!(rot1.c == 1.0f && rot1.s == 0.0f)) {  // m.applyOnTheLeft(0, 1, rot1)
    const float a0 = m[0], a1 = m[1], b0 = m[2], b1 = m[3];
    m[0] = rot1.c * a0 + rot1.s * b0; m[1] = rot1.c * a1 + rot1.s * b1;
    m[2] = -rot1.s * a0 + rot1.c * b0; m[3] = -rot1.s * a1 + rot1.c * b1;
  }
  *jr = make_jacobi(m[0], m[1], m[3]);
  *jl = mul(rot1, transpose(*jr));
}
void jacobi_svd(const float* A, float* U, float* d, float* V) {
  float scale = 0.0f;
  for (int i = 0; i < 9; i++) scale = std::max(scale, std::fabs(A[i]));
  if (scale == 0.0f) scale = 1.0f;
  float W[9];
  for (int i = 0; i < 9; i++) { W[i] = A[i] / scale; U[i] = V[i] = (i % 4 == 0) ? 1.0f : 0.0f; }
  const float precision = 2.0f * FLT_EPSILON, consider_zero = FLT_MIN;
  float maxd = std::max(std::max(std::fabs(W[0]), std::fabs(W[4])), std::fabs(W[8]));
  bool finished = false;
  while (!finished) {
    finished = true;
    for (int p = 1; p < 3; p++)
      for (int q = 0; q < p; q++) {
        const float threshold = std::max(consider_zero, precision * maxd);
        if (std::fabs(W[p * 3 + q]) > threshold || std::fabs(W[q * 3 + p]) > threshold) {
          finished = false;
          Rot jl, jr;
          real_2x2_jacobi_svd(W, p, q, &jl, &jr);
          on_left(W, p, q, jl);
          on_right(U, p, q, transpose(jl));
          on_right(W, p, q, jr);
          on_right(V, p, q, jr);
          maxd = std::max(maxd, std::max(std::fabs(W[p * 4]), std::fabs(W[q * 4])));
        }
      }
  }
  for (int i = 0; i < 3; i++) {
    const float a = W[i * 4];
    d[i] = std::fabs(a);
    if (a < 0.0f)
      for (int k = 0; k < 3; k++) U[k * 3 + i] = -U[k * 3 + i];
  }
  for (int i = 0; i < 3; i++) d[i] *= scale;
  for (int i = 0; i < 3; i++) {
    int pos = i;
    for (int j = i + 1; j < 3; j++)
      if (d[j] > d[pos]) pos = j;
    if (d[pos] == 0.0f) break;
    if (pos != i) {
      std::swap(d[i], d[pos]);
      for (int k = 0; k < 3; k++) { std::swap(U[k * 3 + i], U[k * 3 + pos]); std::swap(V[k * 3 + i], V[k * 3 + pos]); }
    }
  }
}
float det3(const float* m) {
  return (m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6])) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}
float coeff3(float a0, float b0, float a1, float b1, float a2, float b2) { return a0 * b0 + (a1 * b1 + a2 * b2); }
void umeyama(const float* sigma, const float* sm, const float* dm, float* Rt) {
  float U[9], d[3], V[9];
  jacobi_svd(sigma, U, d, V);
  float S[3] = {1.0f, 1.0f, 1.0f};
  if (det3(sigma) < 0.0f) S[2] = -1.0f;
  int rank = 0;
  for (int i = 0; i < 3; i++)
    if (!(std::fabs(d[i]) <= std::fabs(d[0]) * 1e-5f)) ++rank;
  float Sx[3] = {S[0], S[1], S[2]};
  if (rank == 2) Sx[2] = det3(U) * det3(V) > 0.0f ? 1.0f : -1.0f;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      Rt[i * 4 + j] = coeff3(U[i * 3] * Sx[0], V[j * 3], U[i * 3 + 1] * Sx[1], V[j * 3 + 1], U[i * 3 + 2] * Sx[2], V[j * 3 + 2]);
  for (int i = 0; i < 3; i++) Rt[i * 4 + 3] = dm[i] - coeff3(Rt[i * 4], sm[0], Rt[i * 4 + 1], sm[1], Rt[i * 4 + 2], sm[2]);
  Rt[12] = Rt[13] = Rt[14] = 0.0f;
  Rt[15] = 1.0f;
}
bool has_converged(const float* T, int iterations, int max_iterations, double rot_thr, double trans_thr, double mse, double* prev) {
  if (iterations >= max_iterations) return true;
  const double cos_angle = 0.5 * (T[0] + T[5] + T[10] - 1);
  const double tsq = T[3] * T[3] + T[7] * T[7] + T[11] * T[11];
  if (cos_angle >= rot_thr && tsq <= trans_thr) return true;
  if (std::fabs(mse - *prev) < 1e-12) return true;
  *prev = mse;
  return false;
}
void mul4(const float* A, const float* B, float* O) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) O[i * 4 + j] = ((A[i * 4] * B[j] + A[i * 4 + 1] * B[4 + j]) + A[i * 4 + 2] * B[8 + j]) + A[i * 4 + 3] * B[12 + j];
}

std::vector<P3> load(const float* pts, size_t n, size_t stride_f, std::vector<char>& valid) {
  std::vector<P3> p(n);
  valid.assign(n, 0);
  for (size_t i = 0; i < n; i++) {
    p[i] = {pts[i * stride_f], pts[i * stride_f + 1], pts[i * stride_f + 2]};
    valid[i] = finite3(p[i].x, p[i].y, p[i].z);
  }
  return p;
}

struct Corr { int i, j; float d2; };

// determineCorrespondences / determineReciprocalCorrespondences of the moved source `q`
std::vector<Corr> correspondences(const std::vector<P3>& q, const std::vector<char>& qv, const std::vector<P3>& t, const Grid& tg,
                                  double max_dist, bool reciprocal) {
  const double thr2 = max_dist * max_dist;
  std::vector<char> mv(q.size());
  for (size_t i = 0; i < q.size(); i++) mv[i] = qv[i] && finite3(q[i].x, q[i].y, q[i].z);
  Grid sg;
  if (reciprocal) sg.build(q, mv, max_dist);
  std::vector<Corr> out;
  for (size_t i = 0; i < q.size(); i++) {
    if (!mv[i]) continue;
    float d2;
    const int j = tg.nearest(q[i], &d2);
    if (j < 0 || (double)d2 > thr2) continue;
    if (reciprocal) {
      float d2r;
      const int k = sg.nearest(t[j], &d2r);
      if (k < 0 || (double)d2r > thr2 || k != (int)i) continue;
    }
    out.push_back({(int)i, j, d2});
  }
  return out;
}

// TransformationEstimationSVD on the correspondences; sums[17] as b2r_icp_pcl_estimate_at; Rt row-major
void estimate(const std::vector<P3>& q, const std::vector<P3>& t, const std::vector<Corr>& C, float* Rt, double* sums) {
  double S[17] = {0};
  for (const Corr& c : C) {
    S[0] += 1.0; S[1] += (double)c.d2;
    S[2] += (double)q[c.i].x; S[3] += (double)q[c.i].y; S[4] += (double)q[c.i].z;
    S[5] += (double)t[c.j].x; S[6] += (double)t[c.j].y; S[7] += (double)t[c.j].z;
  }
  const double n = S[0];
  float sm[3], dm[3];
  for (int k = 0; k < 3; k++) { sm[k] = (float)(S[2 + k] / n); dm[k] = (float)(S[5 + k] / n); }
  for (const Corr& c : C) {
    const float sd[3] = {q[c.i].x - sm[0], q[c.i].y - sm[1], q[c.i].z - sm[2]};
    const float dd[3] = {t[c.j].x - dm[0], t[c.j].y - dm[1], t[c.j].z - dm[2]};
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) S[8 + a * 3 + b] += (double)dd[a] * (double)sd[b];
  }
  float sigma[9];
  for (int k = 0; k < 9; k++) sigma[k] = (float)(S[8 + k] / n);
  umeyama(sigma, sm, dm, Rt);
  if (sums) std::memcpy(sums, S, sizeof(S));
}

std::vector<P3> moved(const std::vector<P3>& s, const std::vector<char>& v, const float* T) {
  std::vector<P3> q(s);
  for (size_t i = 0; i < s.size(); i++)
    if (v[i]) q[i] = xform(T, s[i]);
  return q;
}

}  // namespace

extern "C" {

void ref_icp_svd(const float* A, float* U, float* d, float* V) { jacobi_svd(A, U, d, V); }
void ref_icp_umeyama(const float* sigma, const float* sm, const float* dm, float* Rt) { umeyama(sigma, sm, dm, Rt); }
int ref_icp_has_converged(const float* T, int iterations, int max_iterations, double rot_thr, double trans_thr, double mse, double* prev) {
  return has_converged(T, iterations, max_iterations, rot_thr, trans_thr, mse, prev) ? 1 : 0;
}

// the source transformed once by T (row-major), one correspondence pass: corr / d2 per source point (-1 / NaN where none); returns the count
size_t ref_icp_correspondences(const float* src, size_t ns, size_t sf, const float* tgt, size_t nt, size_t tf, const float* T, double max_dist,
                               int reciprocal, int32_t* corr, float* d2) {
  std::vector<char> sv, tv;
  const std::vector<P3> s = load(src, ns, sf, sv), t = load(tgt, nt, tf, tv);
  Grid tg;
  tg.build(t, tv, max_dist);
  const std::vector<Corr> C = correspondences(moved(s, sv, T), sv, t, tg, max_dist, reciprocal != 0);
  for (size_t i = 0; i < ns; i++) { corr[i] = -1; d2[i] = NAN; }
  for (const Corr& c : C) { corr[c.i] = c.j; d2[c.i] = c.d2; }
  return C.size();
}

// the same pass, then the estimation: Rt row-major, sums[17]; returns the count (no estimate below 3)
size_t ref_icp_estimate(const float* src, size_t ns, size_t sf, const float* tgt, size_t nt, size_t tf, const float* T, double max_dist, int reciprocal,
                        float* Rt, double* sums) {
  std::vector<char> sv, tv;
  const std::vector<P3> s = load(src, ns, sf, sv), t = load(tgt, nt, tf, tv);
  Grid tg;
  tg.build(t, tv, max_dist);
  const std::vector<P3> q = moved(s, sv, T);
  const std::vector<Corr> C = correspondences(q, sv, t, tg, max_dist, reciprocal != 0);
  if (C.size() >= 3) estimate(q, t, C, Rt, sums);
  return C.size();
}

// computeTransformation: T (row-major out), stats = {converged, iterations}; counts[0 .. cap) = correspondences per loop pass.
// Returns the number of loop passes.
size_t ref_icp_align(const float* src, size_t ns, size_t sf, const float* tgt, size_t nt, size_t tf, const float* guess, double eps, double max_dist,
                     int max_iterations, int reciprocal, float* T, int64_t* stats, int64_t* counts, size_t cap) {
  std::memcpy(T, guess, 16 * sizeof(float));
  stats[0] = 0; stats[1] = 0;
  if (ns == 0 || nt == 0) return 0;
  std::vector<char> sv, tv;
  const std::vector<P3> s = load(src, ns, sf, sv), t = load(tgt, nt, tf, tv);
  Grid tg;
  tg.build(t, tv, max_dist);
  bool ident = true;
  for (int i = 0; i < 16; i++) ident = ident && guess[i] == ((i % 5 == 0) ? 1.0f : 0.0f);
  std::vector<P3> q = ident ? s : moved(s, sv, guess);
  double prev = DBL_MAX;
  int it = 0;
  size_t passes = 0;
  for (;;) {
    const std::vector<Corr> C = correspondences(q, sv, t, tg, max_dist, reciprocal != 0);
    if (passes < cap) counts[passes] = (int64_t)C.size();
    passes++;
    if (C.size() < 3) { stats[0] = 0; break; }
    float Rt[16], F[16];
    estimate(q, t, C, Rt, nullptr);
    for (size_t i = 0; i < q.size(); i++)
      if (sv[i]) q[i] = xform(Rt, q[i]);
    mul4(Rt, T, F);
    std::memcpy(T, F, sizeof(F));
    ++it;
    double mse = 0.0;
    for (const Corr& c : C) mse += (double)c.d2;
    mse /= (double)C.size();
    if (has_converged(Rt, it, max_iterations, 1.0 - eps, eps, mse, &prev)) { stats[0] = 1; break; }
  }
  stats[1] = it;
  return passes;
}

}  // extern "C"
