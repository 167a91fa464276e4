// oracle/gicp.cpp — TEST INFRASTRUCTURE ONLY (CPU oracle; see oracle.h header).
//
// Restates fast_gicp::FastGICP + fast_gicp::LsqRegistration + so3.hpp (SURVEY.md Appendix A.4), the engine the
// reference selects at /root/reference/src/hdl_graph_slam/registrations.cpp:27-36 and drives at
// apps/scan_matching_odometry_nodelet.cpp:172,177,210 and include/hdl_graph_slam/loop_detector.hpp:122,136,143.
// "parity unpinned": fast_gicp is an un-vendored, unpinned dependency and the reference has no tests.
#include "oracle.h"
#include "kdtree.hpp"
#include "linalg.hpp"
#include <omp.h>
#include <vector>
#include <cstdio>
#include <cfloat>

using namespace orc;

extern "C" int orc_max_threads(void) { return omp_get_max_threads(); }

static inline int nthreads(int t) { return t > 0 ? t : omp_get_max_threads(); }

extern "C" void orc_knn(const float* pts, size_t n, size_t stride, const float* queries, size_t nq, size_t qstride, int k,
                        int32_t* idx_out, float* d2_out, int threads) {
  KdTree tree;
  tree.build(pts, n, stride);
#pragma omp parallel for num_threads(nthreads(threads)) schedule(static)
  for (long i = 0; i < (long)nq; i++) {
    int* io = idx_out + (size_t)i * k;
    float* dout = d2_out + (size_t)i * k;
    int c = tree.knn(queries + (size_t)i * qstride, k, io, dout);
    for (int j = c; j < k; j++) { io[j] = -1; dout[j] = INFINITY; }
  }
}

// fast_gicp calculate_covariances (A.4): exact kNN incl. self, centred outer product / k, PLANE regularisation.
static void covariances(const KdTree& tree, const float* pts, size_t n, size_t stride, int k, double* cov_out, int threads) {
#pragma omp parallel for num_threads(nthreads(threads)) schedule(static)
  for (long i = 0; i < (long)n; i++) {
    std::vector<int> idx(k);
    std::vector<float> d2(k);
    int kk = tree.knn(pts + (size_t)i * stride, k, idx.data(), d2.data());
    double mean[3] = {0, 0, 0};
    for (int j = 0; j < kk; j++) {
      const float* p = pts + (size_t)idx[j] * stride;
      mean[0] += (double)p[0]; mean[1] += (double)p[1]; mean[2] += (double)p[2];
    }
    for (int d = 0; d < 3; d++) mean[d] /= (double)kk;
    double c[9] = {0};
    for (int j = 0; j < kk; j++) {
      const float* p = pts + (size_t)idx[j] * stride;
      double v[3] = {(double)p[0] - mean[0], (double)p[1] - mean[1], (double)p[2] - mean[2]};
      for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) c[a * 3 + b] += v[a] * v[b];
    }
    for (int a = 0; a < 9; a++) c[a] /= (double)kk;
    // PLANE: JacobiSVD(cov) -> U diag(1,1,1e-3) V^T; for a symmetric PSD matrix U = V = eigenvectors, values descending.
    double w[3], V[9];
    sym_eigen<3>(c, w, V);  // ascending: V col 2 = largest
    // exactly diagonal (an axis-aligned line, or all k neighbours one point): the eigenvalues tie and the ascending Jacobi above
    // would pick its own column; JacobiSVD's is the one its step-4 sort leaves last (linalg.hpp diagonal_normal).  UPSTREAM-RECALL
    if (c[1] == 0.0 && c[2] == 0.0 && c[5] == 0.0) diagonal_normal(c, V);
    const double vals[3] = {1e-3, 1.0, 1.0};  // smallest eigenvalue -> 1e-3
    double* o = cov_out + (size_t)i * 9;
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) {
        double s = 0.0;
        for (int e = 2; e >= 0; e--) s += vals[e] * V[a * 3 + e] * V[b * 3 + e];
        o[a * 3 + b] = s;
      }
  }
}

extern "C" void orc_gicp_covariances(const float* pts, size_t n, size_t stride, int k, double* cov_out, int threads) {
  KdTree tree;
  tree.build(pts, n, stride);
  covariances(tree, pts, n, stride, k, cov_out, threads);
}

// float32 transform exactly as Eigen's 4x4 * 4-vector column accumulation / pcl::transformPoint without FMA:
// ((m0*x + m1*y) + m2*z) + m3
static inline void xform_f32(const float* Tf /*row-major 4x4*/, const float* p, float* o) {
  for (int r = 0; r < 3; r++) {
    float a = Tf[r * 4 + 0] * p[0];
    float b = Tf[r * 4 + 1] * p[1];
    float c = Tf[r * 4 + 2] * p[2];
    float s = a + b;
    s = s + c;
    o[r] = s + Tf[r * 4 + 3];
  }
}

struct LinAcc {
  double H[36];
  double b[6];
  double e;
  char pad[64];
};

static double linearize_impl(const KdTree& ttree, const float* src, size_t n, size_t sstride, const double* src_cov,
                             const float* tgt, size_t tstride, const double* tgt_cov, const double* T, double max_corr_dist,
                             int32_t* corr, float* d2o, double* mahal, double* H, double* b, int threads) {
  float Tf[16];
  for (int i = 0; i < 16; i++) Tf[i] = (float)T[i];
  const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
  const double thr2 = max_corr_dist * max_corr_dist;
  int nt = nthreads(threads);
  std::vector<LinAcc> acc(nt);
  for (auto& a : acc) { std::memset(a.H, 0, sizeof(a.H)); std::memset(a.b, 0, sizeof(a.b)); a.e = 0; }
#pragma omp parallel num_threads(nt)
  {
    LinAcc& A = acc[omp_get_thread_num()];
#pragma omp for schedule(static)
    for (long i = 0; i < (long)n; i++) {
      const float* p = src + (size_t)i * sstride;
      float q[3];
      xform_f32(Tf, p, q);
      int idx;
      float d2;
      int c = ttree.knn(q, 1, &idx, &d2);
      if (c == 0) { corr[i] = -1; d2o[i] = INFINITY; continue; }
      d2o[i] = d2;
      corr[i] = ((double)d2 < thr2) ? idx : -1;
      if (corr[i] < 0) continue;
      // M = (C_B + R C_A R^T)^-1
      const double* CA = src_cov + (size_t)i * 9;
      const double* CB = tgt_cov + (size_t)idx * 9;
      double tmp[9], rcr[9], M[9];
      mul3(R, CA, tmp);
      mul3_abt(tmp, R, rcr);
      for (int a = 0; a < 9; a++) rcr[a] = CB[a] + rcr[a];
      inv3(rcr, M);
      if (mahal) std::memcpy(mahal + (size_t)i * 9, M, sizeof(M));
      // residual
      const float* tb = tgt + (size_t)idx * tstride;
      double a3[3] = {(double)p[0], (double)p[1], (double)p[2]};
      double tA[3], e[3];
      for (int r = 0; r < 3; r++) tA[r] = T[r * 4 + 0] * a3[0] + T[r * 4 + 1] * a3[1] + T[r * 4 + 2] * a3[2] + T[r * 4 + 3];
      for (int r = 0; r < 3; r++) e[r] = (double)tb[r] - tA[r];
      double Me[3];
      for (int r = 0; r < 3; r++) Me[r] = M[r * 3 + 0] * e[0] + M[r * 3 + 1] * e[1] + M[r * 3 + 2] * e[2];
      A.e += e[0] * Me[0] + e[1] * Me[1] + e[2] * Me[2];
      // J = [skew(tA) | -I]  (3x6)
      double J[18] = {0.0, -tA[2], tA[1], -1, 0, 0, tA[2], 0.0, -tA[0], 0, -1, 0, -tA[1], tA[0], 0.0, 0, 0, -1};
      double MJ[18];
      for (int r = 0; r < 3; r++)
        for (int cc = 0; cc < 6; cc++) MJ[r * 6 + cc] = M[r * 3 + 0] * J[0 * 6 + cc] + M[r * 3 + 1] * J[1 * 6 + cc] + M[r * 3 + 2] * J[2 * 6 + cc];
      for (int r = 0; r < 6; r++) {
        for (int cc = 0; cc < 6; cc++) A.H[r * 6 + cc] += J[0 * 6 + r] * MJ[0 * 6 + cc] + J[1 * 6 + r] * MJ[1 * 6 + cc] + J[2 * 6 + r] * MJ[2 * 6 + cc];
        A.b[r] += J[0 * 6 + r] * Me[0] + J[1 * 6 + r] * Me[1] + J[2 * 6 + r] * Me[2];
      }
    }
  }
  std::memset(H, 0, 36 * sizeof(double));
  std::memset(b, 0, 6 * sizeof(double));
  double e = 0;
  for (int t = 0; t < nt; t++) {
    for (int i = 0; i < 36; i++) H[i] += acc[t].H[i];
    for (int i = 0; i < 6; i++) b[i] += acc[t].b[i];
    e += acc[t].e;
  }
  return e;
}

static double error_impl(const float* src, size_t n, size_t sstride, const float* tgt, size_t tstride, const int32_t* corr,
                         const double* mahal, const double* T, int threads) {
  double sum = 0.0;
  int nt = nthreads(threads);
  std::vector<LinAcc> acc(nt);
  for (auto& a : acc) a.e = 0;
#pragma omp parallel num_threads(nt)
  {
    LinAcc& A = acc[omp_get_thread_num()];
#pragma omp for schedule(static)
    for (long i = 0; i < (long)n; i++) {
      int idx = corr[i];
      if (idx < 0) continue;
      const float* p = src + (size_t)i * sstride;
      const float* tb = tgt + (size_t)idx * tstride;
      const double* M = mahal + (size_t)i * 9;
      double a3[3] = {(double)p[0], (double)p[1], (double)p[2]};
      double e[3];
      for (int r = 0; r < 3; r++) e[r] = (double)tb[r] - (T[r * 4 + 0] * a3[0] + T[r * 4 + 1] * a3[1] + T[r * 4 + 2] * a3[2] + T[r * 4 + 3]);
      double Me[3];
      for (int r = 0; r < 3; r++) Me[r] = M[r * 3 + 0] * e[0] + M[r * 3 + 1] * e[1] + M[r * 3 + 2] * e[2];
      A.e += e[0] * Me[0] + e[1] * Me[1] + e[2] * Me[2];
    }
  }
  for (int t = 0; t < nt; t++) sum += acc[t].e;
  return sum;
}

extern "C" double orc_gicp_linearize(const float* src, size_t n, size_t sstride, const double* src_cov, const float* tgt, size_t m,
                                     size_t tstride, const double* tgt_cov, const double* T, double max_corr_dist,
                                     int32_t* corr_out, float* d2_out, double* mahal_out, double* H, double* b, int threads) {
  KdTree tree;
  tree.build(tgt, m, tstride);
  return linearize_impl(tree, src, n, sstride, src_cov, tgt, tstride, tgt_cov, T, max_corr_dist, corr_out, d2_out, mahal_out, H, b, threads);
}

extern "C" double orc_gicp_error(const float* src, size_t n, size_t sstride, const float* tgt, size_t tstride, const int32_t* corr,
                                 const double* mahal, const double* T, int threads) {
  return error_impl(src, n, sstride, tgt, tstride, corr, mahal, T, threads);
}

// ---- so3.hpp restatement (A.4) -------------------------------------------------------------------------------
static void se3_exp(const double* a, double* D /*4x4 row-major*/) {
  const double ox = a[0], oy = a[1], oz = a[2];
  double theta_sq = ox * ox + oy * oy + oz * oz;
  double theta = std::sqrt(theta_sq);
  // so3_exp -> quaternion (w, x, y, z)
  double imag, real;
  if (theta_sq < 1e-10) {
    double theta_quad = theta_sq * theta_sq;
    imag = 0.5 - 1.0 / 48.0 * theta_sq + 1.0 / 3840.0 * theta_quad;
    real = 1.0 - 1.0 / 8.0 * theta_sq + 1.0 / 384.0 * theta_quad;
  } else {
    double th = std::sqrt(theta_sq);
    double half = 0.5 * th;
    imag = std::sin(half) / th;
    real = std::cos(half);
  }
  double qw = real, qx = imag * ox, qy = imag * oy, qz = imag * oz;
  // Eigen::Quaternion::toRotationMatrix
  double tx = 2 * qx, ty = 2 * qy, tz = 2 * qz;
  double twx = tx * qw, twy = ty * qw, twz = tz * qw;
  double txx = tx * qx, txy = ty * qx, txz = tz * qx;
  double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  double R[9] = {1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)};
  double Om[9] = {0, -oz, oy, oz, 0, -ox, -oy, ox, 0};
  double Om2[9];
  mul3(Om, Om, Om2);
  double V[9];
  if (theta < 1e-10) {
    std::memcpy(V, R, sizeof(V));
  } else {
    double c1 = (1.0 - std::cos(theta)) / theta_sq;
    double c2 = (theta - std::sin(theta)) / (theta_sq * theta);
    for (int i = 0; i < 9; i++) V[i] = ((i % 4 == 0) ? 1.0 : 0.0) + c1 * Om[i] + c2 * Om2[i];
  }
  for (int i = 0; i < 16; i++) D[i] = 0;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) D[r * 4 + c] = R[r * 3 + c];
    D[r * 4 + 3] = V[r * 3 + 0] * a[3] + V[r * 3 + 1] * a[4] + V[r * 3 + 2] * a[5];
  }
  D[15] = 1.0;
}

static bool is_converged(const double* D, double rot_eps, double trans_eps) {
  double mr = 0, mt = 0;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) mr = std::max(mr, 1.0 / rot_eps * std::fabs(D[r * 4 + c] - (r == c ? 1.0 : 0.0)));
    mt = std::max(mt, 1.0 / trans_eps * std::fabs(D[r * 4 + 3]));
  }
  return std::max(mr, mt) < 1;
}

static void mul4_iso(const double* A, const double* B, double* O) {  // Isometry3d product (affine part), last row 0 0 0 1
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 4; c++) {
      double s = A[r * 4 + 0] * B[0 * 4 + c] + A[r * 4 + 1] * B[1 * 4 + c] + A[r * 4 + 2] * B[2 * 4 + c];
      if (c == 3) s += A[r * 4 + 3];
      O[r * 4 + c] = s;
    }
  }
  O[12] = O[13] = O[14] = 0;
  O[15] = 1;
}

// fast_gicp keeps the target's kd-tree and covariances for as long as the same target cloud is set (setInputTarget early-outs on
// the same pointer; A.4): a target context holds them across align() calls — used by the CPU baseline so that the per-frame /
// per-candidate cost is what the reference pays (source kd-tree + source covariances + align), not a rebuilt target tree.
struct orc_gicp_target {
  KdTree tree;
  std::vector<double> cov;
  const float* pts;
  size_t m, stride;
};

static void align_impl(const KdTree& ttree, const float* src, size_t n, size_t sstride, const double* src_cov_in, const float* tgt, size_t m,
                       size_t tstride, const double* tgt_cov_in, const orc_gicp_config* cfg, const float* guess,
                       orc_gicp_result* res, double* trace_H, double* trace_b, double* trace_y, int32_t* corr_out);

extern "C" orc_gicp_target* orc_gicp_target_create(const float* tgt, size_t m, size_t stride, int k, int threads) {
  orc_gicp_target* t = new orc_gicp_target();
  t->pts = tgt; t->m = m; t->stride = stride;
  if (m) {
    t->tree.build(tgt, m, stride);
    t->cov.resize(m * 9);
    covariances(t->tree, tgt, m, stride, k, t->cov.data(), threads);
  }
  return t;
}
extern "C" void orc_gicp_target_free(orc_gicp_target* t) { delete t; }
extern "C" void orc_gicp_align_to(const orc_gicp_target* t, const float* src, size_t n, size_t sstride, const double* src_cov, const orc_gicp_config* cfg,
                                  const float* guess, orc_gicp_result* res, int32_t* corr_out) {
  std::memset(res, 0, sizeof(*res));
  for (int i = 0; i < 16; i++) { res->T[i] = guess[i]; res->T64[i] = (double)guess[i]; }
  if (n == 0 || t->m == 0) return;
  align_impl(t->tree, src, n, sstride, src_cov, t->pts, t->m, t->stride, t->cov.data(), cfg, guess, res, nullptr, nullptr, nullptr, corr_out);
}
// getFitnessScore against a kept target (same arithmetic as orc_fitness)
extern "C" double orc_gicp_target_fitness(const orc_gicp_target* t, const float* src, size_t n, size_t sstride, const float* T, double max_range, int threads) {
  std::vector<float> d2(n);
  std::vector<int32_t> idx(n);
#pragma omp parallel for num_threads(nthreads(threads)) schedule(static)
  for (long i = 0; i < (long)n; i++) {
    float q[3];
    xform_f32(T, src + (size_t)i * sstride, q);
    int id = -1;
    float d = INFINITY;
    t->tree.knn(q, 1, &id, &d);
    d2[i] = d;
    idx[i] = id;
  }
  double sum = 0;
  uint32_t nr = 0;
  for (size_t i = 0; i < n; i++) {
    if (idx[i] < 0) continue;
    if ((double)d2[i] <= max_range) { sum += (double)d2[i]; nr++; }
  }
  return nr > 0 ? sum / nr : DBL_MAX;
}

extern "C" void orc_gicp_align(const float* src, size_t n, size_t sstride, const double* src_cov_in, const float* tgt, size_t m,
                               size_t tstride, const double* tgt_cov_in, const orc_gicp_config* cfg, const float* guess,
                               orc_gicp_result* res, double* trace_H, double* trace_b, double* trace_y, int32_t* corr_out) {
  std::memset(res, 0, sizeof(*res));
  for (int i = 0; i < 16; i++) { res->T[i] = guess[i]; res->T64[i] = (double)guess[i]; }
  if (n == 0 || m == 0) return;  // pcl::Registration::initCompute fails silently -> converged_ stays false
  KdTree ttree;
  ttree.build(tgt, m, tstride);
  align_impl(ttree, src, n, sstride, src_cov_in, tgt, m, tstride, tgt_cov_in, cfg, guess, res, trace_H, trace_b, trace_y, corr_out);
}

static void align_impl(const KdTree& ttree, const float* src, size_t n, size_t sstride, const double* src_cov_in, const float* tgt, size_t m,
                       size_t tstride, const double* tgt_cov_in, const orc_gicp_config* cfg, const float* guess,
                       orc_gicp_result* res, double* trace_H, double* trace_b, double* trace_y, int32_t* corr_out) {
  const int threads = cfg->num_threads;
  std::vector<double> scov_s, tcov_s;
  const double* scov = src_cov_in;
  const double* tcov = tgt_cov_in;
  if (!scov) {
    KdTree stree;
    stree.build(src, n, sstride);
    scov_s.resize(n * 9);
    covariances(stree, src, n, sstride, cfg->k_correspondences, scov_s.data(), threads);
    scov = scov_s.data();
  }
  if (!tcov) {
    tcov_s.resize(m * 9);
    covariances(ttree, tgt, m, tstride, cfg->k_correspondences, tcov_s.data(), threads);
    tcov = tcov_s.data();
  }

  std::vector<int32_t> corr(n);
  std::vector<float> d2(n);
  std::vector<double> mahal(n * 9);

  double x0[16];
  for (int i = 0; i < 16; i++) x0[i] = (double)guess[i];
  x0[12] = x0[13] = x0[14] = 0; x0[15] = 1;
  double lambda = -1.0;
  bool converged = false;
  int it = 0, total_inner = 0;
  bool lm_failed = false;
  double y0 = 0;
  for (it = 0; it < cfg->max_iterations && !converged; it++) {
    // ---- step_lm
    double H[36], b[6], delta[16];
    y0 = linearize_impl(ttree, src, n, sstride, scov, tgt, tstride, tcov, x0, cfg->max_corr_dist, corr.data(), d2.data(), mahal.data(), H, b, threads);
    if (trace_H) std::memcpy(trace_H + (size_t)it * 36, H, sizeof(H));
    if (trace_b) std::memcpy(trace_b + (size_t)it * 6, b, sizeof(b));
    if (trace_y) trace_y[it] = y0;
    if (lambda < 0.0) {
      double mx = 0;
      for (int i = 0; i < 6; i++) mx = std::max(mx, std::fabs(H[i * 6 + i]));
      lambda = 1e-9 * mx;
    }
    double nu = 2.0;
    bool ok = false;
    for (int li = 0; li < 10; li++) {
      total_inner++;
      double A[36], nb[6], d[6];
      for (int i = 0; i < 36; i++) A[i] = H[i] + ((i % 7 == 0) ? lambda : 0.0);
      for (int i = 0; i < 6; i++) nb[i] = -b[i];
      bool solved = ldlt6_solve(A, nb, d);
      for (int i = 0; i < 6; i++) solved &= std::isfinite(d[i]);
      // Deliberate choice (the reference's behaviour is undefined here: Eigen LDLT on a singular system yields NaN/inf and
      // maxCoeff() over NaN is unspecified): a singular / non-finite step ends the optimisation as "lm not converged",
      // the pose keeps its last valid value and converged_ stays false (hdl_graph_slam then skips the frame / candidate).
      if (!solved) break;
      se3_exp(d, delta);
      double xi[16];
      mul4_iso(delta, x0, xi);
      double yi = error_impl(src, n, sstride, tgt, tstride, corr.data(), mahal.data(), xi, threads);
      double den = 0;
      for (int i = 0; i < 6; i++) den += d[i] * (lambda * d[i] - b[i]);
      double rho = (y0 - yi) / den;
      if (rho < 0) {
        if (is_converged(delta, cfg->rotation_epsilon, cfg->transformation_epsilon)) { ok = true; break; }
        lambda = nu * lambda;
        nu = 2 * nu;
        continue;
      }
      double t = 2 * rho - 1;
      lambda = lambda * std::max(1.0 / 3.0, 1 - t * t * t);
      std::memcpy(x0, xi, sizeof(xi));
      ok = true;
      break;
    }
    if (!ok) { lm_failed = true; it++; break; }
    converged = is_converged(delta, cfg->rotation_epsilon, cfg->transformation_epsilon);
  }
  for (int i = 0; i < 16; i++) { res->T64[i] = x0[i]; res->T[i] = (float)x0[i]; }
  res->converged = converged ? 1 : 0;
  res->iterations = it;
  res->lm_failed = lm_failed ? 1 : 0;
  res->last_error = y0;
  res->total_inner = total_inner;
  if (corr_out) std::memcpy(corr_out, corr.data(), n * sizeof(int32_t));
}

// ---- fitness / inliers ---------------------------------------------------------------------------------------
extern "C" void orc_fitness(const float* tgt, size_t m, size_t tstride, const float* src, size_t n, size_t sstride, const float* T,
                            double max_range, float inlier_thresh_sq, double* score, uint32_t* nr_out, uint32_t* n_inliers,
                            int32_t* nn_idx, float* nn_d2, int threads) {
  KdTree tree;
  tree.build(tgt, m, tstride);
  std::vector<float> d2(n);
  std::vector<int32_t> idx(n);
#pragma omp parallel for num_threads(nthreads(threads)) schedule(static)
  for (long i = 0; i < (long)n; i++) {
    float q[3];
    xform_f32(T, src + (size_t)i * sstride, q);
    int id = -1;
    float d = INFINITY;
    tree.knn(q, 1, &id, &d);
    d2[i] = d;
    idx[i] = id;
  }
  // serial accumulation in index order, double, exactly like the reference loop (information_matrix_calculator.cpp:63-74)
  double sum = 0;
  uint32_t nr = 0, inl = 0;
  for (size_t i = 0; i < n; i++) {
    if (idx[i] < 0) continue;
    if ((double)d2[i] <= max_range) { sum += (double)d2[i]; nr++; }
    if (d2[i] < inlier_thresh_sq) inl++;
  }
  *score = nr > 0 ? sum / nr : DBL_MAX;
  *nr_out = nr;
  *n_inliers = inl;
  if (nn_idx) std::memcpy(nn_idx, idx.data(), n * sizeof(int32_t));
  if (nn_d2) std::memcpy(nn_d2, d2.data(), n * sizeof(float));
}

// ---- prefilter chain (SURVEY.md 8f-2): PrefilteringNodelet::distance_filter and pcl::Radius/StatisticalOutlierRemoval ----
// /root/reference/apps/prefiltering_nodelet.cpp:164-180 (distance), :72-93,151-162 (outlier removal).  keep[i] in {0,1}.
extern "C" void orc_distance_filter(const float* pts, size_t n, size_t stride, double near_t, double far_t, unsigned char* keep) {
  for (size_t i = 0; i < n; i++) {
    const float* p = pts + i * stride;
    float sq = p[0] * p[0] + p[1] * p[1];
    sq = sq + p[2] * p[2];
    double d = (double)std::sqrt(sq);  // Eigen Vector3f::norm() in float32, promoted for the comparison
    keep[i] = (std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]) && d > near_t && d < far_t) ? 1 : 0;
  }
}

extern "C" void orc_radius_outlier(const float* pts, size_t n, size_t stride, double radius, int min_neighbors, unsigned char* keep, int threads) {
  KdTree tree;
  tree.build(pts, n, stride);
  const int k = min_neighbors + 1;
  const double r2 = radius * radius;
#pragma omp parallel for num_threads(nthreads(threads)) schedule(static)
  for (long i = 0; i < (long)n; i++) {
    std::vector<int> idx(k);
    std::vector<float> d2(k);
    int c = tree.knn(pts + (size_t)i * stride, k, idx.data(), d2.data());
    // PCL (dense path): nearestKSearch(min_pts + 1); outlier if fewer found or the last one is beyond the radius
    keep[i] = (c == k && !((double)d2[k - 1] > r2)) ? 1 : 0;
  }
}

extern "C" void orc_statistical_outlier(const float* pts, size_t n, size_t stride, int mean_k, double stddev_mul, unsigned char* keep,
                                        float* dist_out, int threads) {
  KdTree tree;
  tree.build(pts, n, stride);
  const int k = mean_k + 1;
  std::vector<float> dist(n);
#pragma omp parallel for num_threads(nthreads(threads)) schedule(static)
  for (long i = 0; i < (long)n; i++) {
    std::vector<int> idx(k);
    std::vector<float> d2(k);
    int c = tree.knn(pts + (size_t)i * stride, k, idx.data(), d2.data());
    double s = 0.0;
    for (int j = 1; j < c; j++) s += (double)std::sqrt(d2[j]);  // first neighbour is the point itself
    dist[i] = (float)(s / (double)mean_k);
  }
  // pcl::StatisticalOutlierRemoval::applyFilterIndices: a non-finite point gets distance 0.0 and is not counted as valid;
  // `sq_sum += distance * distance` multiplies two floats (float32 product, then widened)
  double sum = 0, sq = 0;
  size_t valid = 0;
  for (size_t i = 0; i < n; i++) {
    const float* p = pts + i * stride;
    if (!(std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]))) { dist[i] = 0.0f; continue; }
    valid++;
    const float d = dist[i];
    volatile float dd = d * d;
    sum += (double)d;
    sq += (double)dd;
  }
  double mean = sum / (double)valid;
  double variance = (sq - sum * sum / (double)valid) / ((double)valid - 1.0);
  double thresh = mean + stddev_mul * std::sqrt(variance);
  for (size_t i = 0; i < n; i++) keep[i] = (valid > 0 && !((double)dist[i] > thresh)) ? 1 : 0;
  if (dist_out) std::memcpy(dist_out, dist.data(), n * sizeof(float));
}

// PrefilteringNodelet::deskewing (/root/reference/apps/prefiltering_nodelet.cpp:182-243), float32 in Eigen's evaluation order:
// delta_q = Quaternionf(1, dt/2 wx, dt/2 wy, dt/2 wz) with ang_v already negated (:217); pt_ = delta_q.inverse() * pt
// (inverse = conjugate / squaredNorm; rotation v + w * (2 q x v) + q x (2 q x v)).  angular_velocity = the IMU message's value.
extern "C" void orc_deskew(const float* pts, size_t n, size_t stride, double scan_period, const float* angular_velocity, float* out) {
  const float wx = -angular_velocity[0], wy = -angular_velocity[1], wz = -angular_velocity[2];
  for (size_t i = 0; i < n; i++) {
    const float* p = pts + i * stride;
    float* o = out + i * stride;
    for (size_t k = 0; k < stride; k++) o[k] = p[k];
    const double delta_t = scan_period * (double)i / (double)n;
    const double half = delta_t / 2.0;
    const float qw = 1.0f, qx = (float)(half * (double)wx), qy = (float)(half * (double)wy), qz = (float)(half * (double)wz);
    volatile float a = qx * qx, b = qy * qy, c = qz * qz, d = qw * qw;
    volatile float ab = a + b;
    volatile float abc = ab + c;
    const float n2 = abc + d;
    const float iw = qw / n2, ix = -qx / n2, iy = -qy / n2, iz = -qz / n2;
    const float vx = p[0], vy = p[1], vz = p[2];
    auto cross = [](float ax, float ay, float az, float bx, float by, float bz, float* r) {
      volatile float t0 = ay * bz, t1 = az * by, t2 = az * bx, t3 = ax * bz, t4 = ax * by, t5 = ay * bx;
      r[0] = t0 - t1; r[1] = t2 - t3; r[2] = t4 - t5;
    };
    float u[3], cc[3];
    cross(ix, iy, iz, vx, vy, vz, u);
    u[0] = u[0] + u[0]; u[1] = u[1] + u[1]; u[2] = u[2] + u[2];
    cross(ix, iy, iz, u[0], u[1], u[2], cc);
    volatile float w0 = iw * u[0], w1 = iw * u[1], w2 = iw * u[2];
    volatile float s0 = vx + w0, s1 = vy + w1, s2 = vz + w2;
    o[0] = s0 + cc[0]; o[1] = s1 + cc[1]; o[2] = s2 + cc[2];
  }
}
