/* tests/gicp_pcl_ref.cpp — TEST INFRASTRUCTURE ONLY: the sequential CPU reference of pcl::GeneralizedIterativeClosestPoint (PCL 1.10,
 * the ROS noetic package) that defines the parity of B2R_METHOD_GICP_PCL (hdl_graph_slam_b200/csrc/gicp_pcl.cuh).  No OpenMP; built by
 * the tests with -O2 -ffp-contract=off (no FMA).
 *
 * PCL's sources are not available here: every choice below is UPSTREAM-RECALL (recalled from gicp.h / gicp.hpp / bfgs.h of PCL 1.10)
 * or, where upstream is undefined, this engine's documented rule (ENGINE).  DOUBT marks a recall this contract could not settle.
 *   factory (registrations.cpp:66-76): transformation_epsilon (0.01), max_iterations (64), corr_dist_threshold_ (2.5),
 *     k_correspondences_ (20), max_inner_iterations_ (reg_max_optimizer_iterations, 20); rotation_epsilon_ 2e-3, gicp_epsilon_ 1e-3.
 *     setUseReciprocalCorrespondences is called and GICP never reads the flag.                         UPSTREAM-RECALL (DOUBT)
 *     PCL 1.8 (melodic) is believed to match on every point below; not verified.                                   DOUBT
 *   computeCovariances: nearestKSearch(p, k) in the same cloud, the point itself included, ascending distance; equal distances
 *     in ascending index.                                                                       UPSTREAM-RECALL (tie order: ENGINE)
 *     mean += p (float promoted), cov(k, l) += p_k * p_l with the product in float32, summed in float64 in list order; / k;
 *     cov(k, l) -= mean_k mean_l; JacobiSVD, rebuilt with singular values (1, 1, gicp_epsilon).                  UPSTREAM-RECALL
 *     For the PSD matrices met here the rebuild is I - (1 - eps) n n^T with n the eigenvector of the SMALLEST eigenvalue (this
 *     reference: orc::sym_eigen, the engine: a closed form; they agree within 1e-8).  An indefinite matrix from cancellation would
 *     order SVD's singular values by magnitude instead; the engine keeps the smallest eigenvalue, except on an exactly diagonal
 *     matrix, where the rule below orders by magnitude as JacobiSVD does.                                           ENGINE
 *     An exactly diagonal matrix (a line along an axis whose products are exact, or all neighbours one point) has tied
 *     eigenvalues; n is the column JacobiSVD leaves last: no rotation, then its step-4 sort (first maximum of the remaining
 *     |values| swapped in only when not already in place, stop at a zero maximum).  diag(a, 0, 0) and diag(0, a, 0) give e_z,
 *     diag(0, 0, a) gives e_x, the zero matrix and multiples of I give e_z (orc::diagonal_normal).               UPSTREAM-RECALL
 *   non-finite points are in no search structure: they are nobody's neighbour, have no covariance and no correspondence.  ENGINE
 *   a cloud with fewer than k (finite) points: upstream indexes past the neighbour list (undefined); here the moments run over
 *     the neighbours found and divide by their count.                                                                ENGINE
 *   computeTransformation: transformation_ starts at identity on every align (PCL 1.10 may carry it over from the previous
 *     align of the same object: DOUBT); output = transformPointCloud(input, guess): x' = ((m0 x + m1 y) + m2 z) + m3 in float32,
 *     the order of Eigen's Matrix4f * Vector4f without FMA (PCL's SSE transformer may add in another order: DOUBT).
 *     Each outer iteration: q = transformation_ * output_i (float32, same order); exact 1-NN in the target; the pair is accepted
 *     iff (double)d2 < corr_dist^2 (float64, strict); M_i = (R C1_i R^T + C2_j)^-1 with R the top-left of the float64 triple-loop
 *     product double(transformation_) double(guess), (R C1) R^T + C2 as Eigen's coefficient products ((a0 b0 + a1 b1) + a2 b2), and
 *     Eigen's 3x3 inverse: cofactors c(i, j) = m(i1, j1) m(i2, j2) - m(i1, j2) m(i2, j1), det = (c00 m00 + c10 m10) + c20 m20,
 *     inverse(i, j) = c(j, i) * (1 / det).                                                                          UPSTREAM-RECALL
 *     A non-finite query gets no correspondence (upstream would return from computeTransformation when a search fails).  ENGINE
 *     previous_transformation_ = transformation_; fewer than 4 pairs throw NotEnoughPointsException, caught as a PCLException: the
 *     loop ends, not converged (so m = 0 never reaches f = 0/0).                                                     UPSTREAM-RECALL
 *     delta = max over the 4x4 of |prev - cur| (float difference) / rotation_epsilon on the 3x3 block, / transformation_epsilon
 *     elsewhere; nr_iterations_++; converged when nr_iterations_ >= max_iterations or delta < 1 (hitting the limit counts as
 *     converged).  final = previous_transformation_ * guess (float32, ((a0 b0 + a1 b1) + a2 b2) + a3 b3).             UPSTREAM-RECALL
 *   estimateRigidTransformationBFGS: x = (t, atan2f(r21, r22), asin(-(double)r20), atan2f(r10, r00)) from transformation_ (the float
 *     atan2 overload, the double asin: DOUBT); sigma = rho = 0.01, tau1 = 9, tau2 = 0.05, tau3 = 0.5, order 3, step size 1,
 *     bracket / section iterations 100; minimizeInit then do { minimizeOneStep; break on a nonzero status; testGradient(1e-2) }
 *     while Running and inner < max_inner_iterations_.  NoProgress, Success or the inner limit apply the state; any other status
 *     throws SolverDidntConvergeException (caught: loop ends, not converged) — unreachable with the statuses these routines
 *     return.                                                                                                        UPSTREAM-RECALL
 *   BFGS (bfgs.h, after GSL's vector_bfgs2 / linmin): minimizeOneStep, lineSearch (Fletcher bracketing + sectioning, the
 *     "roundoff prevents progress" NoProgress exit, Success when the iterations run out with alpha_new untouched = 0), interpolate
 *     (cubic when fpb is not NaN or +inf, else quadratic with curvature test c > 0), applyF / applyDF / applyFDF with their alpha
 *     cache keys, changeDirection, the BFGS direction update; norms and dots summed in index order (Eigen's vectorised reductions
 *     may pair terms differently: DOUBT).  The cubic's critical points: gsl_poly_solve_quadratic (PCL: Eigen's PolynomialSolver,
 *     equal up to rounding: DOUBT); Eigen::poly_eval (Horner for |x| <= 1, in 1/x times x^3 beyond).               UPSTREAM-RECALL
 *   applyState(identity, x): AngleAxisf(x5, Z) * AngleAxisf(x4, Y) * AngleAxisf(x3, X) as float quaternions (w = cos(a/2),
 *     v = sin(a/2) axis; Eigen's scalar quaternion product), toRotationMatrix; translation (float)x0..2.             UPSTREAM-RECALL
 *   OptimizationFunctorWithIndices over the m pairs in ascending source index: pp = T(x) output_i (float32), res = (double)(pp - tgt)
 *     (float difference), temp = M res, f += res^T temp, g_t += temp, dR += (double)output_i temp^T; f / m, g_t * (2 / m),
 *     dR * (2 / m); computeRDerivative with matricesInnerProd(a, b) = sum_i sum_j a(j, i) b(i, j).                   UPSTREAM-RECALL
 *     The engine sums the pairs in a fixed tree instead of this order (rel 1e-9 apart), and an evaluation at the pose of the pass
 *     just before reuses that pass; both counters are reported.  Near the minimum the line search compares f values equal to the
 *     last bits, so the number of evaluations (not the outer iterations, flag or pose) can differ by a few with the summation
 *     order.                                                                                                          ENGINE                                           ENGINE
 */
#include "../oracle/kdtree.hpp"
#include "../oracle/linalg.hpp"
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

namespace {

bool finite3(const float* p) { return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]); }

// x' = ((m0 x + m1 y) + m2 z) + m3 per row, float32 (T row-major 4x4)
void xform(const float* T, const float* p, float* o) {
  for (int r = 0; r < 3; r++) o[r] = ((T[r * 4] * p[0] + T[r * 4 + 1] * p[1]) + T[r * 4 + 2] * p[2]) + T[r * 4 + 3];
}

void mul4f(const float* A, const float* B, float* O) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) O[i * 4 + j] = ((A[i * 4] * B[j] + A[i * 4 + 1] * B[4 + j]) + A[i * 4 + 2] * B[8 + j]) + A[i * 4 + 3] * B[12 + j];
}

void covariances(const float* pts, size_t n, size_t stride, int k, double* out) {
  orc::KdTree tree;
  tree.build(pts, n, stride);
  std::vector<int> idx(k);
  std::vector<float> d2(k);
  for (size_t i = 0; i < n; i++) {
    double* o = out + i * 9;
    const float* q = pts + i * stride;
    if (!finite3(q)) { for (int a = 0; a < 9; a++) o[a] = NAN; continue; }
    const int kk = tree.knn(q, k, idx.data(), d2.data());
    double mean[3] = {0, 0, 0}, c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = 0; j < kk; j++) {
      const float* p = pts + (size_t)idx[j] * stride;
      mean[0] += p[0]; mean[1] += p[1]; mean[2] += p[2];
      c[0] += (double)(p[0] * p[0]);
      c[3] += (double)(p[1] * p[0]);
      c[4] += (double)(p[1] * p[1]);
      c[6] += (double)(p[2] * p[0]);
      c[7] += (double)(p[2] * p[1]);
      c[8] += (double)(p[2] * p[2]);
    }
    for (int a = 0; a < 3; a++) mean[a] /= (double)kk;
    for (int a = 0; a < 3; a++)
      for (int b = 0; b <= a; b++) {
        c[a * 3 + b] /= (double)kk;
        c[a * 3 + b] -= mean[a] * mean[b];
        c[b * 3 + a] = c[a * 3 + b];
      }
    double w[3], V[9];
    orc::sym_eigen<3>(c, w, V);  // ascending: column 0 = the smallest eigenvalue's vector
    if (c[1] == 0.0 && c[2] == 0.0 && c[5] == 0.0) orc::diagonal_normal(c, V);  // column 0 = JacobiSVD's last column
    const double vals[3] = {1e-3, 1.0, 1.0};
    for (int a = 0; a < 9; a++) o[a] = 0.0;
    for (int e = 2; e >= 0; e--)  // U's columns in descending singular value
      for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) o[a * 3 + b] += vals[e] * V[a * 3 + e] * V[b * 3 + e];
  }
}

struct Problem {
  const float* src; size_t n, ss;
  const float* tgt; size_t m, ts;
  const double* scov; const double* tcov;
  orc::KdTree tree;
  float G[16];
  double thr2;
  std::vector<float> out;          // output = guess * input (xyz per point)
  std::vector<int> sidx, tidx;     // accepted pairs, ascending source index
  std::vector<double> M;           // 9 per accepted pair
  long corr_passes = 0, cost_passes = 0, evaluations = 0, bfgs_steps = 0;
  // line-search trace: per Success exit of the sigma test (f0, fp0, alpha, f(alpha), f'(alpha))
  std::vector<double>* trace = nullptr;
};

void rel_rotation(const float* T, const float* G, double* R) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      double s = 0.0;
      for (int k = 0; k < 4; k++) s += double(T[i * 4 + k]) * double(G[k * 4 + j]);
      R[i * 3 + j] = s;
    }
}

void inverse3(const double* m, double* o) {
  double c[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
      c[i * 3 + j] = m[i1 * 3 + j1] * m[i2 * 3 + j2] - m[i1 * 3 + j2] * m[i2 * 3 + j1];
    }
  const double det = (c[0] * m[0] + c[3] * m[3]) + c[6] * m[6];
  const double inv = 1.0 / det;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) o[i * 3 + j] = c[j * 3 + i] * inv;
}

// one correspondence update at transformation_ = T
size_t correspond(Problem& P, const float* T) {
  P.corr_passes++;
  double R[9];
  rel_rotation(T, P.G, R);
  P.sidx.clear(); P.tidx.clear(); P.M.clear();
  for (size_t i = 0; i < P.n; i++) {
    const float* o = &P.out[i * 3];
    float q[3];
    xform(T, o, q);
    if (!finite3(o) || !finite3(q)) continue;
    int j;
    float d2;
    if (P.tree.knn(q, 1, &j, &d2) < 1) continue;
    if (!((double)d2 < P.thr2)) continue;
    const double* C1 = P.scov + i * 9;
    const double* C2 = P.tcov + (size_t)j * 9;
    double RC[9], Tm[9], Mi[9];
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) RC[a * 3 + b] = (R[a * 3] * C1[b] + R[a * 3 + 1] * C1[3 + b]) + R[a * 3 + 2] * C1[6 + b];
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) Tm[a * 3 + b] = ((RC[a * 3] * R[b * 3] + RC[a * 3 + 1] * R[b * 3 + 1]) + RC[a * 3 + 2] * R[b * 3 + 2]) + C2[a * 3 + b];
    inverse3(Tm, Mi);
    P.sidx.push_back((int)i);
    P.tidx.push_back(j);
    P.M.insert(P.M.end(), Mi, Mi + 9);
  }
  return P.sidx.size();
}

// the 13 sums of the functor at the float pose T (row-major 4x4)
void cost_sums(const Problem& P, const float* T, double* s) {
  for (int k = 0; k < 13; k++) s[k] = 0.0;
  for (size_t c = 0; c < P.sidx.size(); c++) {
    const float* o = &P.out[(size_t)P.sidx[c] * 3];
    const float* q = P.tgt + (size_t)P.tidx[c] * P.ts;
    float pp[3];
    xform(T, o, pp);
    const double r[3] = {(double)(pp[0] - q[0]), (double)(pp[1] - q[1]), (double)(pp[2] - q[2])};
    const double* M = &P.M[c * 9];
    double t[3];
    for (int a = 0; a < 3; a++) t[a] = (M[a * 3] * r[0] + M[a * 3 + 1] * r[1]) + M[a * 3 + 2] * r[2];
    s[0] += (r[0] * t[0] + r[1] * t[1]) + r[2] * t[2];
    for (int a = 0; a < 3; a++) s[1 + a] += t[a];
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) s[4 + a * 3 + b] += (double)o[a] * t[b];
  }
}

using V6 = std::array<double, 6>;
double dot6(const V6& a, const V6& b) { double s = 0.0; for (int i = 0; i < 6; i++) s += a[i] * b[i]; return s; }
double norm6(const V6& a) { return std::sqrt(dot6(a, a)); }

void apply_state(const V6& x, float* T) {
  struct Q { float w, x, y, z; };
  auto aa = [](float a, int axis) { const float h = 0.5f * a, s = std::sin(h); Q q{std::cos(h), 0.f, 0.f, 0.f}; (axis == 0 ? q.x : axis == 1 ? q.y : q.z) = s; return q; };
  auto mul = [](const Q& a, const Q& b) {
    return Q{a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
             a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
  };
  const Q q = mul(mul(aa((float)x[5], 2), aa((float)x[4], 1)), aa((float)x[3], 0));
  const float tx = 2.f * q.x, ty = 2.f * q.y, tz = 2.f * q.z;
  const float twx = tx * q.w, twy = ty * q.w, twz = tz * q.w, txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y,
              tzz = tz * q.z;
  const float R[9] = {1.f - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1.f - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1.f - (txx + tyy)};
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[r * 4 + c] = R[r * 3 + c];
    T[r * 4 + 3] = (float)x[r];
  }
  T[12] = T[13] = T[14] = 0.f; T[15] = 1.f;
}

void r_derivative(const V6& x, const double* Rs, V6& g) {
  const double phi = x[3], theta = x[4], psi = x[5];
  const double cphi = std::cos(phi), sphi = std::sin(phi), ctheta = std::cos(theta), stheta = std::sin(theta), cpsi = std::cos(psi), spsi = std::sin(psi);
  double a[9], b[9], c[9];
  a[0] = 0.; a[3] = 0.; a[6] = 0.;
  a[1] = sphi * spsi + cphi * cpsi * stheta; a[4] = -cpsi * sphi + cphi * spsi * stheta; a[7] = cphi * ctheta;
  a[2] = cphi * spsi - cpsi * sphi * stheta; a[5] = -cphi * cpsi - sphi * spsi * stheta; a[8] = -ctheta * sphi;
  b[0] = -cpsi * stheta; b[3] = -spsi * stheta; b[6] = -ctheta;
  b[1] = cpsi * ctheta * sphi; b[4] = ctheta * sphi * spsi; b[7] = -sphi * stheta;
  b[2] = cphi * cpsi * ctheta; b[5] = cphi * ctheta * spsi; b[8] = -cphi * stheta;
  c[0] = -ctheta * spsi; c[3] = cpsi * ctheta; c[6] = 0.;
  c[1] = -cphi * cpsi - sphi * spsi * stheta; c[4] = -cphi * spsi + cpsi * sphi * stheta; c[7] = 0.;
  c[2] = cpsi * sphi - cphi * spsi * stheta; c[5] = sphi * spsi + cphi * cpsi * stheta; c[8] = 0.;
  auto inner = [&](const double* m1) {
    double r = 0.;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) r += m1[j * 3 + i] * Rs[i * 3 + j];
    return r;
  };
  g[3] = inner(a); g[4] = inner(b); g[5] = inner(c);
}

struct Functor {
  Problem* P;
  int m;
  float lastT[16];
  double last[13];
  bool have = false;
  void sums(const V6& x, double* s) {
    float T[16];
    apply_state(x, T);
    P->evaluations++;
    if (!(have && std::memcmp(T, lastT, sizeof(T)) == 0)) {
      cost_sums(*P, T, last);
      std::memcpy(lastT, T, sizeof(T));
      have = true;
      P->cost_passes++;
    }
    std::memcpy(s, last, sizeof(last));
  }
  void grad_from(const V6& x, const double* s, V6& g) {
    g = V6{0, 0, 0, 0, 0, 0};
    const double k = 2.0 / m;
    for (int i = 0; i < 3; i++) g[i] = s[1 + i] * k;
    double R[9];
    for (int i = 0; i < 9; i++) R[i] = s[4 + i] * k;
    r_derivative(x, R, g);
  }
  double f(const V6& x) { double s[13]; sums(x, s); return s[0] / m; }
  void df(const V6& x, V6& g) { double s[13]; sums(x, s); grad_from(x, s, g); }
  void fdf(const V6& x, double& fv, V6& g) { double s[13]; sums(x, s); fv = s[0] / m; grad_from(x, s, g); }
};

enum Status { NegativeGradientEpsilon = -3, NotStarted = -2, Running = -1, Success = 0, NoProgress = 1 };

struct Bfgs {
  Functor& fn;
  std::vector<double>* trace;
  double rho = 0.01, sigma = 0.01, tau1 = 9, tau2 = 0.05, tau3 = 0.5, step_size = 1;
  int order = 3, bracket_iters = 100, section_iters = 100;
  double f = 0, delta_f = 0, fp0 = 0, pnorm = 0, g0norm = 0;
  V6 gradient{}, x0{}, dx0{}, dg0{}, g0{}, dx{}, p{}, x_alpha{}, g_alpha{};
  double f_alpha = 0, df_alpha = 0, x_cache_key = 0, f_cache_key = 0, df_cache_key = 0, g_cache_key = 0;
  Bfgs(Functor& f_, std::vector<double>* t) : fn(f_), trace(t) {}

  static double poly_eval(const double* c, double x) {
    if (x * x <= 1.0) {
      double v = c[3];
      for (int i = 2; i >= 0; i--) v = v * x + c[i];
      return v;
    }
    double v = c[0];
    const double ix = 1.0 / x;
    for (int i = 1; i < 4; i++) v = v * ix + c[i];
    return std::pow(x, 3.0) * v;
  }
  static int solve_quadratic(double a, double b, double c, double* x0, double* x1) {
    if (a == 0) {
      if (b == 0) return 0;
      *x0 = -c / b;
      return 1;
    }
    const double disc = b * b - 4 * a * c;
    if (disc > 0) {
      if (b == 0) {
        const double r = std::sqrt(-c / a);
        *x0 = -r; *x1 = r;
      } else {
        const double sgnb = (b > 0 ? 1 : -1);
        const double temp = -0.5 * (b + sgnb * std::sqrt(disc));
        const double r1 = temp / a, r2 = c / temp;
        if (r1 < r2) { *x0 = r1; *x1 = r2; } else { *x0 = r2; *x1 = r1; }
      }
      return 2;
    }
    if (disc == 0) { *x0 = -0.5 * b / a; *x1 = -0.5 * b / a; return 2; }
    return 0;
  }
  static double interpolate(double a, double fa, double fpa, double b, double fb, double fpb, double xmin, double xmax, int order) {
    double ymin = (xmin - a) / (b - a), ymax = (xmax - a) / (b - a), y, fmin;
    if (ymin > ymax) std::swap(ymin, ymax);
    if (order > 2 && !(fpb != fpb) && fpb != std::numeric_limits<double>::infinity()) {
      fpa = fpa * (b - a);
      fpb = fpb * (b - a);
      const double eta = 3 * (fb - fa) - 2 * fpa - fpb, xi = fpa + fpb - 2 * (fb - fa);
      const double c[4] = {fa, fpa, eta, xi};
      y = ymin;
      fmin = poly_eval(c, ymin);
      auto check = [&](double z) { const double v = poly_eval(c, z); if (v < fmin) { y = z; fmin = v; } };
      check(ymax);
      double y0 = 0, y1 = 0;
      const int n = solve_quadratic(3 * c[3], 2 * c[2], c[1], &y0, &y1);
      if (n == 2) {
        if (y0 > y1) std::swap(y0, y1);
        if (y0 > ymin && y0 < ymax) check(y0);
        if (y1 > ymin && y1 < ymax) check(y1);
      } else if (n == 1) {
        if (y0 > ymin && y0 < ymax) check(y0);
      }
    } else {
      fpa = fpa * (b - a);
      const double fl = fa + ymin * (fpa + ymin * (fb - fa - fpa));
      const double fh = fa + ymax * (fpa + ymax * (fb - fa - fpa));
      const double c = 2 * (fb - fa - fpa);
      y = ymin;
      fmin = fl;
      if (fh < fmin) { y = ymax; fmin = fh; }
      if (c > 0) {
        const double z = -fpa / c;
        if (z > ymin && z < ymax) {
          const double fz = fa + z * (fpa + z * (fb - fa - fpa));
          if (fz < fmin) { y = z; fmin = fz; }
        }
      }
    }
    return a + y * (b - a);
  }
  void move_to(double alpha) {
    for (int i = 0; i < 6; i++) x_alpha[i] = x0[i] + alpha * p[i];
    x_cache_key = alpha;
  }
  double slope() const { return dot6(g_alpha, p); }
  double apply_f(double alpha) {
    if (alpha == f_cache_key) return f_alpha;
    move_to(alpha);
    f_alpha = fn.f(x_alpha);
    f_cache_key = alpha;
    return f_alpha;
  }
  double apply_df(double alpha) {
    if (alpha == df_cache_key) return df_alpha;
    move_to(alpha);
    if (alpha != g_cache_key) {
      fn.df(x_alpha, g_alpha);
      g_cache_key = alpha;
    }
    df_alpha = slope();
    df_cache_key = alpha;
    return df_alpha;
  }
  void apply_fdf(double alpha, double& fv, double& dfv) {
    if (alpha == f_cache_key && alpha == df_cache_key) { fv = f_alpha; dfv = df_alpha; return; }
    if (alpha == f_cache_key || alpha == df_cache_key) { fv = apply_f(alpha); dfv = apply_df(alpha); return; }
    move_to(alpha);
    fn.fdf(x_alpha, f_alpha, g_alpha);
    f_cache_key = alpha; g_cache_key = alpha;
    df_alpha = slope();
    df_cache_key = alpha;
    fv = f_alpha; dfv = df_alpha;
  }
  void change_direction() {
    x_alpha = x0; x_cache_key = 0.0;
    f_cache_key = 0.0;
    g_alpha = g0; g_cache_key = 0.0;
    df_alpha = slope(); df_cache_key = 0.0;
  }
  void log(double f0, double fp0l, double alpha, double fa, double fpa) {
    if (trace) { trace->push_back(f0); trace->push_back(fp0l); trace->push_back(alpha); trace->push_back(fa); trace->push_back(fpa); }
  }
  int line_search(double alpha1, double& alpha_new) {
    double f0, fp0l, falpha, falpha_prev, fpalpha, fpalpha_prev, delta, alpha_next;
    double alpha = alpha1, alpha_prev = 0.0, a, b, fa, fb, fpa, fpb;
    int i = 0;
    apply_fdf(0.0, f0, fp0l);
    falpha_prev = f0; fpalpha_prev = fp0l;
    a = 0.0; b = alpha; fa = f0; fb = 0.0; fpa = fp0l; fpb = 0.0;
    while (i++ < bracket_iters) {
      falpha = apply_f(alpha);
      if (falpha > f0 + alpha * rho * fp0l || falpha >= falpha_prev) {
        a = alpha_prev; fa = falpha_prev; fpa = fpalpha_prev;
        b = alpha; fb = falpha; fpb = std::numeric_limits<double>::quiet_NaN();
        break;
      }
      fpalpha = apply_df(alpha);
      if (std::fabs(fpalpha) <= -sigma * fp0l) { alpha_new = alpha; log(f0, fp0l, alpha, falpha, fpalpha); return Success; }
      if (fpalpha >= 0) {
        a = alpha; fa = falpha; fpa = fpalpha;
        b = alpha_prev; fb = falpha_prev; fpb = fpalpha_prev;
        break;
      }
      delta = alpha - alpha_prev;
      alpha_next = interpolate(alpha_prev, falpha_prev, fpalpha_prev, alpha, falpha, fpalpha, alpha + delta, alpha + tau1 * delta, order);
      alpha_prev = alpha; falpha_prev = falpha; fpalpha_prev = fpalpha;
      alpha = alpha_next;
    }
    while (i++ < section_iters) {
      delta = b - a;
      alpha = interpolate(a, fa, fpa, b, fb, fpb, a + tau2 * delta, b - tau3 * delta, order);
      falpha = apply_f(alpha);
      if ((a - alpha) * fpa <= std::numeric_limits<double>::epsilon()) return NoProgress;
      if (falpha > f0 + rho * alpha * fp0l || falpha >= fa) {
        b = alpha; fb = falpha; fpb = std::numeric_limits<double>::quiet_NaN();
      } else {
        fpalpha = apply_df(alpha);
        if (std::fabs(fpalpha) <= -sigma * fp0l) { alpha_new = alpha; log(f0, fp0l, alpha, falpha, fpalpha); return Success; }
        if (((b - a) >= 0 && fpalpha >= 0) || ((b - a) <= 0 && fpalpha <= 0)) {
          b = a; fb = fa; fpb = fpa;
          a = alpha; fa = falpha; fpa = fpalpha;
        } else {
          a = alpha; fa = falpha; fpa = fpalpha;
        }
      }
    }
    return Success;
  }
  void minimize_init(const V6& x) {
    delta_f = 0;
    dx = V6{};
    fn.fdf(x, f, gradient);
    x0 = x;
    g0 = gradient;
    g0norm = norm6(g0);
    for (int i = 0; i < 6; i++) p[i] = gradient[i] * -1 / g0norm;
    pnorm = norm6(p);
    fp0 = -g0norm;
    x_alpha = x0; x_cache_key = 0;
    f_alpha = f; f_cache_key = 0;
    g_alpha = g0; g_cache_key = 0;
    df_alpha = slope(); df_cache_key = 0;
  }
  int minimize_one_step(V6& x) {
    double alpha = 0.0, alpha1;
    const double f0 = f;
    if (pnorm == 0.0 || g0norm == 0.0 || fp0 == 0) { dx = V6{}; return NoProgress; }
    if (delta_f < 0) {
      const double del = std::max(-delta_f, 10 * std::numeric_limits<double>::epsilon() * std::fabs(f0));
      alpha1 = std::min(1.0, 2.0 * del / (-fp0));
    } else {
      alpha1 = std::fabs(step_size);
    }
    const int status = line_search(alpha1, alpha);
    if (status != Success) return status;
    {
      double fv, dfv;
      apply_fdf(alpha, fv, dfv);
      f = f_alpha; x = x_alpha; gradient = g_alpha;
    }
    delta_f = f - f0;
    for (int i = 0; i < 6; i++) { dx0[i] = x[i] - x0[i]; dg0[i] = gradient[i] - g0[i]; }
    dx = dx0;
    const double dxg = dot6(dx0, gradient), dgg = dot6(dg0, gradient), dxdg = dot6(dx0, dg0), dgnorm = norm6(dg0);
    double A = 0, B = 0;
    if (dxdg != 0) {
      B = dxg / dxdg;
      A = -(1.0 + dgnorm * dgnorm / dxdg) * B + dgg / dxdg;
    }
    for (int i = 0; i < 6; i++) { p[i] = -A * dx0[i]; p[i] += -B * dg0[i]; p[i] += gradient[i]; }
    g0 = gradient;
    x0 = x;
    g0norm = norm6(g0);
    pnorm = norm6(p);
    const double dir = (dot6(p, gradient) > 0) ? -1.0 : 1.0;
    for (int i = 0; i < 6; i++) p[i] *= dir / pnorm;
    pnorm = norm6(p);
    fp0 = dot6(p, g0);
    change_direction();
    return Success;
  }
  int test_gradient(double eps) const {
    if (eps < 0) return NegativeGradientEpsilon;
    return norm6(gradient) < eps ? Success : Running;
  }
};

void init_problem(Problem& P, const float* src, size_t n, size_t ss, const double* scov, const float* tgt, size_t m, size_t ts, const double* tcov,
                  const float* guess_row, double corr_dist) {
  P.src = src; P.n = n; P.ss = ss; P.tgt = tgt; P.m = m; P.ts = ts; P.scov = scov; P.tcov = tcov;
  P.tree.build(tgt, m, ts);
  std::memcpy(P.G, guess_row, sizeof(P.G));
  P.thr2 = corr_dist * corr_dist;
  P.out.resize(n * 3 + 3);
  for (size_t i = 0; i < n; i++) xform(P.G, src + i * ss, &P.out[i * 3]);
}

}  // namespace

extern "C" {

// covariances of a cloud (n x 9, NaN rows for non-finite points)
void ref_gicp_pcl_covariances(const float* pts, size_t n, size_t stride, int k, double* out) { covariances(pts, n, stride, k, out); }

// one correspondence pass: corr[n] (target index or -1), M[9 n] (NaN where none); returns the accepted count
size_t ref_gicp_pcl_correspondences(const float* src, size_t n, size_t ss, const double* scov, const float* tgt, size_t m, size_t ts, const double* tcov,
                                    const float* guess_row, const float* Trel_row, double corr_dist, int32_t* corr, double* M) {
  Problem P;
  init_problem(P, src, n, ss, scov, tgt, m, ts, tcov, guess_row, corr_dist);
  const size_t cnt = correspond(P, Trel_row);
  for (size_t i = 0; i < n; i++) {
    corr[i] = -1;
    for (int a = 0; a < 9; a++) M[i * 9 + a] = NAN;
  }
  for (size_t c = 0; c < cnt; c++) {
    corr[P.sidx[c]] = P.tidx[c];
    std::memcpy(M + (size_t)P.sidx[c] * 9, &P.M[c * 9], 9 * sizeof(double));
  }
  return cnt;
}

// one cost pass at T_row over the correspondences of (guess, T_rel): sums[13] = f, sum temp (3), sum p temp^T (9, row-major)
size_t ref_gicp_pcl_cost(const float* src, size_t n, size_t ss, const double* scov, const float* tgt, size_t m, size_t ts, const double* tcov,
                         const float* guess_row, const float* Trel_row, double corr_dist, const float* T_row, double* sums) {
  Problem P;
  init_problem(P, src, n, ss, scov, tgt, m, ts, tcov, guess_row, corr_dist);
  const size_t cnt = correspond(P, Trel_row);
  cost_sums(P, T_row, sums);
  return cnt;
}

// f and the 6-gradient of the functor at x over the correspondences of (guess, T_rel); returns m
size_t ref_gicp_pcl_fdf(const float* src, size_t n, size_t ss, const double* scov, const float* tgt, size_t m, size_t ts, const double* tcov,
                        const float* guess_row, const float* Trel_row, double corr_dist, const double* x, double* f, double* g) {
  Problem P;
  init_problem(P, src, n, ss, scov, tgt, m, ts, tcov, guess_row, corr_dist);
  const size_t cnt = correspond(P, Trel_row);
  if (cnt == 0) return 0;
  Functor fn{&P, (int)cnt};
  V6 xv, gv;
  for (int i = 0; i < 6; i++) xv[i] = x[i];
  fn.fdf(xv, *f, gv);
  for (int i = 0; i < 6; i++) g[i] = gv[i];
  return cnt;
}

// applyState(identity, x) as a row-major float 4x4
void ref_gicp_pcl_apply_state(const double* x, float* T) {
  V6 xv;
  for (int i = 0; i < 6; i++) xv[i] = x[i];
  apply_state(xv, T);
}

// the whole align.  cfg = {transformation_epsilon, rotation_epsilon, corr_dist}, icfg = {max_iterations, max_inner_iterations};
// T_out row-major float 4x4; stats = {converged, outer iterations, correspondence passes, cost passes, evaluations, bfgs steps};
// trace (may be NULL, capacity trace_cap doubles): 5 doubles per accepted line-search step; returns the doubles written
size_t ref_gicp_pcl_align(const float* src, size_t n, size_t ss, const double* scov, const float* tgt, size_t m, size_t ts, const double* tcov,
                          const float* guess_row, const double* cfg, const int* icfg, float* T_out, long* stats, double* trace, size_t trace_cap) {
  Problem P;
  std::vector<double> tr;
  P.trace = &tr;
  init_problem(P, src, n, ss, scov, tgt, m, ts, tcov, guess_row, cfg[2]);
  float Tcur[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}, Tprev[16];
  std::memcpy(Tprev, Tcur, sizeof(Tprev));
  bool conv = false;
  long outer = 0;
  if (n > 0 && m > 0) {
    while (!conv) {
      const size_t cnt = correspond(P, Tcur);
      std::memcpy(Tprev, Tcur, sizeof(Tprev));
      if (cnt < 4) break;
      V6 x{(double)Tcur[3], (double)Tcur[7], (double)Tcur[11], (double)std::atan2(Tcur[9], Tcur[10]), std::asin(-(double)Tcur[8]),
           (double)std::atan2(Tcur[4], Tcur[0])};
      Functor fn{&P, (int)cnt};
      Bfgs bfgs(fn, &tr);
      bfgs.minimize_init(x);
      int result = Running, inner = 0;
      do {
        inner++;
        P.bfgs_steps++;
        result = bfgs.minimize_one_step(x);
        if (result) break;
        result = bfgs.test_gradient(1e-2);
      } while (result == Running && inner < icfg[1]);
      if (!(result == NoProgress || result == Success || inner == icfg[1])) break;
      apply_state(x, Tcur);
      double delta = 0.;
      for (int k = 0; k < 4; k++)
        for (int l = 0; l < 4; l++) {
          const double ratio = (k < 3 && l < 3) ? 1. / cfg[1] : 1. / cfg[0];
          const double c = ratio * std::fabs(Tprev[k * 4 + l] - Tcur[k * 4 + l]);
          if (c > delta) delta = c;
        }
      outer++;
      if (outer >= icfg[0] || delta < 1) {
        conv = true;
        std::memcpy(Tprev, Tcur, sizeof(Tprev));
      }
    }
  }
  mul4f(Tprev, P.G, T_out);
  stats[0] = conv; stats[1] = outer; stats[2] = P.corr_passes; stats[3] = P.cost_passes; stats[4] = P.evaluations; stats[5] = P.bfgs_steps;
  const size_t w = std::min(tr.size(), trace ? trace_cap : (size_t)0);
  if (w) std::memcpy(trace, tr.data(), w * sizeof(double));
  return tr.size();
}

}  // extern "C"
