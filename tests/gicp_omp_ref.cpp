/* tests/gicp_omp_ref.cpp — TEST INFRASTRUCTURE ONLY: the sequential CPU reference of pclomp::GeneralizedIterativeClosestPoint (ndt_omp's
 * OpenMP copy of PCL's GICP, the factory's GICP_OMP branch) that defines the parity of B2R_METHOD_GICP_OMP
 * (hdl_graph_slam_b200/csrc/gicp_pcl.cuh).  No OpenMP; built by the tests with -O2 -ffp-contract=off (no FMA).
 *
 * It is tests/gicp_pcl_ref.cpp (included below, unchanged) with one rule changed; every other rule, and its mark, is that file's.
 * Neither ndt_omp's nor PCL's sources are available here: every choice is UPSTREAM-RECALL, ENGINE (the engine's rule where upstream is
 * undefined) or DOUBT (a recall this contract could not settle).
 *   factory (registrations.cpp:76-86): the GICP branch's six setters — transformation epsilon, maximum iterations, the reciprocal flag
 *     (never read), correspondence distance, k and maximum optimizer iterations; reg_num_threads is not set.      UPSTREAM-RECALL
 *   the sources are PCL 1.8-era GICP (gicp.h / gicp.hpp) with PCL's own pcl/registration/bfgs.h: covariances, the correspondence
 *     query transformation_ (guess p) in float32, the strict float64 threshold, M = (R C1 R^T + C2)^-1 with R from the float64
 *     triple-loop product, the fewer-than-4-pairs exit, the BFGS (x seeded from transformation_, minimizeInit, minimizeOneStep,
 *     testGradient(1e-2)), transformation_ = applyState(I, x) after each BFGS run, the delta test and final =
 *     previous_transformation_ guess are gicp_pcl_ref.cpp's rules and run as its code: ref_gicp_omp_fdf / _align ARE
 *     ref_gicp_pcl_fdf / _align, with the functor's cost sums switched to the rule below.               UPSTREAM-RECALL (DOUBT)
 *   THE ONE DIFFERENCE: pclomp keeps base_transformation_ = guess and does not transform the source by the guess before the functor.
 *     OptimizationFunctorWithIndices evaluates at T'(x) = applyState(guess, x) = [R(x) R_g | t_g + t(x)], the 3x3 product in float32
 *     ((a0 b0 + a1 b1) + a2 b2), the translation t_g + (float)x0..2, the bottom row the guess's, applied to the RAW source point:
 *     pp = T'(x) p (float32, the unfused row order of xform).  The dR term is over (double)(guess p) = output_i, as in GICP.
 *     Here: omp_pose and omp_cost_sums, one place to change.                                             UPSTREAM-RECALL (DOUBT)
 *     Consequence: the functor's pose and the correspondence pose differ by (R(x) - I) t_g, so with a translated guess the end pose
 *     differs from GICP's by about (R(x*) - I) t_g; at an identity guess the two are the same align.
 *   the correspondence list's order (an atomic counter under OpenMP upstream): ascending source index.                 ENGINE
 *   the functor's sums (per-thread partials, then std::accumulate upstream): index order here, the engine's fixed tree on the
 *     device (rel 1e-9 apart; see gicp_pcl_ref.cpp on what that moves).                                                ENGINE
 *   an evaluation at the pose of the cost pass just before (within one correspondence pass) reuses that pass; the pose is
 *     applyState(guess, x), so states whose translations differ only below the guess's float32 rounding share a pass.   ENGINE
 *
 * How the switch is made without editing gicp_pcl_ref.cpp: its Problem type is compiled as omp_hook::Problem (a name change only), so
 * the call cost_sums(*P, T, last) in its Functor also finds omp_hook::cost_sums by argument-dependent lookup, which is the better
 * match for the functor's non-const arguments.  That hook runs pcl GICP's cost_sums unless an omp entry point below is active on this
 * thread (OmpRule), in which case it evaluates pclomp's functor at applyState(guess, x) from the functor's applyState(I, x).  Every
 * other call of cost_sums in that file passes const arguments and never reaches the hook, and its ref_gicp_pcl_* entry points compute
 * what they compute in their own library.
 */
#include <array>

namespace {
namespace omp_hook {
struct Problem;
void cost_sums(Problem& P, float* T, double* s);
}  // namespace omp_hook
}  // namespace

#define Problem omp_hook::Problem
#include "gicp_pcl_ref.cpp"
#undef Problem

namespace {

using omp_hook::Problem;

thread_local bool omp_rule = false;  // an omp entry point is running on this thread
// the pose of the last pclomp cost pass, and the problem and correspondence pass it belongs to
thread_local struct { const Problem* P; long corr; float T[16]; } last_pass = {nullptr, -1, {}};

struct OmpRule {
  OmpRule() { omp_rule = true; last_pass.P = nullptr; }
  ~OmpRule() { omp_rule = false; last_pass.P = nullptr; }
};

// applyState(guess, x) from A = applyState(I, x) (row-major float 4x4s): [R(x) R_g | t_g + t(x)], bottom row the guess's
void omp_pose(const float* A, const float* G, float* T) {
  float R[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) R[i * 3 + j] = (A[i * 4] * G[j] + A[i * 4 + 1] * G[4 + j]) + A[i * 4 + 2] * G[8 + j];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) T[i * 4 + j] = R[i * 3 + j];
    T[i * 4 + 3] = G[i * 4 + 3] + A[i * 4 + 3];
  }
  for (int j = 0; j < 4; j++) T[12 + j] = G[12 + j];
}

// pclomp's 13 sums at the pose T (applyState(guess, x)): pp = T p on the raw source point, res = (double)(pp - tgt), temp = M res,
// f += res^T temp, g += temp, dR += (double)output_i temp^T, pairs in ascending source index
void omp_cost_sums(const Problem& P, const float* T, double* s) {
  for (int k = 0; k < 13; k++) s[k] = 0.0;
  for (size_t c = 0; c < P.sidx.size(); c++) {
    const float* o = &P.out[(size_t)P.sidx[c] * 3];
    const float* q = P.tgt + (size_t)P.tidx[c] * P.ts;
    float pp[3];
    xform(T, P.src + (size_t)P.sidx[c] * P.ss, pp);
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

// gicp_pcl_ref.cpp's own cost_sums (const arguments: the hook is not viable here)
void pcl_cost_sums(const Problem& P, const float* T, double* s) { cost_sums(P, T, s); }

}  // namespace

// the functor's cost pass at T = applyState(I, x)
void omp_hook::cost_sums(Problem& P, float* T, double* s) {
  if (!omp_rule) {
    pcl_cost_sums(P, T, s);
    return;
  }
  float Tp[16];
  omp_pose(T, P.G, Tp);
  // gicp_pcl_ref.cpp's functor reuses a pass when applyState(I, x) repeats; the engine's reuses it when the pass's own pose repeats
  // (ENGINE: the sums depend on nothing else).  Two states whose translations differ only below the guess's float32 rounding give the
  // same applyState(guess, x): that evaluation is not counted as a pass here either.
  if (last_pass.P == &P && last_pass.corr == P.corr_passes && std::memcmp(Tp, last_pass.T, sizeof(Tp)) == 0) P.cost_passes--;
  last_pass.P = &P;
  last_pass.corr = P.corr_passes;
  std::memcpy(last_pass.T, Tp, sizeof(Tp));
  omp_cost_sums(P, Tp, s);
}

extern "C" {

// one cost pass at the pose T_row (applyState(guess, x) in an align) over the correspondences of (guess, T_rel), on the raw source
size_t ref_gicp_omp_cost(const float* src, size_t n, size_t ss, const double* scov, const float* tgt, size_t m, size_t ts, const double* tcov,
                         const float* guess_row, const float* Trel_row, double corr_dist, const float* T_row, double* sums) {
  Problem P;
  init_problem(P, src, n, ss, scov, tgt, m, ts, tcov, guess_row, corr_dist);
  const size_t cnt = correspond(P, Trel_row);
  omp_cost_sums(P, T_row, sums);
  return cnt;
}

// f and the 6-gradient of pclomp's functor at x over the correspondences of (guess, T_rel); returns m
size_t ref_gicp_omp_fdf(const float* src, size_t n, size_t ss, const double* scov, const float* tgt, size_t m, size_t ts, const double* tcov,
                        const float* guess_row, const float* Trel_row, double corr_dist, const double* x, double* f, double* g) {
  OmpRule on;
  return ref_gicp_pcl_fdf(src, n, ss, scov, tgt, m, ts, tcov, guess_row, Trel_row, corr_dist, x, f, g);
}

// the whole align under pclomp's pose rule (arguments and stats as ref_gicp_pcl_align)
size_t ref_gicp_omp_align(const float* src, size_t n, size_t ss, const double* scov, const float* tgt, size_t m, size_t ts, const double* tcov,
                          const float* guess_row, const double* cfg, const int* icfg, float* T_out, long* stats, double* trace, size_t trace_cap) {
  OmpRule on;
  return ref_gicp_pcl_align(src, n, ss, scov, tgt, m, ts, tcov, guess_row, cfg, icfg, T_out, stats, trace, trace_cap);
}

// applyState(guess, x) as a row-major float 4x4 (the pose of pclomp's functor at x)
void ref_gicp_omp_pose(const double* x, const float* guess_row, float* T) {
  V6 xv;
  for (int i = 0; i < 6; i++) xv[i] = x[i];
  float A[16];
  apply_state(xv, A);
  omp_pose(A, guess_row, T);
}

}  // extern "C"
