/* tests/vgicp_ref.cpp — TEST INFRASTRUCTURE ONLY: the sequential CPU reference of fast_gicp::FastVGICP that defines the parity of
 * B2R_METHOD_VGICP (hdl_graph_slam_b200/csrc/vgicp.cuh).  Built by the tests with -O2 -ffp-contract=off (no FMA, as the oracle).
 *
 * fast_gicp is an unpinned dependency that is not part of the reference tree, so every choice below is UPSTREAM-RECALL (recalled from
 * fast_vgicp_impl.hpp / gaussian_voxelmap.hpp, as in SURVEY Appendix A) or, where upstream is undefined, this engine's documented rule:
 *   factory (registrations.cpp:48-56): reg_resolution (1.0), reg_transformation_epsilon (0.01), reg_maximum_iterations (64),
 *     reg_correspondence_randomness (20); rotation_epsilon 2e-3; reg_max_correspondence_distance is not read; neighbour search DIRECT1
 *     and voxel mode ADDITIVE (fast_gicp's defaults: hdl never calls the setters).                                  UPSTREAM-RECALL
 *   covariances: FastGICP::calculate_covariances (PLANE) of both clouds, passed in by the caller (the oracle computes them).
 *   voxel map (GaussianVoxelMap::create_voxelmap) of the target: cell = (int)floor((double)p / resolution) per axis, a float64 DIVISION
 *     (recall uncertain: GaussianVoxelMap::voxel_coord may subtract half a cell, floor(p / resolution - 0.5), which would move every
 *     cell and every correspondence by half a voxel; fast_gicp is not available to settle it, and this contract keeps floor(p / res));
 *     points appended in ascending index: num_points++, mean += (x, y, z) in float64, cov += C_i; finalize: mean /= num_points,
 *     cov /= num_points; no minimum point count.                                                                   UPSTREAM-RECALL
 *   a point with a non-finite coordinate belongs to no voxel and has no correspondence (upstream's int cast is undefined there).  ENGINE
 *   cells are limited to [-2^20, 2^20) per axis (21-bit keys): a finite target point beyond fails the build (status 1); a source point
 *     that transforms beyond has no correspondence (no voxel can be there).                                        ENGINE
 *   update_correspondences (DIRECT1): t = T (x, y, z, 1) in float64 with T the LM's Isometry3d, each row ((r0 x + r1 y) + r2 z) + t0;
 *     the correspondence is the voxel of cell floor(t / resolution), or none;
 *     M = (cov_B + R cov_A R^T)^-1 (3x3, the (3,3) entry of the 4x4 pinned), GICP's operation order.               UPSTREAM-RECALL
 *   linearize: w = sqrt((double)num_points), e = mean_B - T mean_A, cost += w e^T M e, H += w J^T M J, b += w J^T M e,
 *     J = [skew(T mean_A) | -I]; compute_error(xi) reuses the correspondences and M of the linearisation point.    UPSTREAM-RECALL
 *   optimiser: LsqRegistration::step_lm with FastGICP's convergence test, exactly the oracle's (a singular / non-finite step ends the
 *     registration as "lm not converged", pose kept).
 */
#include "../oracle/linalg.hpp"
#include <array>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <algorithm>
#include <map>
#include <vector>

using orc::inv3;
using orc::ldlt6_solve;
using orc::mul3;
using orc::mul3_abt;

namespace {

constexpr long long kBias = 1ll << 20;

struct Voxel {
  int n = 0;
  double mean[3] = {0, 0, 0};
  double cov[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
};

struct VMap {
  double res;
  std::map<std::array<int, 3>, int> index;  // cell -> voxel index (ascending cell order)
  std::vector<std::array<int, 3>> cells;
  std::vector<Voxel> vox;
};

bool finite3(const float* p) { return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]); }

// false: outside the key range (or not finite)
bool cell_of(const double* t, double res, std::array<int, 3>& c) {
  for (int a = 0; a < 3; a++) {
    const double f = std::floor(t[a] / res);
    if (!(f >= -(double)kBias && f < (double)kBias)) return false;
    c[a] = (int)f;
  }
  return true;
}

void xform(const double* T, const float* p, double* t) {
  const double x = p[0], y = p[1], z = p[2];
  for (int r = 0; r < 3; r++) t[r] = ((T[r * 4 + 0] * x + T[r * 4 + 1] * y) + T[r * 4 + 2] * z) + T[r * 4 + 3];
}

double linearize(const VMap& M, const float* src, size_t n, size_t stride, const double* scov, const double* T, int32_t* vox_of,
                 double* mahal, double* H, double* b) {
  const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
  double cost = 0.0;
  std::memset(H, 0, 36 * sizeof(double));
  std::memset(b, 0, 6 * sizeof(double));
  for (size_t i = 0; i < n; i++) {
    const float* p = src + i * stride;
    vox_of[i] = -1;
    if (!finite3(p)) continue;
    double t[3];
    xform(T, p, t);
    std::array<int, 3> c;
    if (!cell_of(t, M.res, c)) continue;
    auto it = M.index.find(c);
    if (it == M.index.end()) continue;
    const int v = it->second;
    vox_of[i] = v;
    const Voxel& V = M.vox[v];
    double tmp[9], rcr[9], Mi[9];
    mul3(R, scov + i * 9, tmp);
    mul3_abt(tmp, R, rcr);
    for (int a = 0; a < 9; a++) rcr[a] = V.cov[a] + rcr[a];
    inv3(rcr, Mi);
    std::memcpy(mahal + i * 9, Mi, sizeof(Mi));
    const double w = std::sqrt((double)V.n);
    double e[3], Me[3];
    for (int r = 0; r < 3; r++) e[r] = V.mean[r] - t[r];
    for (int r = 0; r < 3; r++) Me[r] = Mi[r * 3 + 0] * e[0] + Mi[r * 3 + 1] * e[1] + Mi[r * 3 + 2] * e[2];
    cost += w * (e[0] * Me[0] + e[1] * Me[1] + e[2] * Me[2]);
    const double J[18] = {0.0, -t[2], t[1], -1, 0, 0, t[2], 0.0, -t[0], 0, -1, 0, -t[1], t[0], 0.0, 0, 0, -1};
    double MJ[18];
    for (int r = 0; r < 3; r++)
      for (int cc = 0; cc < 6; cc++) MJ[r * 6 + cc] = Mi[r * 3 + 0] * J[0 * 6 + cc] + Mi[r * 3 + 1] * J[1 * 6 + cc] + Mi[r * 3 + 2] * J[2 * 6 + cc];
    for (int r = 0; r < 6; r++) {
      for (int cc = 0; cc < 6; cc++) H[r * 6 + cc] += w * (J[0 * 6 + r] * MJ[0 * 6 + cc] + J[1 * 6 + r] * MJ[1 * 6 + cc] + J[2 * 6 + r] * MJ[2 * 6 + cc]);
      b[r] += w * (J[0 * 6 + r] * Me[0] + J[1 * 6 + r] * Me[1] + J[2 * 6 + r] * Me[2]);
    }
  }
  return cost;
}

double error(const VMap& M, const float* src, size_t n, size_t stride, const int32_t* vox_of, const double* mahal, const double* T) {
  double cost = 0.0;
  for (size_t i = 0; i < n; i++) {
    const int v = vox_of[i];
    if (v < 0) continue;
    const Voxel& V = M.vox[v];
    double t[3], e[3], Me[3];
    xform(T, src + i * stride, t);
    const double* Mi = mahal + i * 9;
    for (int r = 0; r < 3; r++) e[r] = V.mean[r] - t[r];
    for (int r = 0; r < 3; r++) Me[r] = Mi[r * 3 + 0] * e[0] + Mi[r * 3 + 1] * e[1] + Mi[r * 3 + 2] * e[2];
    cost += std::sqrt((double)V.n) * (e[0] * Me[0] + e[1] * Me[1] + e[2] * Me[2]);
  }
  return cost;
}

// so3 / se3 restatement (SURVEY A.4), as the oracle's LM uses it
void se3_exp(const double* a, double* D) {
  const double ox = a[0], oy = a[1], oz = a[2];
  const double theta_sq = ox * ox + oy * oy + oz * oz;
  const double theta = std::sqrt(theta_sq);
  double imag, real;
  if (theta_sq < 1e-10) {
    const double theta_quad = theta_sq * theta_sq;
    imag = 0.5 - 1.0 / 48.0 * theta_sq + 1.0 / 3840.0 * theta_quad;
    real = 1.0 - 1.0 / 8.0 * theta_sq + 1.0 / 384.0 * theta_quad;
  } else {
    const double th = std::sqrt(theta_sq);
    imag = std::sin(0.5 * th) / th;
    real = std::cos(0.5 * th);
  }
  const double qw = real, qx = imag * ox, qy = imag * oy, qz = imag * oz;
  const double tx = 2 * qx, ty = 2 * qy, tz = 2 * qz;
  const double twx = tx * qw, twy = ty * qw, twz = tz * qw;
  const double txx = tx * qx, txy = ty * qx, txz = tz * qx;
  const double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  const double R[9] = {1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)};
  const double Om[9] = {0, -oz, oy, oz, 0, -ox, -oy, ox, 0};
  double Om2[9], V[9];
  mul3(Om, Om, Om2);
  if (theta < 1e-10) {
    std::memcpy(V, R, sizeof(V));
  } else {
    const double c1 = (1.0 - std::cos(theta)) / theta_sq;
    const double c2 = (theta - std::sin(theta)) / (theta_sq * theta);
    for (int i = 0; i < 9; i++) V[i] = ((i % 4 == 0) ? 1.0 : 0.0) + c1 * Om[i] + c2 * Om2[i];
  }
  for (int i = 0; i < 16; i++) D[i] = 0;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) D[r * 4 + c] = R[r * 3 + c];
    D[r * 4 + 3] = V[r * 3 + 0] * a[3] + V[r * 3 + 1] * a[4] + V[r * 3 + 2] * a[5];
  }
  D[15] = 1.0;
}

bool is_converged(const double* D, double rot_eps, double trans_eps) {
  double mr = 0, mt = 0;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) mr = std::max(mr, 1.0 / rot_eps * std::fabs(D[r * 4 + c] - (r == c ? 1.0 : 0.0)));
    mt = std::max(mt, 1.0 / trans_eps * std::fabs(D[r * 4 + 3]));
  }
  return std::max(mr, mt) < 1;
}

void mul4_iso(const double* A, const double* B, double* O) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++) {
      double s = A[r * 4 + 0] * B[0 * 4 + c] + A[r * 4 + 1] * B[1 * 4 + c] + A[r * 4 + 2] * B[2 * 4 + c];
      if (c == 3) s += A[r * 4 + 3];
      O[r * 4 + c] = s;
    }
  O[12] = O[13] = O[14] = 0;
  O[15] = 1;
}

}  // namespace

extern "C" {

/* voxel map of the target; cov: m x 9 (row-major 3x3, rows of non-finite points are ignored).  *status = 1: a finite point lies
 * beyond the 21-bit cell range (the map is returned empty) */
void* ref_vgicp_map(const float* tgt, size_t m, size_t stride, const double* cov, double res, int* status) {
  VMap* M = new VMap();
  M->res = res;
  *status = 0;
  std::map<std::array<int, 3>, Voxel> acc;
  for (size_t i = 0; i < m; i++) {
    const float* p = tgt + i * stride;
    if (!finite3(p)) continue;
    const double t[3] = {(double)p[0], (double)p[1], (double)p[2]};
    std::array<int, 3> c;
    if (!cell_of(t, res, c)) { *status = 1; continue; }
    Voxel& V = acc[c];
    V.n++;
    for (int a = 0; a < 3; a++) V.mean[a] += t[a];
    for (int a = 0; a < 9; a++) V.cov[a] += cov[i * 9 + a];
  }
  if (*status) return M;
  for (auto& kv : acc) {
    Voxel V = kv.second;
    for (int a = 0; a < 3; a++) V.mean[a] /= V.n;
    for (int a = 0; a < 9; a++) V.cov[a] /= V.n;
    M->index[kv.first] = (int)M->vox.size();
    M->cells.push_back(kv.first);
    M->vox.push_back(V);
  }
  return M;
}

void ref_vgicp_free(void* m) { delete static_cast<VMap*>(m); }

/* returns V; arrays (cells 3V, counts V, mean 3V, cov 9V) may be NULL */
size_t ref_vgicp_voxels(const void* m, int32_t* cells, int32_t* counts, double* mean, double* cov) {
  const VMap& M = *static_cast<const VMap*>(m);
  for (size_t v = 0; v < M.vox.size(); v++) {
    if (cells) for (int a = 0; a < 3; a++) cells[v * 3 + a] = M.cells[v][a];
    if (counts) counts[v] = M.vox[v].n;
    if (mean) for (int a = 0; a < 3; a++) mean[v * 3 + a] = M.vox[v].mean[a];
    if (cov) for (int a = 0; a < 9; a++) cov[v * 9 + a] = M.vox[v].cov[a];
  }
  return M.vox.size();
}

/* update_correspondences + linearize at T (row-major 4x4 double): H[36], b[6], vox_of[n]; returns the cost */
double ref_vgicp_linearize(const void* m, const float* src, size_t n, size_t stride, const double* scov, const double* T, double* H, double* b,
                           int32_t* vox_of) {
  std::vector<double> mahal(n * 9 + 9);
  return linearize(*static_cast<const VMap*>(m), src, n, stride, scov, T, vox_of, mahal.data(), H, b);
}

/* compute_error at T2 with the correspondences and M of the linearisation at T1 */
double ref_vgicp_error(const void* m, const float* src, size_t n, size_t stride, const double* scov, const double* T1, const double* T2) {
  std::vector<double> mahal(n * 9 + 9);
  std::vector<int32_t> vox(n + 1);
  double H[36], b[6];
  const VMap& M = *static_cast<const VMap*>(m);
  linearize(M, src, n, stride, scov, T1, vox.data(), mahal.data(), H, b);
  return error(M, src, n, stride, vox.data(), mahal.data(), T2);
}

/* align(): cfg_d = {transformation_epsilon, rotation_epsilon}, cfg_i = {max_iterations}; guess / T_out row-major float;
 * out = {converged, iterations, lm_failed}; T64 (16, may be NULL) = the pose before the float cast */
void ref_vgicp_align(const void* m, const float* src, size_t n, size_t stride, const double* scov, const double* cfg_d, const int* cfg_i,
                     const float* guess, float* T_out, int* out, double* T64) {
  const VMap& M = *static_cast<const VMap*>(m);
  double x0[16];
  for (int i = 0; i < 16; i++) x0[i] = (double)guess[i];
  x0[12] = x0[13] = x0[14] = 0; x0[15] = 1;
  out[0] = out[1] = out[2] = 0;
  std::vector<int32_t> vox(n + 1);
  std::vector<double> mahal(n * 9 + 9);
  double lambda = -1.0;
  bool converged = false, lm_failed = false;
  int it = 0;
  for (it = 0; it < cfg_i[0] && !converged; it++) {
    double H[36], b[6], delta[16];
    const double y0 = linearize(M, src, n, stride, scov, x0, vox.data(), mahal.data(), H, b);
    if (lambda < 0.0) {
      double mx = 0;
      for (int i = 0; i < 6; i++) mx = std::max(mx, std::fabs(H[i * 6 + i]));
      lambda = 1e-9 * mx;
    }
    double nu = 2.0;
    bool ok = false;
    for (int li = 0; li < 10; li++) {
      double A[36], nb[6], d[6];
      for (int i = 0; i < 36; i++) A[i] = H[i] + ((i % 7 == 0) ? lambda : 0.0);
      for (int i = 0; i < 6; i++) nb[i] = -b[i];
      bool solved = ldlt6_solve(A, nb, d);
      for (int i = 0; i < 6; i++) solved &= std::isfinite(d[i]);
      if (!solved) break;
      se3_exp(d, delta);
      double xi[16];
      mul4_iso(delta, x0, xi);
      const double yi = error(M, src, n, stride, vox.data(), mahal.data(), xi);
      double den = 0;
      for (int i = 0; i < 6; i++) den += d[i] * (lambda * d[i] - b[i]);
      const double rho = (y0 - yi) / den;
      if (rho < 0) {
        if (is_converged(delta, cfg_d[1], cfg_d[0])) { ok = true; break; }
        lambda = nu * lambda;
        nu = 2 * nu;
        continue;
      }
      const double t = 2 * rho - 1;
      lambda = lambda * std::max(1.0 / 3.0, 1 - t * t * t);
      std::memcpy(x0, xi, sizeof(xi));
      ok = true;
      break;
    }
    if (!ok) { lm_failed = true; it++; break; }
    converged = is_converged(delta, cfg_d[1], cfg_d[0]);
  }
  for (int i = 0; i < 16; i++) T_out[i] = (float)x0[i];
  if (T64) std::memcpy(T64, x0, sizeof(x0));
  out[0] = converged ? 1 : 0;
  out[1] = it;
  out[2] = lm_failed ? 1 : 0;
}

}  // extern "C"
