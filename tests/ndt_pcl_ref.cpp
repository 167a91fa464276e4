// tests/ndt_pcl_ref.cpp — TEST INFRASTRUCTURE ONLY: the sequential CPU reference of pcl::NormalDistributionsTransform (PCL 1.10),
// the factory's `NDT` branch (registrations.cpp:93-100), which the engine's B2R_METHOD_NDT_PCL must reproduce.  PCL itself cannot be
// built here (it is fetched unpinned, with Eigen and FLANN), so this file DEFINES parity; the choices, written from PCL 1.10:
//  * Factory: transformation epsilon, maximum iterations and resolution only; step size 0.1 and outlier ratio 0.55 are PCL's
//    defaults; reg_nn_search_method / reg_num_threads are not read.
//  * Target: the voxel map is the oracle's (oracle/ndt.cpp: keys, means, covariances, 1 % eigenvalue clamp, inverse, nr_points = -1
//    invalidation), passed in from its dump.  In addition VoxelGridCovariance::filter(true) emits, for every leaf of >= 6 points
//    (counted BEFORE invalidation), a centroid into the searchable cloud, in ascending leaf key: the float32 sum of the leaf's
//    x, y, z in input index order divided by (float)nr_points.  An emitted leaf that is invalidated stays searchable with the
//    inverse it has: zero when its eigenvalue check failed, the non-finite inverse when that was the failure.
//  * Neighbourhood: target_cells_.radiusSearch(x_trans_pt, resolution_): FLANN KDTreeSingleIndex<L2_Simple<float>> with the radius
//    passed as (float)(r * r): a centroid is a neighbour iff ((dx*dx + dy*dy) + dz*dz) < r2 in float32 without FMA, d = q - c
//    (strict).  Results ascend by (d2, centroid index); the order only moves float64 rounding.  Returned leaves are not checked for
//    nr_points >= 6; a non-finite transformed point has no neighbours.
//  * Per (point, neighbour), float64, in exactly the order written in term() (left to right, no FMA: -ffp-contract=off):
//    updateDerivatives with computePointDerivatives(x) of the ORIGINAL point promoted to double.  When e = d2 exp(...) fails
//    the range check the term adds nothing, not even its score (updateDerivatives returns 0).  x_trans . (C * 0) outside the
//    angular block of point_hessian_ is taken as 0.  H holds all 36 entries as accumulated (not symmetrised).
//  * computeHessian / updateHessian (after a line search that iterated) is the same term's Hessian part.
//  * Per-point sums are added serially in point index order.
//  * Driver: computeTransformation / computeStepLengthMT as oracle/ndt.cpp (guess pre-transform, Eigen 3.3 eulerAngles(0,1,2),
//    the 6x6 SVD solve, More-Thuente with the mt_interval_flag polarity, fixed_iterations).
#include "../oracle/kdtree.hpp"
#include "../oracle/linalg.hpp"
#include <omp.h>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <algorithm>
#include <unordered_map>
#include <vector>

namespace {

struct Leaf {
  int64_t key;
  int npts;
  double mean[3], icov[9];
};

struct Map {
  float leaf = 0.f, inv_leaf = 0.f;
  int min_b[3] = {0, 0, 0}, div_b[3] = {0, 0, 0};
  bool empty = true;
  std::vector<Leaf> leaves;       // ascending key (the oracle's dump)
  std::vector<int> cent_leaf;     // centroid index -> leaf slot
  std::vector<float> cent;        // centroid cloud (x, y, z)
  orc::KdTree tree;
};

struct Cfg {
  double resolution, step_size, outlier_ratio, transformation_epsilon;
  int max_iterations, mt_interval_flag, fixed_iterations, threads;
};

struct Consts {
  double d1, d2;
  double jang[8][3], hang[15][3];
};

void gauss(const Cfg& c, Consts& K) {
  double gauss_c1 = 10 * (1 - c.outlier_ratio);
  double gauss_c2 = c.outlier_ratio / std::pow(c.resolution, 3);
  double gauss_d3 = -std::log(gauss_c2);
  K.d1 = -std::log(gauss_c1 + gauss_c2) - gauss_d3;
  K.d2 = -2 * std::log((-std::log(gauss_c1 * std::exp(-0.5) + gauss_c2) - gauss_d3) / K.d1);
}

void angle_derivs(const double* p, Consts& K) {
  double cx, cy, cz, sx, sy, sz;
  if (std::fabs(p[3]) < 10e-5) { cx = 1.0; sx = 0.0; } else { cx = std::cos(p[3]); sx = std::sin(p[3]); }
  if (std::fabs(p[4]) < 10e-5) { cy = 1.0; sy = 0.0; } else { cy = std::cos(p[4]); sy = std::sin(p[4]); }
  if (std::fabs(p[5]) < 10e-5) { cz = 1.0; sz = 0.0; } else { cz = std::cos(p[5]); sz = std::sin(p[5]); }
  const double J[8][3] = {
      {(-sx * sz + cx * sy * cz), (-sx * cz - cx * sy * sz), (-cx * cy)},
      {(cx * sz + sx * sy * cz), (cx * cz - sx * sy * sz), (-sx * cy)},
      {(-sy * cz), sy * sz, cy},
      {sx * cy * cz, (-sx * cy * sz), sx * sy},
      {(-cx * cy * cz), cx * cy * sz, (-cx * sy)},
      {(-cy * sz), (-cy * cz), 0},
      {(cx * cz - sx * sy * sz), (-cx * sz - sx * sy * cz), 0},
      {(sx * cz + cx * sy * sz), (cx * sy * cz - sx * sz), 0}};
  const double Hh[15][3] = {
      {(-cx * sz - sx * sy * cz), (-cx * cz + sx * sy * sz), sx * cy},
      {(-sx * sz + cx * sy * cz), (-cx * sy * sz - sx * cz), (-cx * cy)},
      {(cx * cy * cz), (-cx * cy * sz), (cx * sy)},
      {(sx * cy * cz), (-sx * cy * sz), (sx * sy)},
      {(-sx * cz - cx * sy * sz), (sx * sz - cx * sy * cz), 0},
      {(cx * cz - sx * sy * sz), (-sx * sy * cz - cx * sz), 0},
      {(-cy * cz), (cy * sz), (sy)},
      {(-sx * sy * cz), (sx * sy * sz), (sx * cy)},
      {(cx * sy * cz), (-cx * sy * sz), (-cx * cy)},
      {(sy * sz), (sy * cz), 0},
      {(-sx * cy * sz), (-sx * cy * cz), 0},
      {(cx * cy * sz), (cx * cy * cz), 0},
      {(-cy * cz), (cy * sz), 0},
      {(-cx * sz - sx * sy * cz), (-cx * cz + sx * sy * sz), 0},
      {(-sx * sz + cx * sy * cz), (-cx * sy * sz - sx * cz), 0}};
  std::memcpy(K.jang, J, sizeof(J));
  std::memcpy(K.hang, Hh, sizeof(Hh));
}

// Translation * AngleAxis(x) * AngleAxis(y) * AngleAxis(z), float32, row-major 4x4 (oracle/ndt.cpp pose_to_matrix_f32)
void pose_to_matrix(const double* p, float* T) {
  float ang[3] = {(float)p[3], (float)p[4], (float)p[5]};
  float R[3][9];
  for (int a = 0; a < 3; a++) {
    float s = (float)std::sin((double)ang[a]);
    float c = (float)std::cos((double)ang[a]);
    float omc = 1.0f - c;
    float diag_axis = omc + c;
    float m[9] = {c, 0, 0, 0, c, 0, 0, 0, c};
    if (a == 0) { m[0] = diag_axis; m[5] = 0.f - s; m[7] = 0.f + s; }
    if (a == 1) { m[4] = diag_axis; m[2] = 0.f + s; m[6] = 0.f - s; }
    if (a == 2) { m[8] = diag_axis; m[1] = 0.f - s; m[3] = 0.f + s; }
    std::memcpy(R[a], m, sizeof(m));
  }
  auto mm = [](const float* A, const float* B, float* O) {
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) {
        float u = A[r * 3 + 0] * B[0 * 3 + c];
        float v = A[r * 3 + 1] * B[1 * 3 + c];
        u = u + v;
        v = A[r * 3 + 2] * B[2 * 3 + c];
        O[r * 3 + c] = u + v;
      }
  };
  float xy[9], xyz[9];
  mm(R[0], R[1], xy);
  mm(xy, R[2], xyz);
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[r * 4 + c] = xyz[r * 3 + c];
    T[r * 4 + 3] = (float)p[r];
  }
  T[12] = T[13] = T[14] = 0.f;
  T[15] = 1.f;
}

void euler_xyz(const float* T, float* out) {
  auto m = [&](int r, int c) { return T[r * 4 + c]; };
  float res0 = std::atan2(m(1, 2), m(2, 2));
  float c2 = std::sqrt(m(0, 0) * m(0, 0) + m(0, 1) * m(0, 1));
  float res1;
  if (res0 > 0.f) {
    res0 -= (float)M_PI;
    res1 = std::atan2(-m(0, 2), -c2);
  } else {
    res1 = std::atan2(-m(0, 2), c2);
  }
  float s1 = std::sin(res0), c1 = std::cos(res0);
  float res2 = std::atan2(s1 * m(2, 0) - c1 * m(1, 0), c1 * m(1, 1) - s1 * m(2, 1));
  out[0] = -res0; out[1] = -res1; out[2] = -res2;
}

inline void xform(const float* Tf, const float* p, float* o) {
  for (int r = 0; r < 3; r++) {
    float a = Tf[r * 4 + 0] * p[0];
    float b = Tf[r * 4 + 1] * p[1];
    float c = Tf[r * 4 + 2] * p[2];
    float s = a + b;
    s = s + c;
    o[r] = s + Tf[r * 4 + 3];
  }
}

void radius_rec(const orc::KdTree& T, int node, const float* q, float r2, std::vector<std::pair<float, int>>& out) {
  const orc::KdTree::Node& nd = T.nodes[node];
  if (!(orc::KdTree::box_dist2(q, nd) < r2)) return;  // a lower bound of every d2 in the box, in the same float32 order
  if (nd.left < 0) {
    for (int i = nd.begin; i < nd.end; i++) {
      const int pi = T.perm[i];
      const float d2 = orc::KdTree::dist2(q, T.P(pi));
      if (d2 < r2) out.emplace_back(d2, pi);
    }
    return;
  }
  radius_rec(T, nd.left, q, r2, out);
  radius_rec(T, nd.right, q, r2, out);
}

// radiusSearch: centroid indices ascending by (d2, index)
void radius(const Map& M, const float* q, float r2, std::vector<std::pair<float, int>>& out) {
  out.clear();
  if (M.cent_leaf.empty() || !(std::isfinite(q[0]) && std::isfinite(q[1]) && std::isfinite(q[2]))) return;
  radius_rec(M.tree, 0, q, r2, out);
  std::sort(out.begin(), out.end());
}

// one (point, neighbour) term of updateDerivatives, the order of every float64 operation as written
void term(const Consts& K, const Leaf& L, const double* xt, const double* jx, const double* hx, bool hess, double& score, double* g, double* H) {
  const double q0 = xt[0] - L.mean[0], q1 = xt[1] - L.mean[1], q2 = xt[2] - L.mean[2];
  const double* C = L.icov;
  double Cq[3];
  for (int r = 0; r < 3; r++) Cq[r] = (C[r * 3 + 0] * q0 + C[r * 3 + 1] * q1) + C[r * 3 + 2] * q2;
  const double qCq = (q0 * Cq[0] + q1 * Cq[1]) + q2 * Cq[2];
  double e = std::exp((-K.d2 * qCq) / 2.0);
  const double score_inc = -K.d1 * e;
  e = K.d2 * e;
  if (e > 1 || e < 0 || e != e) return;
  e = e * K.d1;
  score += score_inc;
  const double J[3][6] = {{1.0, 0.0, 0.0, 0.0, jx[2], jx[5]}, {0.0, 1.0, 0.0, jx[0], jx[3], jx[6]}, {0.0, 0.0, 1.0, jx[1], jx[4], jx[7]}};
  double CJ[3][6], gq[6];
  for (int r = 0; r < 3; r++)
    for (int i = 0; i < 6; i++) CJ[r][i] = (C[r * 3 + 0] * J[0][i] + C[r * 3 + 1] * J[1][i]) + C[r * 3 + 2] * J[2][i];
  for (int i = 0; i < 6; i++) {
    gq[i] = (q0 * CJ[0][i] + q1 * CJ[1][i]) + q2 * CJ[2][i];
    g[i] += gq[i] * e;
  }
  if (!hess) return;
  const double PH[6][3] = {{0.0, hx[0], hx[1]}, {0.0, hx[2], hx[3]}, {0.0, hx[4], hx[5]}, {hx[6], hx[7], hx[8]}, {hx[9], hx[10], hx[11]}, {hx[12], hx[13], hx[14]}};
  const int blk[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
  for (int ii = 0; ii < 6; ii++)
    for (int jj = 0; jj < 6; jj++) {
      double xh = 0.0;
      if (ii >= 3 && jj >= 3) {
        const double* v = PH[blk[ii - 3][jj - 3]];
        double Cv[3];
        for (int r = 0; r < 3; r++) Cv[r] = (C[r * 3 + 0] * v[0] + C[r * 3 + 1] * v[1]) + C[r * 3 + 2] * v[2];
        xh = (q0 * Cv[0] + q1 * Cv[1]) + q2 * Cv[2];
      }
      const double jcj = (J[0][jj] * CJ[0][ii] + J[1][jj] * CJ[1][ii]) + J[2][jj] * CJ[2][ii];
      H[ii * 6 + jj] += e * (((-K.d2 * gq[ii]) * gq[jj] + xh) + jcj);
    }
}

double derivatives(const Map& M, const float* src, size_t n, size_t stride, const float* Tf, const Cfg& cfg, const Consts& K, double* g_out,
                   double* H_out, bool hess, uint64_t* n_pairs) {
  std::vector<double> sc(n, 0.0), gr(n * 6, 0.0), he(hess ? n * 36 : 0, 0.0);
  std::vector<uint32_t> np(n, 0);
  const float r2 = (float)(cfg.resolution * cfg.resolution);
#pragma omp parallel num_threads(cfg.threads > 0 ? cfg.threads : omp_get_max_threads())
  {
    std::vector<std::pair<float, int>> nb;
#pragma omp for schedule(guided, 64)
    for (long i = 0; i < (long)n; i++) {
      const float* x = src + (size_t)i * stride;
      float xt[3];
      xform(Tf, x, xt);
      radius(M, xt, r2, nb);
      if (nb.empty()) continue;
      const double xd[3] = {(double)x[0], (double)x[1], (double)x[2]};
      double jx[8], hx[15];
      for (int r = 0; r < 8; r++) jx[r] = (xd[0] * K.jang[r][0] + xd[1] * K.jang[r][1]) + xd[2] * K.jang[r][2];
      for (int r = 0; r < 15; r++) hx[r] = (xd[0] * K.hang[r][0] + xd[1] * K.hang[r][1]) + xd[2] * K.hang[r][2];
      const double xtd[3] = {(double)xt[0], (double)xt[1], (double)xt[2]};
      for (const auto& e : nb)
        term(K, M.leaves[M.cent_leaf[e.second]], xtd, jx, hx, hess, sc[i], &gr[(size_t)i * 6], hess ? &he[(size_t)i * 36] : nullptr);
      np[i] = (uint32_t)nb.size();
    }
  }
  double score = 0;
  for (int k = 0; k < 6; k++) g_out[k] = 0;
  if (hess) for (int k = 0; k < 36; k++) H_out[k] = 0;
  uint64_t pairs = 0;
  for (size_t i = 0; i < n; i++) {
    score += sc[i];
    for (int k = 0; k < 6; k++) g_out[k] += gr[i * 6 + k];
    if (hess) for (int k = 0; k < 36; k++) H_out[k] += he[i * 36 + k];
    pairs += np[i];
  }
  if (n_pairs) *n_pairs = pairs;
  return score;
}

double psiMT(double a, double f_a, double f_0, double g_0, double mu) { return f_a - f_0 - mu * g_0 * a; }
double dpsiMT(double g_a, double g_0, double mu) { return g_a - mu * g_0; }
double trialMT(double a_l, double f_l, double g_l, double a_u, double f_u, double g_u, double a_t, double f_t, double g_t) {
  if (f_t > f_l) {
    double z = 3 * (f_t - f_l) / (a_t - a_l) - g_t - g_l;
    double w = std::sqrt(z * z - g_t * g_l);
    double a_c = a_l + (a_t - a_l) * (w - g_l - z) / (g_t - g_l + 2 * w);
    double a_q = a_l - 0.5 * (a_l - a_t) * g_l / (g_l - (f_l - f_t) / (a_l - a_t));
    return (std::fabs(a_c - a_l) < std::fabs(a_q - a_l)) ? a_c : 0.5 * (a_q + a_c);
  } else if (g_t * g_l < 0) {
    double z = 3 * (f_t - f_l) / (a_t - a_l) - g_t - g_l;
    double w = std::sqrt(z * z - g_t * g_l);
    double a_c = a_l + (a_t - a_l) * (w - g_l - z) / (g_t - g_l + 2 * w);
    double a_s = a_l - (a_l - a_t) / (g_l - g_t) * g_l;
    return (std::fabs(a_c - a_t) >= std::fabs(a_s - a_t)) ? a_c : a_s;
  } else if (std::fabs(g_t) <= std::fabs(g_l)) {
    double z = 3 * (f_t - f_l) / (a_t - a_l) - g_t - g_l;
    double w = std::sqrt(z * z - g_t * g_l);
    double a_c = a_l + (a_t - a_l) * (w - g_l - z) / (g_t - g_l + 2 * w);
    double a_s = a_l - (a_l - a_t) / (g_l - g_t) * g_l;
    double a_t_next = (std::fabs(a_c - a_t) < std::fabs(a_s - a_t)) ? a_c : a_s;
    return (a_t > a_l) ? std::min(a_t + 0.66 * (a_u - a_t), a_t_next) : std::max(a_t + 0.66 * (a_u - a_t), a_t_next);
  }
  double z = 3 * (f_t - f_u) / (a_t - a_u) - g_t - g_u;
  double w = std::sqrt(z * z - g_t * g_u);
  return a_u + (a_t - a_u) * (w - g_u - z) / (g_t - g_u + 2 * w);
}
bool updateMT(double& a_l, double& f_l, double& g_l, double& a_u, double& f_u, double& g_u, double a_t, double f_t, double g_t) {
  if (f_t > f_l) { a_u = a_t; f_u = f_t; g_u = g_t; return false; }
  if (g_t * (a_l - a_t) > 0) { a_l = a_t; f_l = f_t; g_l = g_t; return false; }
  if (g_t * (a_l - a_t) < 0) { a_u = a_l; f_u = f_l; g_u = g_l; a_l = a_t; f_l = f_t; g_l = g_t; return false; }
  return true;
}

Cfg make_cfg(const double* d, const int* i) {
  Cfg c;
  c.resolution = d[0]; c.step_size = d[1]; c.outlier_ratio = d[2]; c.transformation_epsilon = d[3];
  c.max_iterations = i[0]; c.mt_interval_flag = i[1]; c.fixed_iterations = i[2]; c.threads = i[3];
  return c;
}

}  // namespace

extern "C" {

// the map: the target cloud, the resolution and the oracle's voxel dump (leaf keys ascending)
void* ref_pcl_map(const float* tgt, size_t m, size_t stride, float leaf, size_t nv, const int64_t* keys, const int32_t* npts, const double* mean,
                  const double* icov, const int32_t* min_b, const int32_t* div_b) {
  Map* M = new Map();
  M->leaf = leaf;
  M->inv_leaf = 1.0f / leaf;
  M->empty = nv == 0;
  for (int d = 0; d < 3; d++) { M->min_b[d] = min_b[d]; M->div_b[d] = div_b[d]; }
  std::unordered_map<int64_t, int> slot;
  M->leaves.resize(nv);
  for (size_t v = 0; v < nv; v++) {
    Leaf& L = M->leaves[v];
    L.key = keys[v];
    L.npts = npts[v];
    std::memcpy(L.mean, mean + 3 * v, sizeof(L.mean));
    std::memcpy(L.icov, icov + 9 * v, sizeof(L.icov));
    slot[L.key] = (int)v;
  }
  if (M->empty) return M;
  // centroids: sequential float32 sums in input index order
  std::vector<float> sum(3 * nv, 0.f);
  std::vector<int> cnt(nv, 0);
  const int64_t mul1 = div_b[0], mul2 = (int64_t)div_b[0] * div_b[1];
  for (size_t i = 0; i < m; i++) {
    const float* p = tgt + i * stride;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
    const int64_t i0 = (int64_t)(std::floor(p[0] * M->inv_leaf) - (float)min_b[0]);
    const int64_t i1 = (int64_t)(std::floor(p[1] * M->inv_leaf) - (float)min_b[1]);
    const int64_t i2 = (int64_t)(std::floor(p[2] * M->inv_leaf) - (float)min_b[2]);
    const int v = slot.at(i0 + i1 * mul1 + i2 * mul2);
    for (int d = 0; d < 3; d++) sum[3 * v + d] += p[d];
    cnt[v]++;
  }
  for (size_t v = 0; v < nv; v++) {
    if (cnt[v] < 6) continue;
    const float fc = (float)cnt[v];
    for (int d = 0; d < 3; d++) M->cent.push_back(sum[3 * v + d] / fc);
    M->cent_leaf.push_back((int)v);
  }
  M->tree.build(M->cent.data(), M->cent_leaf.size(), 3);
  return M;
}

void ref_pcl_free(void* M) { delete static_cast<Map*>(M); }

size_t ref_pcl_centroids(const void* m, int64_t* keys, float* xyz) {
  const Map* M = static_cast<const Map*>(m);
  const size_t c = M->cent_leaf.size();
  for (size_t k = 0; k < c; k++) {
    if (keys) keys[k] = M->leaves[M->cent_leaf[k]].key;
    if (xyz) std::memcpy(xyz + 3 * k, &M->cent[3 * k], 3 * sizeof(float));
  }
  return c;
}

// radius neighbours of every source point at pose p: counts[n]; leaf keys ascending within each point (first `capacity`)
size_t ref_pcl_neighbors(const void* m, const float* src, size_t n, size_t stride, const double* cfg_d, const int* cfg_i, const double* p,
                         uint32_t* counts, int64_t* keys, size_t capacity) {
  const Map* M = static_cast<const Map*>(m);
  const Cfg cfg = make_cfg(cfg_d, cfg_i);
  float Tf[16];
  pose_to_matrix(p, Tf);
  const float r2 = (float)(cfg.resolution * cfg.resolution);
  std::vector<std::pair<float, int>> nb;
  std::vector<int64_t> ks;
  size_t total = 0;
  for (size_t i = 0; i < n; i++) {
    float xt[3];
    xform(Tf, src + i * stride, xt);
    radius(*M, xt, r2, nb);
    ks.clear();
    for (const auto& e : nb) ks.push_back(M->leaves[M->cent_leaf[e.second]].key);
    std::sort(ks.begin(), ks.end());
    for (size_t t = 0; t < ks.size(); t++)
      if (keys && total + t < capacity) keys[total + t] = ks[t];
    if (counts) counts[i] = (uint32_t)ks.size();
    total += ks.size();
  }
  return total;
}

double ref_pcl_derivatives(const void* m, const float* src, size_t n, size_t stride, const double* cfg_d, const int* cfg_i, const double* p,
                           double* g, double* H, uint64_t* n_pairs) {
  const Map* M = static_cast<const Map*>(m);
  const Cfg cfg = make_cfg(cfg_d, cfg_i);
  Consts K;
  gauss(cfg, K);
  angle_derivs(p, K);
  float Tf[16];
  pose_to_matrix(p, Tf);
  return derivatives(*M, src, n, stride, Tf, cfg, K, g, H, true, n_pairs);
}

// out_i: converged, iterations, derivative passes, Hessian passes; T: row-major float 4x4; guess: row-major float 4x4
void ref_pcl_align(const void* m, const float* src, size_t n, size_t stride, const double* cfg_d, const int* cfg_i, const float* guess, float* T_out,
                   int* out_i, double* p_out) {
  const Map* M = static_cast<const Map*>(m);
  const Cfg cfg = make_cfg(cfg_d, cfg_i);
  float Tfinal[16];
  for (int i = 0; i < 16; i++) Tfinal[i] = (i % 5 == 0) ? 1.f : 0.f;
  std::memcpy(T_out, Tfinal, sizeof(Tfinal));
  out_i[0] = out_i[1] = out_i[2] = out_i[3] = 0;
  if (n == 0 || M->empty) return;
  Consts K;
  gauss(cfg, K);
  bool ident = true;
  for (int i = 0; i < 16; i++) ident &= (guess[i] == ((i % 5 == 0) ? 1.f : 0.f));
  if (!ident) std::memcpy(Tfinal, guess, sizeof(Tfinal));
  double p[6];
  {
    float e[3];
    euler_xyz(Tfinal, e);
    p[0] = Tfinal[3]; p[1] = Tfinal[7]; p[2] = Tfinal[11];
    p[3] = e[0]; p[4] = e[1]; p[5] = e[2];
  }
  double g[6], H[36];
  int passes = 0, hpasses = 0;
  angle_derivs(p, K);
  double score = derivatives(*M, src, n, stride, Tfinal, cfg, K, g, H, true, nullptr);
  passes++;
  int nr_iterations = 0;
  bool converged = false;
  while (!converged) {
    double ng[6], dp[6];
    for (int i = 0; i < 6; i++) ng[i] = -g[i];
    orc::svd6_solve_sym(H, ng, dp);
    double nrm = 0;
    for (int i = 0; i < 6; i++) nrm += dp[i] * dp[i];
    nrm = std::sqrt(nrm);
    if (nrm == 0 || nrm != nrm) { converged = (nrm == nrm); break; }
    for (int i = 0; i < 6; i++) dp[i] /= nrm;
    double step_max = cfg.step_size, step_min = cfg.transformation_epsilon / 2;
    double phi_0 = -score, d_phi_0 = 0;
    for (int i = 0; i < 6; i++) d_phi_0 += g[i] * dp[i];
    d_phi_0 = -d_phi_0;
    double a_t = 0;
    bool skip = false;
    if (d_phi_0 >= 0) {
      if (d_phi_0 == 0) { skip = true; a_t = 0; }
      else { d_phi_0 *= -1; for (int i = 0; i < 6; i++) dp[i] *= -1; }
    }
    if (!skip) {
      const double mu = 1.e-4, nu = 0.9;
      double a_l = 0, a_u = 0;
      double f_l = psiMT(a_l, phi_0, phi_0, d_phi_0, mu), g_l = dpsiMT(d_phi_0, d_phi_0, mu);
      double f_u = psiMT(a_u, phi_0, phi_0, d_phi_0, mu), g_u = dpsiMT(d_phi_0, d_phi_0, mu);
      bool interval_converged = cfg.mt_interval_flag ? ((step_max - step_min) < 0) : ((step_max - step_min) > 0);
      bool open_interval = true;
      int step_iterations = 0;
      a_t = std::max(std::min(nrm, step_max), step_min);
      double x_t[6];
      for (int i = 0; i < 6; i++) x_t[i] = p[i] + dp[i] * a_t;
      pose_to_matrix(x_t, Tfinal);
      angle_derivs(x_t, K);
      score = derivatives(*M, src, n, stride, Tfinal, cfg, K, g, H, true, nullptr);
      passes++;
      double phi_t = -score, d_phi_t = 0;
      for (int i = 0; i < 6; i++) d_phi_t += g[i] * dp[i];
      d_phi_t = -d_phi_t;
      double psi_t = psiMT(a_t, phi_t, phi_0, d_phi_0, mu), d_psi_t = dpsiMT(d_phi_t, d_phi_0, mu);
      while (!interval_converged && step_iterations < 10 && !(psi_t <= 0 && d_phi_t <= -nu * d_phi_0)) {
        if (open_interval) a_t = trialMT(a_l, f_l, g_l, a_u, f_u, g_u, a_t, psi_t, d_psi_t);
        else a_t = trialMT(a_l, f_l, g_l, a_u, f_u, g_u, a_t, phi_t, d_phi_t);
        a_t = std::max(std::min(a_t, step_max), step_min);
        for (int i = 0; i < 6; i++) x_t[i] = p[i] + dp[i] * a_t;
        pose_to_matrix(x_t, Tfinal);
        angle_derivs(x_t, K);
        score = derivatives(*M, src, n, stride, Tfinal, cfg, K, g, H, false, nullptr);
        passes++;
        phi_t = -score;
        d_phi_t = 0;
        for (int i = 0; i < 6; i++) d_phi_t += g[i] * dp[i];
        d_phi_t = -d_phi_t;
        psi_t = psiMT(a_t, phi_t, phi_0, d_phi_0, mu);
        d_psi_t = dpsiMT(d_phi_t, d_phi_0, mu);
        if (open_interval && (psi_t <= 0 && d_psi_t >= 0)) {
          open_interval = false;
          f_l = f_l + phi_0 - mu * d_phi_0 * a_l;
          g_l = g_l + mu * d_phi_0;
          f_u = f_u + phi_0 - mu * d_phi_0 * a_u;
          g_u = g_u + mu * d_phi_0;
        }
        if (open_interval) interval_converged = updateMT(a_l, f_l, g_l, a_u, f_u, g_u, a_t, psi_t, d_psi_t);
        else interval_converged = updateMT(a_l, f_l, g_l, a_u, f_u, g_u, a_t, phi_t, d_phi_t);
        step_iterations++;
      }
      if (step_iterations) {  // computeHessian: updateDerivatives' Hessian term at the accepted pose
        double gs[6];
        derivatives(*M, src, n, stride, Tfinal, cfg, K, gs, H, true, nullptr);
        passes++;
        hpasses++;
      }
    }
    const double delta_p_norm = a_t;
    for (int i = 0; i < 6; i++) { dp[i] *= delta_p_norm; p[i] += dp[i]; }
    if (cfg.fixed_iterations > 0) {
      if (nr_iterations + 1 >= cfg.fixed_iterations) converged = true;
    } else if (nr_iterations > cfg.max_iterations || (nr_iterations && (std::fabs(delta_p_norm) < cfg.transformation_epsilon))) {
      converged = true;
    }
    nr_iterations++;
  }
  std::memcpy(T_out, Tfinal, sizeof(Tfinal));
  out_i[0] = converged ? 1 : 0;
  out_i[1] = nr_iterations;
  out_i[2] = passes;
  out_i[3] = hpasses;
  if (p_out) std::memcpy(p_out, p, sizeof(p));
}

}  // extern "C"
