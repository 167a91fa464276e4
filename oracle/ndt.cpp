// oracle/ndt.cpp — TEST INFRASTRUCTURE ONLY (CPU oracle; see oracle.h header).
//
// Restates pclomp::NormalDistributionsTransform + pclomp::VoxelGridCovariance (koide3/ndt_omp; SURVEY.md A.2/A.3),
// the default engine of the reference's factory (/root/reference/src/hdl_graph_slam/registrations.cpp:26,101-120),
// and pcl::VoxelGrid (A.5; apps/prefiltering_nodelet.cpp:54-58,138-149).   "parity unpinned" (see oracle.h).
//
// Deliberate, documented choices (SURVEY.md §7 "Upstream drift"):
//  * per-(point,cell) math is float32 exactly in the operation order written in ndt_point_cell() below
//    (left-to-right accumulation, no FMA); exp/sin/cos of float arguments are evaluated as
//    (float)f((double)x), i.e. the correctly-rounded float result, so that the CUDA path can be bit-compatible;
//  * per-point results are accumulated in float64 and summed SERIALLY in point-index order (ndt_omp does this);
//  * Euler angles of the guess follow Eigen 3.3 `eulerAngles(0,1,2)` (first angle in [0,pi]);
//  * More-Thuente: `mt_interval_flag` selects the polarity of ndt_omp's `interval_converged` initialiser.
#include "oracle.h"
#include "linalg.hpp"
#include <omp.h>
#include <vector>
#include <unordered_map>
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>

using namespace orc;

static inline int nthreads(int t) { return t > 0 ? t : omp_get_max_threads(); }

// ================================================================= pcl::VoxelGrid (A.5)
extern "C" int orc_voxelgrid(const float* in, size_t n, size_t stride, float leaf, float* out_xyzi, int32_t* out_keys,
                             int32_t* out_counts, size_t* n_out) {
  const bool has_i = stride >= 5;
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (size_t i = 0; i < n; i++) {
    const float* p = in + i * stride;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
    for (int d = 0; d < 3; d++) { mn[d] = std::min(mn[d], p[d]); mx[d] = std::max(mx[d], p[d]); }
  }
  *n_out = 0;
  if (n == 0 || !(mn[0] <= mx[0])) return 0;
  const float inv = 1.0f / leaf;
  int64_t dx = (int64_t)((mx[0] - mn[0]) * inv) + 1, dy = (int64_t)((mx[1] - mn[1]) * inv) + 1, dz = (int64_t)((mx[2] - mn[2]) * inv) + 1;
  // PCL forms dx * dy * dz in int64, which overflows (undefined) once the extents pass ~2^21 leaves per axis and can then let a
  // far too fine grid through; the volume is checked factor by factor instead (as the engine does), without overflow
  const bool too_small = dx > INT_MAX || dy > INT_MAX || dz > INT_MAX || dx * dy > INT_MAX || dx * dy * dz > INT_MAX;
  if (too_small) {  // "Leaf size is too small for the input dataset" -> output = input
    for (size_t i = 0; i < n; i++) {
      const float* p = in + i * stride;
      out_xyzi[i * 4 + 0] = p[0]; out_xyzi[i * 4 + 1] = p[1]; out_xyzi[i * 4 + 2] = p[2]; out_xyzi[i * 4 + 3] = has_i ? p[4] : 0.f;
      if (out_keys) out_keys[i] = -1;
      if (out_counts) out_counts[i] = 1;
    }
    *n_out = n;
    return 1;
  }
  int minb[3], maxb[3], divb[3];
  for (int d = 0; d < 3; d++) {
    minb[d] = (int)std::floor(mn[d] * inv);
    maxb[d] = (int)std::floor(mx[d] * inv);
    divb[d] = maxb[d] - minb[d] + 1;
  }
  const int mul[3] = {1, divb[0], divb[0] * divb[1]};
  std::vector<std::pair<int32_t, int32_t>> ki;
  ki.reserve(n);
  for (size_t i = 0; i < n; i++) {
    const float* p = in + i * stride;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
    int i0 = (int)(std::floor(p[0] * inv) - (float)minb[0]);
    int i1 = (int)(std::floor(p[1] * inv) - (float)minb[1]);
    int i2 = (int)(std::floor(p[2] * inv) - (float)minb[2]);
    ki.emplace_back(i0 * mul[0] + i1 * mul[1] + i2 * mul[2], (int32_t)i);
  }
  std::sort(ki.begin(), ki.end());  // (key, point index): the oracle pins within-voxel order to ascending index
  size_t o = 0, a = 0;
  while (a < ki.size()) {
    size_t b = a;
    float s[4] = {0, 0, 0, 0};
    while (b < ki.size() && ki[b].first == ki[a].first) {
      const float* p = in + (size_t)ki[b].second * stride;
      s[0] += p[0]; s[1] += p[1]; s[2] += p[2]; s[3] += has_i ? p[4] : 0.f;
      b++;
    }
    float cnt = (float)(b - a);
    for (int d = 0; d < 4; d++) out_xyzi[o * 4 + d] = s[d] / cnt;
    if (out_keys) out_keys[o] = ki[a].first;
    if (out_counts) out_counts[o] = (int32_t)(b - a);
    o++;
    a = b;
  }
  *n_out = o;
  return 0;
}

// ================================================================= VoxelGridCovariance (A.3)
struct Leaf {
  int64_t key;
  int nr_points;
  double mean[3];
  double cov[9];
  double icov[9];
};

struct orc_ndt_map {
  float leaf, inv_leaf;
  int min_b[3], max_b[3], div_b[3];
  int64_t mul[3];
  std::vector<Leaf> leaves;                 // ascending key
  std::unordered_map<int64_t, int> index;   // key -> leaf slot
  bool empty = true;
};

extern "C" int orc_ndt_voxel_gaussian(int n, const double* S, const double* S2, double* mean, double* cov, double* icov) {
  const double nn = (double)n;
  for (int d = 0; d < 3; d++) mean[d] = S[d] / nn;
  for (int a = 0; a < 9; a++) { cov[a] = 0.0; icov[a] = 0.0; }
  if (n < 6) return n;
  // cov = (S2 - 2*(sum*mean^T))/n + mean*mean^T ; cov *= (n-1)/n
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) cov[a * 3 + b] = (S2[a * 3 + b] - 2 * (S[a] * mean[b])) / nn + mean[a] * mean[b];
  double f = (nn - 1.0) / nn;
  for (int a = 0; a < 9; a++) cov[a] *= f;
  double w[3], V[9];
  sym_eigen<3>(cov, w, V);
  if (w[0] < 0 || w[1] < 0 || w[2] <= 0) return -1;
  double minv = 0.01 * w[2];
  if (w[0] < minv) {
    w[0] = minv;
    if (w[1] < minv) w[1] = minv;
    double Vi[9], VD[9];
    inv3(V, Vi);
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) VD[a * 3 + b] = V[a * 3 + b] * w[b];
    mul3(VD, Vi, cov);
  }
  inv3(cov, icov);
  double mxv = -INFINITY, mnv = INFINITY;
  for (int a = 0; a < 9; a++) { mxv = std::max(mxv, icov[a]); mnv = std::min(mnv, icov[a]); }
  if (mxv == INFINITY || mnv == -INFINITY || mxv != mxv || mnv != mnv) return -1;
  return n;
}

extern "C" orc_ndt_map* orc_ndt_build(const float* tgt, size_t m, size_t stride, float resolution) {
  orc_ndt_map* M = new orc_ndt_map();
  M->leaf = resolution;
  M->inv_leaf = 1.0f / resolution;
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (size_t i = 0; i < m; i++) {
    const float* p = tgt + i * stride;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
    for (int d = 0; d < 3; d++) { mn[d] = std::min(mn[d], p[d]); mx[d] = std::max(mx[d], p[d]); }
  }
  if (m == 0 || !(mn[0] <= mx[0])) return M;
  for (int d = 0; d < 3; d++) {
    M->min_b[d] = (int)std::floor(mn[d] * M->inv_leaf);
    M->max_b[d] = (int)std::floor(mx[d] * M->inv_leaf);
    M->div_b[d] = M->max_b[d] - M->min_b[d] + 1;
  }
  M->mul[0] = 1; M->mul[1] = M->div_b[0]; M->mul[2] = (int64_t)M->div_b[0] * M->div_b[1];
  M->empty = false;

  struct Acc { double s[3]; double c[9]; int n; };
  std::unordered_map<int64_t, Acc> acc;
  acc.reserve(m / 4 + 16);
  for (size_t i = 0; i < m; i++) {
    const float* p = tgt + i * stride;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
    int64_t i0 = (int64_t)(std::floor(p[0] * M->inv_leaf) - (float)M->min_b[0]);
    int64_t i1 = (int64_t)(std::floor(p[1] * M->inv_leaf) - (float)M->min_b[1]);
    int64_t i2 = (int64_t)(std::floor(p[2] * M->inv_leaf) - (float)M->min_b[2]);
    int64_t key = i0 * M->mul[0] + i1 * M->mul[1] + i2 * M->mul[2];
    auto it = acc.find(key);
    if (it == acc.end()) { Acc z; std::memset(&z, 0, sizeof(z)); it = acc.emplace(key, z).first; }
    Acc& A = it->second;
    double q[3] = {(double)p[0], (double)p[1], (double)p[2]};
    for (int a = 0; a < 3; a++) {
      A.s[a] += q[a];
      for (int b = 0; b < 3; b++) A.c[a * 3 + b] += q[a] * q[b];
    }
    A.n++;
  }
  M->leaves.reserve(acc.size());
  for (auto& kv : acc) {
    Leaf L;
    std::memset(&L, 0, sizeof(L));
    L.key = kv.first;
    const Acc& A = kv.second;
    L.nr_points = orc_ndt_voxel_gaussian(A.n, A.s, A.c, L.mean, L.cov, L.icov);
    M->leaves.push_back(L);
  }
  std::sort(M->leaves.begin(), M->leaves.end(), [](const Leaf& a, const Leaf& b) { return a.key < b.key; });
  M->index.reserve(M->leaves.size() * 2);
  for (size_t i = 0; i < M->leaves.size(); i++) M->index[M->leaves[i].key] = (int)i;
  return M;
}

extern "C" void orc_ndt_free(orc_ndt_map* M) { delete M; }

extern "C" size_t orc_ndt_dump(const orc_ndt_map* M, int64_t* keys, int32_t* npts, double* mean, double* cov, double* icov,
                               int32_t* min_b, int32_t* div_b) {
  size_t V = M->leaves.size();
  for (size_t i = 0; i < V; i++) {
    const Leaf& L = M->leaves[i];
    if (keys) keys[i] = L.key;
    if (npts) npts[i] = L.nr_points;
    if (mean) std::memcpy(mean + i * 3, L.mean, sizeof(L.mean));
    if (cov) std::memcpy(cov + i * 9, L.cov, sizeof(L.cov));
    if (icov) std::memcpy(icov + i * 9, L.icov, sizeof(L.icov));
  }
  if (min_b) for (int d = 0; d < 3; d++) min_b[d] = M->empty ? 0 : M->min_b[d];
  if (div_b) for (int d = 0; d < 3; d++) div_b[d] = M->empty ? 0 : M->div_b[d];
  return V;
}

// ================================================================= NDT derivatives (A.2)
struct NdtConsts {
  double d1, d2;      // gauss_d1_, gauss_d2_
  float jang[8][3];   // j_ang rows (float)
  float hang[15][3];  // h_ang rows (float)
  double jang_d[8][3], hang_d[15][3];
};

static void gauss_consts(const orc_ndt_config* c, NdtConsts& K) {
  double gauss_c1 = 10 * (1 - c->outlier_ratio);
  double gauss_c2 = c->outlier_ratio / std::pow(c->resolution, 3);
  double gauss_d3 = -std::log(gauss_c2);
  K.d1 = -std::log(gauss_c1 + gauss_c2) - gauss_d3;
  K.d2 = -2 * std::log((-std::log(gauss_c1 * std::exp(-0.5) + gauss_c2) - gauss_d3) / K.d1);
}

static void angle_derivs(const double* p, NdtConsts& K) {
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
      {(-cx * sz - sx * sy * cz), (-cx * cz + sx * sy * sz), sx * cy},   // a2
      {(-sx * sz + cx * sy * cz), (-cx * sy * sz - sx * cz), (-cx * cy)},  // a3
      {(cx * cy * cz), (-cx * cy * sz), (cx * sy)},                        // b2
      {(sx * cy * cz), (-sx * cy * sz), (sx * sy)},                        // b3
      {(-sx * cz - cx * sy * sz), (sx * sz - cx * sy * cz), 0},            // c2
      {(cx * cz - sx * sy * sz), (-sx * sy * cz - cx * sz), 0},            // c3
      {(-cy * cz), (cy * sz), (sy)},                                       // d1
      {(-sx * sy * cz), (sx * sy * sz), (sx * cy)},                        // d2
      {(cx * sy * cz), (-cx * sy * sz), (-cx * cy)},                       // d3
      {(sy * sz), (sy * cz), 0},                                           // e1
      {(-sx * cy * sz), (-sx * cy * cz), 0},                               // e2
      {(cx * cy * sz), (cx * cy * cz), 0},                                 // e3
      {(-cy * cz), (cy * sz), 0},                                          // f1
      {(-cx * sz - sx * sy * cz), (-cx * cz + sx * sy * sz), 0},           // f2
      {(-sx * sz + cx * sy * cz), (-cx * sy * sz - sx * cz), 0}};          // f3
  for (int r = 0; r < 8; r++)
    for (int c = 0; c < 3; c++) { K.jang_d[r][c] = J[r][c]; K.jang[r][c] = (float)J[r][c]; }
  for (int r = 0; r < 15; r++)
    for (int c = 0; c < 3; c++) { K.hang_d[r][c] = Hh[r][c]; K.hang[r][c] = (float)Hh[r][c]; }
}

static inline float dot3f(const float* a, float x, float y, float z) {
  float s = a[0] * x;
  float t = a[1] * y;
  s = s + t;
  t = a[2] * z;
  return s + t;
}

// float32 per-(point,cell) update == ndt_omp updateDerivatives (float path). Returns score_inc.
static inline double ndt_point_cell(const NdtConsts& K, const float J[3][6], const float PH[3][3][3] /*[i-3][j-3][r]*/,
                                    const float q[3], const float C[9], double* g, double* H) {
  const float d2f = (float)K.d2;
  // qC = q^T * C
  float qC[3];
  for (int j = 0; j < 3; j++) {
    float s = q[0] * C[0 * 3 + j];
    float t = q[1] * C[1 * 3 + j];
    s = s + t;
    t = q[2] * C[2 * 3 + j];
    qC[j] = s + t;
  }
  float s = q[0] * qC[0];
  float t = q[1] * qC[1];
  s = s + t;
  t = q[2] * qC[2];
  float qCq = s + t;
  float arg = ((-d2f) * qCq) * 0.5f;
  float e = (float)std::exp((double)arg);
  float score_inc = (float)(-K.d1 * (double)e);
  e = d2f * e;
  if (e > 1 || e < 0 || e != e) return 0.0;
  e = (float)((double)e * K.d1);
  // CJ = C * J  (3x6)
  float CJ[3][6];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 6; c++) {
      float a = C[r * 3 + 0] * J[0][c];
      float b = C[r * 3 + 1] * J[1][c];
      a = a + b;
      b = C[r * 3 + 2] * J[2][c];
      CJ[r][c] = a + b;
    }
  float gq[6];  // q^T * CJ
  for (int c = 0; c < 6; c++) {
    float a = q[0] * CJ[0][c];
    float b = q[1] * CJ[1][c];
    a = a + b;
    b = q[2] * CJ[2][c];
    gq[c] = a + b;
  }
  for (int c = 0; c < 6; c++) g[c] += (double)(e * gq[c]);
  if (H) {
    float P[6][6];  // J^T * CJ
    for (int a = 0; a < 6; a++)
      for (int b = 0; b < 6; b++) {
        float u = J[0][a] * CJ[0][b];
        float v = J[1][a] * CJ[1][b];
        u = u + v;
        v = J[2][a] * CJ[2][b];
        P[a][b] = u + v;
      }
    for (int i = 0; i < 6; i++) {
      for (int j = 0; j < 6; j++) {
        float xh = 0.f;
        if (i >= 3 && j >= 3) {
          const float* v = PH[i - 3][j - 3];
          float a = qC[0] * v[0];
          float b = qC[1] * v[1];
          a = a + b;
          b = qC[2] * v[2];
          xh = a + b;
        }
        float u = (-d2f) * gq[i];
        u = u * gq[j];
        u = u + xh;
        u = u + P[j][i];
        H[i * 6 + j] += (double)(e * u);
      }
    }
  }
  return (double)score_inc;
}

static const int kOff7[7][3] = {{0, 0, 0}, {1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};

// getNeighborhoodAtPoint's base cell, floor(xt / leaf) per axis.  ndt_omp casts without a guard, which is undefined for a
// non-finite point or a cell beyond int range; the oracle (like the engine) drops such a point: it contributes no pair.
static inline bool base_cell(const orc_ndt_map* M, const float* xt, int* ijk) {
  for (int d = 0; d < 3; d++) {
    if (!std::isfinite(xt[d])) return false;
    const float f = std::floor(xt[d] / M->leaf);
    if (!(std::fabs(f) < 1.0e9f)) return false;
    ijk[d] = (int)f;
  }
  return true;
}

// Row-major float 4x4 from p = (t, euler xyz): Translation * AngleAxis(x) * AngleAxis(y) * AngleAxis(z) in float32
static void pose_to_matrix_f32(const double* p, float* T) {
  float ang[3] = {(float)p[3], (float)p[4], (float)p[5]};
  float R[3][9];
  for (int a = 0; a < 3; a++) {
    float s = (float)std::sin((double)ang[a]);
    float c = (float)std::cos((double)ang[a]);
    float omc = 1.0f - c;
    float diag_axis = omc + c;  // (1-c)*1*1 + c
    float m[9] = {c, 0, 0, 0, c, 0, 0, 0, c};
    // Eigen AngleAxis::toRotationMatrix with a unit basis axis: off-axis diagonal = 0 + c, axis diagonal = (1-c) + c
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

static inline void xform_f32(const float* Tf, const float* p, float* o) {
  for (int r = 0; r < 3; r++) {
    float a = Tf[r * 4 + 0] * p[0];
    float b = Tf[r * 4 + 1] * p[1];
    float c = Tf[r * 4 + 2] * p[2];
    float s = a + b;
    s = s + c;
    o[r] = s + Tf[r * 4 + 3];
  }
}

// computeDerivatives over a transformed cloud (trans = T*src in float32)
static double derivatives(const orc_ndt_map* M, const float* src, size_t n, size_t stride, const float* Tf, const orc_ndt_config* cfg,
                          const NdtConsts& K, double* g_out, double* H_out, bool compute_hessian, uint64_t* n_pairs, uint8_t* cells_out) {
  std::vector<double> sc(n), gr(n * 6), he(compute_hessian ? n * 36 : 0);
  std::vector<uint8_t> masks(n);
  const int ncell = cfg->search_method == 1 ? 1 : 7;
#pragma omp parallel for num_threads(nthreads(cfg->num_threads)) schedule(guided, 8)
  for (long i = 0; i < (long)n; i++) {
    const float* x = src + (size_t)i * stride;
    float xt[3];
    xform_f32(Tf, x, xt);
    double score_pt = 0, g[6] = {0}, H[36] = {0};
    uint8_t mask = 0;
    bool have_pd = false;
    float J[3][6], PH[3][3][3];
    int ijk[3];
    if (!M->empty && base_cell(M, xt, ijk)) {
      for (int c = 0; c < ncell; c++) {
        int cc[3] = {ijk[0] + kOff7[c][0], ijk[1] + kOff7[c][1], ijk[2] + kOff7[c][2]};
        bool inb = true;
        for (int d = 0; d < 3; d++) inb &= (cc[d] >= M->min_b[d] && cc[d] <= M->max_b[d]);
        if (!inb) continue;
        int64_t key = (int64_t)(cc[0] - M->min_b[0]) * M->mul[0] + (int64_t)(cc[1] - M->min_b[1]) * M->mul[1] + (int64_t)(cc[2] - M->min_b[2]) * M->mul[2];
        auto it = M->index.find(key);
        if (it == M->index.end()) continue;
        const Leaf& L = M->leaves[it->second];
        if (L.nr_points < 6) continue;
        mask |= (uint8_t)(1u << c);
        if (!have_pd) {  // computePointDerivatives(x): depends on the ORIGINAL point only
          for (int r = 0; r < 3; r++)
            for (int cI = 0; cI < 6; cI++) J[r][cI] = (r == cI) ? 1.f : 0.f;
          float xj[8];
          for (int r = 0; r < 8; r++) xj[r] = dot3f(K.jang[r], x[0], x[1], x[2]);
          J[1][3] = xj[0]; J[2][3] = xj[1]; J[0][4] = xj[2]; J[1][4] = xj[3]; J[2][4] = xj[4]; J[0][5] = xj[5]; J[1][5] = xj[6]; J[2][5] = xj[7];
          float xh[15];
          for (int r = 0; r < 15; r++) xh[r] = dot3f(K.hang[r], x[0], x[1], x[2]);
          const float a[3] = {0, xh[0], xh[1]}, b[3] = {0, xh[2], xh[3]}, cV[3] = {0, xh[4], xh[5]};
          const float dV[3] = {xh[6], xh[7], xh[8]}, eV[3] = {xh[9], xh[10], xh[11]}, fV[3] = {xh[12], xh[13], xh[14]};
          const float* tab[3][3] = {{a, b, cV}, {b, dV, eV}, {cV, eV, fV}};
          for (int u = 0; u < 3; u++)
            for (int v = 0; v < 3; v++)
              for (int r = 0; r < 3; r++) PH[u][v][r] = tab[u][v][r];
          have_pd = true;
        }
        float q[3], C[9];
        for (int d = 0; d < 3; d++) q[d] = (float)((double)xt[d] - L.mean[d]);
        for (int d = 0; d < 9; d++) C[d] = (float)L.icov[d];
        score_pt += ndt_point_cell(K, J, PH, q, C, g, compute_hessian ? H : nullptr);
      }
    }
    sc[i] = score_pt;
    std::memcpy(&gr[(size_t)i * 6], g, sizeof(g));
    if (compute_hessian) std::memcpy(&he[(size_t)i * 36], H, sizeof(H));
    masks[i] = mask;
  }
  double score = 0;
  for (int k = 0; k < 6; k++) g_out[k] = 0;
  if (compute_hessian) for (int k = 0; k < 36; k++) H_out[k] = 0;
  uint64_t np = 0;
  for (size_t i = 0; i < n; i++) {  // "invariant against the summing up order": serial, index order
    score += sc[i];
    for (int k = 0; k < 6; k++) g_out[k] += gr[i * 6 + k];
    if (compute_hessian) for (int k = 0; k < 36; k++) H_out[k] += he[i * 36 + k];
    np += (uint64_t)__builtin_popcount(masks[i]);
  }
  if (n_pairs) *n_pairs = np;
  if (cells_out) std::memcpy(cells_out, masks.data(), n);
  return score;
}

// ndt_omp computeHessian/updateHessian (float64 path; only reached when the More-Thuente loop ran)
static void hessian_only(const orc_ndt_map* M, const float* src, size_t n, size_t stride, const float* Tf, const orc_ndt_config* cfg,
                         const NdtConsts& K, double* H_out) {
  const int ncell = cfg->search_method == 1 ? 1 : 7;
  std::vector<double> he(n * 36, 0.0);
#pragma omp parallel for num_threads(nthreads(cfg->num_threads)) schedule(guided, 8)
  for (long i = 0; i < (long)n; i++) {
    const float* xf = src + (size_t)i * stride;
    float xt[3];
    xform_f32(Tf, xf, xt);
    if (M->empty) continue;
    double x[3] = {(double)xf[0], (double)xf[1], (double)xf[2]};
    double J[3][6] = {{1, 0, 0, 0, 0, 0}, {0, 1, 0, 0, 0, 0}, {0, 0, 1, 0, 0, 0}};
    auto dj = [&](int r) { return x[0] * K.jang_d[r][0] + x[1] * K.jang_d[r][1] + x[2] * K.jang_d[r][2]; };
    auto dh = [&](int r) { return x[0] * K.hang_d[r][0] + x[1] * K.hang_d[r][1] + x[2] * K.hang_d[r][2]; };
    J[1][3] = dj(0); J[2][3] = dj(1); J[0][4] = dj(2); J[1][4] = dj(3); J[2][4] = dj(4); J[0][5] = dj(5); J[1][5] = dj(6); J[2][5] = dj(7);
    const double a[3] = {0, dh(0), dh(1)}, b[3] = {0, dh(2), dh(3)}, cV[3] = {0, dh(4), dh(5)};
    const double dV[3] = {dh(6), dh(7), dh(8)}, eV[3] = {dh(9), dh(10), dh(11)}, fV[3] = {dh(12), dh(13), dh(14)};
    const double* tab[3][3] = {{a, b, cV}, {b, dV, eV}, {cV, eV, fV}};
    double* H = &he[(size_t)i * 36];
    int ijk[3];
    if (!base_cell(M, xt, ijk)) continue;
    for (int c = 0; c < ncell; c++) {
      int cc[3] = {ijk[0] + kOff7[c][0], ijk[1] + kOff7[c][1], ijk[2] + kOff7[c][2]};
      bool inb = true;
      for (int d = 0; d < 3; d++) inb &= (cc[d] >= M->min_b[d] && cc[d] <= M->max_b[d]);
      if (!inb) continue;
      int64_t key = (int64_t)(cc[0] - M->min_b[0]) * M->mul[0] + (int64_t)(cc[1] - M->min_b[1]) * M->mul[1] + (int64_t)(cc[2] - M->min_b[2]) * M->mul[2];
      auto it = M->index.find(key);
      if (it == M->index.end()) continue;
      const Leaf& L = M->leaves[it->second];
      if (L.nr_points < 6) continue;
      double q[3];
      for (int d = 0; d < 3; d++) q[d] = (double)xt[d] - L.mean[d];
      const double* C = L.icov;
      double Cq[3];
      for (int r = 0; r < 3; r++) Cq[r] = C[r * 3 + 0] * q[0] + C[r * 3 + 1] * q[1] + C[r * 3 + 2] * q[2];
      double e = K.d2 * std::exp(-K.d2 * (q[0] * Cq[0] + q[1] * Cq[1] + q[2] * Cq[2]) / 2);
      if (e > 1 || e < 0 || e != e) continue;
      e *= K.d1;
      double CJ[3][6], qCJ[6];
      for (int r = 0; r < 3; r++)
        for (int k = 0; k < 6; k++) CJ[r][k] = C[r * 3 + 0] * J[0][k] + C[r * 3 + 1] * J[1][k] + C[r * 3 + 2] * J[2][k];
      for (int k = 0; k < 6; k++) qCJ[k] = q[0] * CJ[0][k] + q[1] * CJ[1][k] + q[2] * CJ[2][k];
      for (int ii = 0; ii < 6; ii++)
        for (int jj = 0; jj < 6; jj++) {
          double xh = 0;
          if (ii >= 3 && jj >= 3) {
            const double* v = tab[ii - 3][jj - 3];
            double Cv[3];
            for (int r = 0; r < 3; r++) Cv[r] = C[r * 3 + 0] * v[0] + C[r * 3 + 1] * v[1] + C[r * 3 + 2] * v[2];
            xh = q[0] * Cv[0] + q[1] * Cv[1] + q[2] * Cv[2];
          }
          double jcj = J[0][jj] * CJ[0][ii] + J[1][jj] * CJ[1][ii] + J[2][jj] * CJ[2][ii];
          H[ii * 6 + jj] += e * (-K.d2 * qCJ[ii] * qCJ[jj] + xh + jcj);
        }
    }
  }
  for (int k = 0; k < 36; k++) H_out[k] = 0;
  for (size_t i = 0; i < n; i++)
    for (int k = 0; k < 36; k++) H_out[k] += he[i * 36 + k];
}

extern "C" double orc_ndt_derivatives(const orc_ndt_map* M, const float* src, size_t n, size_t stride, const orc_ndt_config* cfg,
                                      const double* p, double* g, double* H, uint64_t* n_pairs, uint8_t* per_point_cells) {
  NdtConsts K;
  gauss_consts(cfg, K);
  angle_derivs(p, K);
  float Tf[16];
  pose_to_matrix_f32(p, Tf);
  return derivatives(M, src, n, stride, Tf, cfg, K, g, H, true, n_pairs, per_point_cells);
}

extern "C" void orc_ndt_hessian_at(const orc_ndt_map* M, const float* src, size_t n, size_t stride, const orc_ndt_config* cfg,
                                   const double* p, double* H) {
  NdtConsts K;
  gauss_consts(cfg, K);
  angle_derivs(p, K);
  float Tf[16];
  pose_to_matrix_f32(p, Tf);
  hessian_only(M, src, n, stride, Tf, cfg, K, H);
}

// ---- More-Thuente helpers (PCL ndt.hpp; SURVEY A.2)
static double psiMT(double a, double f_a, double f_0, double g_0, double mu) { return f_a - f_0 - mu * g_0 * a; }
static double dpsiMT(double g_a, double g_0, double mu) { return g_a - mu * g_0; }

static double trialValueSelectionMT(double a_l, double f_l, double g_l, double a_u, double f_u, double g_u, double a_t, double f_t, double g_t) {
  if (f_t > f_l) {
    double z = 3 * (f_t - f_l) / (a_t - a_l) - g_t - g_l;
    double w = std::sqrt(z * z - g_t * g_l);
    double a_c = a_l + (a_t - a_l) * (w - g_l - z) / (g_t - g_l + 2 * w);
    double a_q = a_l - 0.5 * (a_l - a_t) * g_l / (g_l - (f_l - f_t) / (a_l - a_t));
    if (std::fabs(a_c - a_l) < std::fabs(a_q - a_l)) return a_c;
    return 0.5 * (a_q + a_c);
  } else if (g_t * g_l < 0) {
    double z = 3 * (f_t - f_l) / (a_t - a_l) - g_t - g_l;
    double w = std::sqrt(z * z - g_t * g_l);
    double a_c = a_l + (a_t - a_l) * (w - g_l - z) / (g_t - g_l + 2 * w);
    double a_s = a_l - (a_l - a_t) / (g_l - g_t) * g_l;
    if (std::fabs(a_c - a_t) >= std::fabs(a_s - a_t)) return a_c;
    return a_s;
  } else if (std::fabs(g_t) <= std::fabs(g_l)) {
    double z = 3 * (f_t - f_l) / (a_t - a_l) - g_t - g_l;
    double w = std::sqrt(z * z - g_t * g_l);
    double a_c = a_l + (a_t - a_l) * (w - g_l - z) / (g_t - g_l + 2 * w);
    double a_s = a_l - (a_l - a_t) / (g_l - g_t) * g_l;
    double a_t_next = (std::fabs(a_c - a_t) < std::fabs(a_s - a_t)) ? a_c : a_s;
    if (a_t > a_l) return std::min(a_t + 0.66 * (a_u - a_t), a_t_next);
    return std::max(a_t + 0.66 * (a_u - a_t), a_t_next);
  } else {
    double z = 3 * (f_t - f_u) / (a_t - a_u) - g_t - g_u;
    double w = std::sqrt(z * z - g_t * g_u);
    return a_u + (a_t - a_u) * (w - g_u - z) / (g_t - g_u + 2 * w);
  }
}

static bool updateIntervalMT(double& a_l, double& f_l, double& g_l, double& a_u, double& f_u, double& g_u, double a_t, double f_t, double g_t) {
  if (f_t > f_l) { a_u = a_t; f_u = f_t; g_u = g_t; return false; }
  else if (g_t * (a_l - a_t) > 0) { a_l = a_t; f_l = f_t; g_l = g_t; return false; }
  else if (g_t * (a_l - a_t) < 0) { a_u = a_l; f_u = f_l; g_u = g_l; a_l = a_t; f_l = f_t; g_l = g_t; return false; }
  return true;
}

// Eigen 3.3 Matrix3f::eulerAngles(0,1,2) in float32 (first angle in [0, pi])
static void euler_xyz_eigen33(const float* T /*row-major 4x4*/, float* out) {
  auto m = [&](int r, int c) { return T[r * 4 + c]; };
  const int i = 0, j = 1, k = 2;  // odd = 0
  float res0 = std::atan2(m(j, k), m(k, k));
  float c2 = std::sqrt(m(i, i) * m(i, i) + m(i, j) * m(i, j));
  float res1;
  if (res0 > 0.f) {
    if (res0 > 0.f) res0 -= (float)M_PI; else res0 += (float)M_PI;
    res1 = std::atan2(-m(i, k), -c2);
  } else {
    res1 = std::atan2(-m(i, k), c2);
  }
  float s1 = std::sin(res0), c1 = std::cos(res0);
  float res2 = std::atan2(s1 * m(k, i) - c1 * m(j, i), c1 * m(j, j) - s1 * m(k, j));
  out[0] = -res0; out[1] = -res1; out[2] = -res2;
}

extern "C" void orc_ndt_align(const orc_ndt_map* M, const float* src, size_t n, size_t stride, const orc_ndt_config* cfg,
                              const float* guess, orc_ndt_result* res, double* trace_p) {
  std::memset(res, 0, sizeof(*res));
  float Tfinal[16];
  for (int i = 0; i < 16; i++) Tfinal[i] = (i % 5 == 0) ? 1.f : 0.f;
  for (int i = 0; i < 16; i++) res->T[i] = Tfinal[i];
  if (n == 0 || M->empty) return;
  NdtConsts K;
  gauss_consts(cfg, K);
  bool guess_is_identity = true;
  for (int i = 0; i < 16; i++) guess_is_identity &= (guess[i] == ((i % 5 == 0) ? 1.f : 0.f));
  if (!guess_is_identity) std::memcpy(Tfinal, guess, sizeof(Tfinal));
  double p[6];
  {
    float e[3];
    euler_xyz_eigen33(Tfinal, e);
    p[0] = Tfinal[3]; p[1] = Tfinal[7]; p[2] = Tfinal[11];
    p[3] = e[0]; p[4] = e[1]; p[5] = e[2];
  }
  if (trace_p) std::memcpy(trace_p, p, sizeof(p));
  double g[6], H[36];
  uint64_t passes = 0;
  angle_derivs(p, K);
  // first pass uses the cloud transformed by the GUESS matrix itself (not the re-composed pose)
  double score = derivatives(M, src, n, stride, Tfinal, cfg, K, g, H, true, nullptr, nullptr);
  passes++;
  int nr_iterations = 0;
  bool converged = false;
  const int max_it = cfg->max_iterations;
  while (!converged) {
    double ng[6], dp[6];
    for (int i = 0; i < 6; i++) ng[i] = -g[i];
    svd6_solve_sym(H, ng, dp);
    double nrm = 0;
    for (int i = 0; i < 6; i++) nrm += dp[i] * dp[i];
    nrm = std::sqrt(nrm);
    if (nrm == 0 || nrm != nrm) {
      converged = (nrm == nrm);
      break;
    }
    for (int i = 0; i < 6; i++) dp[i] /= nrm;
    // ---- computeStepLengthMT(p, dp, nrm, step_size, eps/2, ...)
    double step_max = cfg->step_size, step_min = cfg->transformation_epsilon / 2;
    double phi_0 = -score;
    double d_phi_0 = 0;
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
      bool interval_converged = cfg->mt_interval_flag ? ((step_max - step_min) < 0) : ((step_max - step_min) > 0);
      bool open_interval = true;
      int step_iterations = 0;
      a_t = nrm;
      a_t = std::min(a_t, step_max);
      a_t = std::max(a_t, step_min);
      double x_t[6];
      for (int i = 0; i < 6; i++) x_t[i] = p[i] + dp[i] * a_t;
      pose_to_matrix_f32(x_t, Tfinal);
      angle_derivs(x_t, K);
      score = derivatives(M, src, n, stride, Tfinal, cfg, K, g, H, true, nullptr, nullptr);
      passes++;
      double phi_t = -score, d_phi_t = 0;
      for (int i = 0; i < 6; i++) d_phi_t += g[i] * dp[i];
      d_phi_t = -d_phi_t;
      double psi_t = psiMT(a_t, phi_t, phi_0, d_phi_0, mu), d_psi_t = dpsiMT(d_phi_t, d_phi_0, mu);
      while (!interval_converged && step_iterations < 10 && !(psi_t <= 0 && d_phi_t <= -nu * d_phi_0)) {
        if (open_interval) a_t = trialValueSelectionMT(a_l, f_l, g_l, a_u, f_u, g_u, a_t, psi_t, d_psi_t);
        else a_t = trialValueSelectionMT(a_l, f_l, g_l, a_u, f_u, g_u, a_t, phi_t, d_phi_t);
        a_t = std::min(a_t, step_max);
        a_t = std::max(a_t, step_min);
        for (int i = 0; i < 6; i++) x_t[i] = p[i] + dp[i] * a_t;
        pose_to_matrix_f32(x_t, Tfinal);
        angle_derivs(x_t, K);
        score = derivatives(M, src, n, stride, Tfinal, cfg, K, g, H, false, nullptr, nullptr);
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
        if (open_interval) interval_converged = updateIntervalMT(a_l, f_l, g_l, a_u, f_u, g_u, a_t, psi_t, d_psi_t);
        else interval_converged = updateIntervalMT(a_l, f_l, g_l, a_u, f_u, g_u, a_t, phi_t, d_phi_t);
        step_iterations++;
      }
      if (step_iterations) { hessian_only(M, src, n, stride, Tfinal, cfg, K, H); passes++; res->hessian_passes++; }
    }
    double delta_p_norm = a_t;
    for (int i = 0; i < 6; i++) { dp[i] *= delta_p_norm; p[i] += dp[i]; }
    if (trace_p && nr_iterations + 1 <= max_it + 3) std::memcpy(trace_p + (size_t)(nr_iterations + 1) * 6, p, sizeof(p));
    if (cfg->fixed_iterations > 0) {
      if (nr_iterations + 1 >= cfg->fixed_iterations) converged = true;
    } else if (nr_iterations > max_it || (nr_iterations && (std::fabs(delta_p_norm) < cfg->transformation_epsilon))) {
      converged = true;
    }
    nr_iterations++;
  }
  for (int i = 0; i < 16; i++) res->T[i] = Tfinal[i];
  res->converged = converged ? 1 : 0;
  res->iterations = nr_iterations;
  res->trans_probability = score / (double)n;
  for (int i = 0; i < 6; i++) res->p[i] = p[i];
  res->derivative_passes = passes;
}
