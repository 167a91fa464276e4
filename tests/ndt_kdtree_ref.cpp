/* tests/ndt_kdtree_ref.cpp — TEST INFRASTRUCTURE ONLY: the sequential CPU reference of pclomp::NormalDistributionsTransform with
 * reg_nn_search_method = KDTREE (registrations.cpp:112-113) that defines the parity of B2R_METHOD_NDT_KDTREE
 * (hdl_graph_slam_b200/csrc/ndt_kdtree.cuh).  Built by the tests with -O2 -fopenmp -ffp-contract=off (no FMA).
 *
 * It restates none of the rules the existing references state: it compiles oracle/ndt.cpp (ndt_omp) and tests/ndt_pcl_ref.cpp (pcl
 * NDT) unchanged into one library and joins them.  ndt_omp is not available here: every rule is UPSTREAM-RECALL or ENGINE.
 *   factory: NDT_OMP's resolution, transformation epsilon and maximum iterations; step size 0.1, outlier ratio 0.55; the search-method
 *     value is what selects this mode and is not otherwise read.                                                   UPSTREAM-RECALL
 *   target: the oracle's NDT_OMP voxel map unchanged (keys, moments, eigenvalue clamp, inverse, nr_points = -1 invalidation), and on
 *     top of it filter(true)'s centroid cloud exactly as ndt_pcl_ref.cpp builds it: ndt_omp's VoxelGridCovariance is a copy of
 *     PCL's.                                                                                                        UPSTREAM-RECALL
 *   neighbourhood: computeDerivatives and computeHessian both call target_cells_.radiusSearch(x_trans_pt, resolution_):
 *     ndt_pcl_ref.cpp's radius() (strict float32 d2 < (float)r^2, ascending (d2, centroid)), with no nr_points >= 6 check and no
 *     cell index (the oracle's drop of points beyond 1e9 cells does not apply); a non-finite point has no neighbours.
 *                                                                                                                   UPSTREAM-RECALL
 *   derivative pass: each (point, neighbour) is the oracle's own pass (oracle/ndt.cpp derivatives(): computePointDerivatives and the
 *     float32 ndt_point_cell) over a one-leaf map that holds the neighbour's Gaussian at the point's base cell; the per-point sums
 *     add the terms in neighbour order, the pass adds the points serially in index order, as the oracle does.     UPSTREAM-RECALL
 *   Hessian-only pass (after a line search that iterated): likewise the oracle's hessian_only() per (point, neighbour).
 *                                                                                                                   UPSTREAM-RECALL
 *   driver: orc_ndt_align (computeTransformation / computeStepLengthMT, mt_interval_flag, fixed_iterations) unchanged.  UPSTREAM-RECALL
 *   n_pairs: the number of (point, radius neighbour) pairs, as for pcl NDT.                                          ENGINE
 *
 * How the neighbourhood is switched without editing oracle/ndt.cpp: its driver and its two entry points call derivatives() and
 * hessian_only() with a non-const float* pose.  The hooks declared below, before the file is included, take the pose as float* and
 * are the better overloads for exactly those calls.  With no KDTREE entry point active on the thread (KdRule) they call the oracle's
 * own functions (const float* pose), so the oracle's entry points compiled into this library compute what they compute in liboracle.
 * Three names of ndt_pcl_ref.cpp that would clash with the oracle's (Leaf, psiMT, dpsiMT) are renamed while it is included.
 */
#include "../oracle/oracle.h"
#include <cstddef>
#include <cstdint>

struct NdtConsts;
static double derivatives(const orc_ndt_map* M, const float* src, size_t n, size_t stride, float* Tf, const orc_ndt_config* cfg, const NdtConsts& K,
                          double* g_out, double* H_out, bool compute_hessian, uint64_t* n_pairs, uint8_t* cells_out);
static void hessian_only(const orc_ndt_map* M, const float* src, size_t n, size_t stride, float* Tf, const orc_ndt_config* cfg, const NdtConsts& K,
                         double* H_out);

#include "../oracle/ndt.cpp"

#define Leaf PclLeaf
#define psiMT pcl_psiMT
#define dpsiMT pcl_dpsiMT
#include "ndt_pcl_ref.cpp"
#undef Leaf
#undef psiMT
#undef dpsiMT

#include <cfloat>

namespace {

thread_local const Map* kd_rule = nullptr;  // the centroid cloud of the KDTREE entry point running on this thread

struct KdRule {
  explicit KdRule(const Map* m) { kd_rule = m; }
  ~KdRule() { kd_rule = nullptr; }
};

// a map of one leaf at the base cell of the point it is placed for: the oracle's passes over it visit exactly that leaf.  The leaf
// size is the largest float, so every finite point has a base cell (|floor(x / leaf)| <= 1); the term never reads the leaf size.
struct OneLeaf {
  orc_ndt_map M;
  orc_ndt_config cfg;
  explicit OneLeaf(const orc_ndt_config* c) : cfg(*c) {
    cfg.search_method = 1;  // the base cell only
    cfg.num_threads = 1;
    M.leaf = FLT_MAX;
    M.inv_leaf = 1.0f / FLT_MAX;
    M.empty = false;
    for (int d = 0; d < 3; d++) M.div_b[d] = 1;
    M.mul[0] = 1; M.mul[1] = 1; M.mul[2] = 1;
    ::Leaf L;
    std::memset(&L, 0, sizeof(L));
    M.leaves.push_back(L);
    M.index[0] = 0;
  }
  // the neighbour L at the base cell of xt (the transformed point the pass computes from the same pose); false: no base cell
  bool place(const float* xt, const PclLeaf& L) {
    int ijk[3];
    if (!base_cell(&M, xt, ijk)) return false;
    for (int d = 0; d < 3; d++) { M.min_b[d] = ijk[d]; M.max_b[d] = ijk[d]; }
    ::Leaf& O = M.leaves[0];
    O.key = 0;
    O.nr_points = 6;  // KDTREE: a returned leaf is not checked for nr_points >= 6
    std::memcpy(O.mean, L.mean, sizeof(O.mean));
    std::memcpy(O.icov, L.icov, sizeof(O.icov));
    return true;
  }
};

}  // namespace

// computeDerivatives (the oracle's driver and orc_ndt_derivatives call it with a non-const pose)
static double derivatives(const orc_ndt_map* M, const float* src, size_t n, size_t stride, float* Tf, const orc_ndt_config* cfg, const NdtConsts& K,
                          double* g_out, double* H_out, bool compute_hessian, uint64_t* n_pairs, uint8_t* cells_out) {
  const Map* P = kd_rule;
  if (!P) return derivatives(M, src, n, stride, static_cast<const float*>(Tf), cfg, K, g_out, H_out, compute_hessian, n_pairs, cells_out);
  std::vector<double> sc(n, 0.0), gr(n * 6, 0.0), he(compute_hessian ? n * 36 : 0, 0.0);
  std::vector<uint32_t> np(n, 0);
  const float r2 = (float)(cfg->resolution * cfg->resolution);
#pragma omp parallel num_threads(nthreads(cfg->num_threads))
  {
    OneLeaf one(cfg);
    std::vector<std::pair<float, int>> nb;
#pragma omp for schedule(guided, 64)
    for (long i = 0; i < (long)n; i++) {
      const float* x = src + (size_t)i * stride;
      float xt[3];
      xform_f32(Tf, x, xt);
      radius(*P, xt, r2, nb);
      for (const auto& e : nb) {
        if (!one.place(xt, P->leaves[P->cent_leaf[e.second]])) continue;
        double g[6], H[36];
        sc[i] += derivatives(&one.M, x, 1, stride, static_cast<const float*>(Tf), &one.cfg, K, g, H, compute_hessian, nullptr, nullptr);
        for (int k = 0; k < 6; k++) gr[(size_t)i * 6 + k] += g[k];
        if (compute_hessian) for (int k = 0; k < 36; k++) he[(size_t)i * 36 + k] += H[k];
      }
      np[i] = (uint32_t)nb.size();
    }
  }
  double score = 0;
  for (int k = 0; k < 6; k++) g_out[k] = 0;
  if (compute_hessian) for (int k = 0; k < 36; k++) H_out[k] = 0;
  uint64_t pairs = 0;
  for (size_t i = 0; i < n; i++) {
    score += sc[i];
    for (int k = 0; k < 6; k++) g_out[k] += gr[i * 6 + k];
    if (compute_hessian) for (int k = 0; k < 36; k++) H_out[k] += he[i * 36 + k];
    pairs += np[i];
  }
  if (n_pairs) *n_pairs = pairs;
  if (cells_out) std::memset(cells_out, 0, n);  // no DIRECT7 offsets in this mode
  return score;
}

// computeHessian (the oracle's driver and orc_ndt_hessian_at call it with a non-const pose)
static void hessian_only(const orc_ndt_map* M, const float* src, size_t n, size_t stride, float* Tf, const orc_ndt_config* cfg, const NdtConsts& K,
                         double* H_out) {
  const Map* P = kd_rule;
  if (!P) return hessian_only(M, src, n, stride, static_cast<const float*>(Tf), cfg, K, H_out);
  std::vector<double> he(n * 36, 0.0);
  const float r2 = (float)(cfg->resolution * cfg->resolution);
#pragma omp parallel num_threads(nthreads(cfg->num_threads))
  {
    OneLeaf one(cfg);
    std::vector<std::pair<float, int>> nb;
#pragma omp for schedule(guided, 64)
    for (long i = 0; i < (long)n; i++) {
      const float* x = src + (size_t)i * stride;
      float xt[3];
      xform_f32(Tf, x, xt);
      radius(*P, xt, r2, nb);
      for (const auto& e : nb) {
        if (!one.place(xt, P->leaves[P->cent_leaf[e.second]])) continue;
        double H[36];
        hessian_only(&one.M, x, 1, stride, static_cast<const float*>(Tf), &one.cfg, K, H);
        for (int k = 0; k < 36; k++) he[(size_t)i * 36 + k] += H[k];
      }
    }
  }
  for (int k = 0; k < 36; k++) H_out[k] = 0;
  for (size_t i = 0; i < n; i++)
    for (int k = 0; k < 36; k++) H_out[k] += he[i * 36 + k];
}

namespace {
struct KdMap {
  orc_ndt_map* om = nullptr;  // the NDT_OMP voxel map
  Map* pm = nullptr;          // the same leaves with the searchable centroid cloud (ndt_pcl_ref.cpp)
};
}  // namespace

extern "C" {

void* ref_kd_map(const float* tgt, size_t m, size_t stride, float resolution) {
  KdMap* K = new KdMap();
  K->om = orc_ndt_build(tgt, m, stride, resolution);
  const size_t nv = orc_ndt_dump(K->om, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
  std::vector<int64_t> keys(nv + 1);
  std::vector<int32_t> npts(nv + 1);
  std::vector<double> mean(3 * nv + 3), icov(9 * nv + 9);
  int32_t min_b[3], div_b[3];
  orc_ndt_dump(K->om, keys.data(), npts.data(), mean.data(), nullptr, icov.data(), min_b, div_b);
  K->pm = static_cast<Map*>(ref_pcl_map(tgt, m, stride, resolution, nv, keys.data(), npts.data(), mean.data(), icov.data(), min_b, div_b));
  return K;
}

void ref_kd_free(void* k) {
  KdMap* K = static_cast<KdMap*>(k);
  orc_ndt_free(K->om);
  ref_pcl_free(K->pm);
  delete K;
}

// the two halves, for the oracle's orc_ndt_dump and ndt_pcl_ref's ref_pcl_centroids / ref_pcl_neighbors compiled into this library
const void* ref_kd_voxels(const void* k) { return static_cast<const KdMap*>(k)->om; }
const void* ref_kd_search(const void* k) { return static_cast<const KdMap*>(k)->pm; }

double ref_kd_derivatives(const void* k, const float* src, size_t n, size_t stride, const orc_ndt_config* cfg, const double* p, double* g,
                          double* H, uint64_t* n_pairs) {
  const KdMap* K = static_cast<const KdMap*>(k);
  KdRule on(K->pm);
  return orc_ndt_derivatives(K->om, src, n, stride, cfg, p, g, H, n_pairs, nullptr);
}

void ref_kd_hessian_at(const void* k, const float* src, size_t n, size_t stride, const orc_ndt_config* cfg, const double* p, double* H) {
  const KdMap* K = static_cast<const KdMap*>(k);
  KdRule on(K->pm);
  orc_ndt_hessian_at(K->om, src, n, stride, cfg, p, H);
}

void ref_kd_align(const void* k, const float* src, size_t n, size_t stride, const orc_ndt_config* cfg, const float* guess, orc_ndt_result* res) {
  const KdMap* K = static_cast<const KdMap*>(k);
  KdRule on(K->pm);
  orc_ndt_align(K->om, src, n, stride, cfg, guess, res, nullptr);
}

}  // extern "C"
