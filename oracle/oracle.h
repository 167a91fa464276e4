/* oracle/oracle.h — TEST INFRASTRUCTURE ONLY.
 *
 * C entry points of the CPU oracle: a from-scratch restatement (C++/OpenMP, built with
 * -O2 -ffp-contract=off, mirroring the reference's SSE4.2/no-FMA flags, /root/reference/CMakeLists.txt:10-11)
 * of the scan-matching arithmetic behind hdl_graph_slam's pcl::Registration handle:
 *   fast_gicp::FastGICP / LsqRegistration   (selected at src/hdl_graph_slam/registrations.cpp:27-36)
 *   pclomp::NormalDistributionsTransform    (registrations.cpp:101-120)
 *   pcl::VoxelGrid<PointXYZI>               (apps/prefiltering_nodelet.cpp:54-58,138-149)
 *   pcl::Registration::getFitnessScore / the inlier loop (apps/scan_matching_odometry_nodelet.cpp:298-335,
 *                                            src/hdl_graph_slam/information_matrix_calculator.cpp:49-80)
 * Those packages are un-vendored, unpinned third-party dependencies (docker/noetic/Dockerfile:14-15) that
 * cannot be built in this image, and the reference holds no tests or golden vectors:  **parity unpinned**.
 * The algorithm notes followed are SURVEY.md Appendix A.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load this
 * library.  The product (libb200reg.so) never links, loads or calls it.
 *
 * Conventions: points are float32 with x,y,z at offsets 0,4,8 of a record `stride` FLOATS long
 * (4 for packed float4, 8 for the 32-byte pcl::PointXYZI; intensity at float offset 4 of the latter).
 * All matrices crossing this API are ROW-MAJOR.
 */
#ifndef ORACLE_H
#define ORACLE_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

int orc_max_threads(void);

/* exact kNN (float32 d2, ties -> lowest index), result ascending by (d2, idx). */
void orc_knn(const float* pts, size_t n, size_t stride, const float* queries, size_t nq, size_t qstride, int k,
             int32_t* idx_out, float* d2_out, int threads);

/* fast_gicp::FastGICP::calculate_covariances, PLANE regularisation. cov_out: n x 9 doubles (3x3 row-major). */
void orc_gicp_covariances(const float* pts, size_t n, size_t stride, int k, double* cov_out, int threads);

/* fast_gicp::FastGICP::update_correspondences + linearize at pose T (4x4 double row-major).
 * corr_out[n] (index or -1), d2_out[n] (float NN d2), mahal_out[n*9] (may be NULL), H[36], b[6], returns sum e^T M e */
double orc_gicp_linearize(const float* src, size_t n, size_t sstride, const double* src_cov, const float* tgt, size_t m,
                          size_t tstride, const double* tgt_cov, const double* T, double max_corr_dist, int32_t* corr_out,
                          float* d2_out, double* mahal_out, double* H, double* b, int threads);

/* fast_gicp::FastGICP::compute_error with existing correspondences / mahalanobis. */
double orc_gicp_error(const float* src, size_t n, size_t sstride, const float* tgt, size_t tstride, const int32_t* corr,
                      const double* mahal, const double* T, int threads);

typedef struct {
  int max_iterations;            /* reg_maximum_iterations (64) */
  double transformation_epsilon; /* reg_transformation_epsilon (0.01) */
  double rotation_epsilon;       /* fast_gicp default 2e-3 */
  double max_corr_dist;          /* reg_max_correspondence_distance (2.5) */
  int k_correspondences;         /* reg_correspondence_randomness (20) */
  int num_threads;               /* reg_num_threads; 0 = all */
} orc_gicp_config;

typedef struct {
  float T[16];      /* final_transformation_ (row-major) */
  double T64[16];   /* x0 before the float cast */
  int converged;
  int iterations;   /* number of step_lm calls executed */
  int lm_failed;    /* "lm not converged!!" break */
  double last_error; /* y0 of the last linearize */
  int total_inner;  /* total LM trial solves */
} orc_gicp_result;

/* Full fast_gicp align(). src_cov/tgt_cov may be NULL (computed inside, as setInputSource/Target+align would).
 * trace_H (max_iterations*36), trace_b (max_iterations*6), trace_y (max_iterations) may be NULL.
 * corr_out (n) = correspondences of the LAST linearize, may be NULL. */
void orc_gicp_align(const float* src, size_t n, size_t sstride, const double* src_cov, const float* tgt, size_t m,
                    size_t tstride, const double* tgt_cov, const orc_gicp_config* cfg, const float* guess,
                    orc_gicp_result* res, double* trace_H, double* trace_b, double* trace_y, int32_t* corr_out);

/* A kept target: fast_gicp holds the target's kd-tree and covariances while the same target cloud stays set (SURVEY A.4), so
 * the per-frame / per-candidate cost of the reference is source kd-tree + source covariances + align.  `tgt` must outlive it. */
typedef struct orc_gicp_target orc_gicp_target;
orc_gicp_target* orc_gicp_target_create(const float* tgt, size_t m, size_t stride, int k, int threads);
void orc_gicp_target_free(orc_gicp_target* t);
void orc_gicp_align_to(const orc_gicp_target* t, const float* src, size_t n, size_t sstride, const double* src_cov /* or NULL */,
                       const orc_gicp_config* cfg, const float* guess, orc_gicp_result* res, int32_t* corr_out);
double orc_gicp_target_fitness(const orc_gicp_target* t, const float* src, size_t n, size_t sstride, const float* T, double max_range, int threads);

/* pcl::Registration::getFitnessScore(max_range) twin (information_matrix_calculator.cpp:49-80) plus the
 * inlier loop of scan_matching_odometry_nodelet.cpp:309-320.  T is float32 row-major. nn_idx/nn_d2 may be NULL. */
void orc_fitness(const float* tgt, size_t m, size_t tstride, const float* src, size_t n, size_t sstride, const float* T,
                 double max_range, float inlier_thresh_sq, double* score, uint32_t* nr, uint32_t* n_inliers,
                 int32_t* nn_idx, float* nn_d2, int threads);

/* pcl::VoxelGrid<PointXYZI>::filter with setLeafSize(leaf,leaf,leaf), downsample_all_data=true.
 * in: records of `stride` floats, intensity at float offset 4 (PointXYZI) — for stride 4 intensity = 0.
 * out_xyzi: capacity n*4 floats; out_keys/out_counts capacity n (may be NULL). returns 0 ok, 1 = leaf too small
 * (input passed through), n_out written. */
int orc_voxelgrid(const float* in, size_t n, size_t stride, float leaf, float* out_xyzi, int32_t* out_keys,
                  int32_t* out_counts, size_t* n_out);

/* prefilter chain ("next" rows): keep flags of PrefilteringNodelet::distance_filter, pcl::RadiusOutlierRemoval,
 * pcl::StatisticalOutlierRemoval (apps/prefiltering_nodelet.cpp:72-93,151-180). */
void orc_distance_filter(const float* pts, size_t n, size_t stride, double near_t, double far_t, unsigned char* keep);
void orc_radius_outlier(const float* pts, size_t n, size_t stride, double radius, int min_neighbors, unsigned char* keep, int threads);
void orc_statistical_outlier(const float* pts, size_t n, size_t stride, int mean_k, double stddev_mul, unsigned char* keep, float* dist_out,
                             int threads);

/* PrefilteringNodelet::deskewing (apps/prefiltering_nodelet.cpp:182-243); out: n records of `stride` floats */
void orc_deskew(const float* pts, size_t n, size_t stride, double scan_period, const float* angular_velocity, float* out);

/* ---- NDT (pclomp::NormalDistributionsTransform + VoxelGridCovariance) ---- */
typedef struct orc_ndt_map orc_ndt_map;
/* VoxelGridCovariance::applyFilter's finalisation of one voxel from its float64 moments (n points, sums S[3], second moments
 * S2[9] row-major): mean[3], cov[9] (after the eigenvalue clamp), icov[9].  Returns n, or -1 for an invalidated voxel. */
int orc_ndt_voxel_gaussian(int n, const double* S, const double* S2, double* mean, double* cov, double* icov);
orc_ndt_map* orc_ndt_build(const float* tgt, size_t m, size_t stride, float resolution);
void orc_ndt_free(orc_ndt_map*);
/* voxel table dump: returns number of leaves (all occupied leaves, ascending key). Arrays may be NULL to query size.
 * keys[V], npts[V] (-1 = invalidated), mean[V*3], cov[V*9], icov[V*9]; grid: min_b[3], div_b[3] */
size_t orc_ndt_dump(const orc_ndt_map*, int64_t* keys, int32_t* npts, double* mean, double* cov, double* icov,
                    int32_t* min_b, int32_t* div_b);

typedef struct {
  int max_iterations;             /* 64 */
  double transformation_epsilon;  /* 0.01 */
  double step_size;               /* 0.1 */
  double outlier_ratio;           /* 0.55 */
  double resolution;              /* 1.0 / 0.5 */
  int search_method;              /* 1 = DIRECT1, 7 = DIRECT7 */
  int num_threads;
  int mt_interval_flag;           /* 0 = ndt_omp polarity "(step_max-step_min) > 0" (line search loop never runs);
                                     1 = fixed polarity "< 0" (More-Thuente loop active) */
  int fixed_iterations;           /* >0: run exactly this many iterations, convergence test disabled (BASELINE config 3) */
} orc_ndt_config;

/* one computeDerivatives pass at parameter vector p (tx,ty,tz,rx,ry,rz). Returns score; g[6], H[36];
 * n_pairs = number of (point, cell) contributions visited (valid-cell lookups). per_point_cells (n, may be NULL) =
 * bitmask of DIRECT7 offsets accepted for each point (bit k = k-th offset in SURVEY A.3 order). */
double orc_ndt_derivatives(const orc_ndt_map*, const float* src, size_t n, size_t stride, const orc_ndt_config* cfg,
                           const double* p, double* g, double* H, uint64_t* n_pairs, uint8_t* per_point_cells);

/* ndt_omp computeHessian (float64, the pass run after an active More-Thuente loop) at p. H[36] row-major. */
void orc_ndt_hessian_at(const orc_ndt_map*, const float* src, size_t n, size_t stride, const orc_ndt_config* cfg,
                        const double* p, double* H);

typedef struct {
  float T[16];
  int converged;
  int iterations;
  double trans_probability;
  double p[6];
  uint64_t derivative_passes;     /* every pass over the source, the Hessian passes included */
  uint64_t hessian_passes;        /* float64 computeHessian passes (one after every More-Thuente loop that iterated) */
} orc_ndt_result;

void orc_ndt_align(const orc_ndt_map*, const float* src, size_t n, size_t stride, const orc_ndt_config* cfg,
                   const float* guess, orc_ndt_result* res, double* trace_p /* (max_iter+1)*6 or NULL */);

#ifdef __cplusplus
}
#endif
#endif
