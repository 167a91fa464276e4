/* b200reg.h — C ABI of libb200reg.so, the GPU-native (H100, sm_90a) scan-matching engine that drops in behind the
 * pcl::Registration<pcl::PointXYZI, pcl::PointXYZI> handle of koide3/hdl_graph_slam.
 *
 * Every entry point names the reference interface it replaces (paths relative to /root/reference).  The seam is
 * `select_registration_method()` (include/hdl_graph_slam/registrations.hpp:17, src/hdl_graph_slam/registrations.cpp:22-124);
 * its two consumers are ScanMatchingOdometryNodelet (apps/scan_matching_odometry_nodelet.cpp:106,165-262,298-335) and
 * LoopDetector (include/hdl_graph_slam/loop_detector.hpp:47,117-171).  INTEGRATION.md shows the adapter class and the
 * factory branch a maintainer adds.
 *
 * Conventions
 *   - Point records: float32 x,y,z at byte offsets 0,4,8 of a record `stride_bytes` long (16 = packed float4,
 *     32 = pcl::PointXYZI with intensity at offset 16).  Host pointers may be pageable or pinned (pinned buffers
 *     are DMA'd directly); the engine copies, the caller keeps ownership: when b2r_set_source / b2r_set_target /
 *     b2r_odometry_matching / b2r_loop_matching return, the copy out of the caller's buffer has finished and the buffer may be
 *     reused.  Only the explicitly asynchronous entry points keep reading it after they return: b2r_prefetch_source /
 *     b2r_odometry_prefetch (until the b2r_set_source that adopts the cloud returns; a buffer rewritten in between is detected by
 *     a content stamp and uploaded afresh) and b2r_batch_add_cloud with pinned memory (until the next b2r_batch_* call that
 *     aligns or synchronises returns).  DEVICE pointers (b2r_set_*_device, b2r_odometry_matching_device, b2r_*_add_cloud_device) are
 *     read in place, never copied, while the cloud's search structure and covariances are built: keep them valid and unmodified
 *     until the align / matching / batch call that first uses the cloud returns (an NDT handle takes a device-to-device copy instead,
 *     because a target's voxel map is built only when the cloud has been promoted to target).  b2r_get_aligned re-reads the
 *     source buffer.
 *   - 4x4 matrices are COLUMN-major (what Eigen::Matrix4f::data() / Eigen::Matrix4d::data() hand out).
 *   - Every function returns 0 on success or a negative B2R_E* code; nothing throws or aborts; on failure
 *     b2r_last_error() holds a message and results report converged = 0 (the reference's failure signal,
 *     scan_matching_odometry_nodelet.cpp:214-218, loop_detector.hpp:147).
 *   - A handle is used by one thread at a time; distinct handles are independent (own stream and buffers), matching
 *     the reference's two concurrently-live registration objects (odometry + loop closure).
 *   - There is no CPU fallback: without a CUDA device b2r_create fails with B2R_ENODEVICE.
 */
#ifndef B200REG_H
#define B200REG_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B2R_OK 0
#define B2R_EINVAL (-1)     /* bad argument */
#define B2R_ENODEVICE (-2)  /* no CUDA device / CUDA initialisation failed */
#define B2R_ECUDA (-3)      /* CUDA runtime error (message in b2r_last_error) */
#define B2R_ESTATE (-4)     /* source/target not set */
#define B2R_EUNSUPPORTED (-5) /* registration_method that this engine does not re-create */
#define B2R_ENCCL (-6)

#define B2R_METHOD_GICP 0 /* fast_gicp::FastGICP semantics   (registrations.cpp:27-36)   */
#define B2R_METHOD_NDT 1  /* pclomp::NormalDistributionsTransform semantics (registrations.cpp:101-120) */
#define B2R_METHOD_NDT_PCL 2 /* pcl::NormalDistributionsTransform semantics (registrations.cpp:93-100): radius neighbourhood over the
                                voxel centroids, float64 derivatives; reads ndt_resolution / ndt_step_size / ndt_outlier_ratio /
                                ndt_mt_interval_flag / ndt_fixed_iterations, not ndt_search_method */
#define B2R_METHOD_VGICP 3 /* fast_gicp::FastVGICP semantics (registrations.cpp:48-56): FastGICP's covariances, the target's Gaussian voxel
                              map at ndt_resolution (reg_resolution), DIRECT1 voxel correspondences, weights sqrt(num_points); reads
                              max_iterations / k_correspondences / transformation_epsilon, not max_correspondence_distance */
#define B2R_METHOD_GICP_PCL 4 /* pcl::GeneralizedIterativeClosestPoint semantics (PCL 1.10, registrations.cpp:66-76): raw-moment k-NN
                                 covariances, exact 1-NN Mahalanobis correspondences, PCL's BFGS over (t, euler ZYX); reads
                                 max_iterations / k_correspondences / transformation_epsilon / max_correspondence_distance /
                                 max_optimizer_iterations; rotation_epsilon stays 2e-3.  The BFGS runs on the host (one device pass per correspondence
                                 update and per functor evaluation); a batch gathers every pair's pass of a round into shared launches */
#define B2R_METHOD_ICP_PCL 5 /* pcl::IterativeClosestPoint semantics (PCL 1.10, registrations.cpp:57-65): exact 1-NN correspondences accepted at
                                d2 <= max_correspondence_distance^2 (optionally reciprocal), pcl::umeyama's SVD step, DefaultConvergenceCriteria;
                                reads max_iterations / transformation_epsilon / max_correspondence_distance / use_reciprocal_correspondences.
                                The whole loop runs on the device: 2 launches per iteration, 4 with the reciprocal check */
#define B2R_METHOD_VGICP_CUDA 6 /* fast_gicp::FastVGICPCuda semantics (registrations.cpp:37-47, opted into as B200_VGICP_CUDA):
                                   float32 raw-moment k-NN covariances with float32 PLANE, the target's float32 Gaussian voxel map at
                                   ndt_resolution (reg_resolution) with cells floor(p / res - 0.5), DIRECT1 voxel correspondences and
                                   float32 terms weighted sqrt(num_points), summed in float64; reads max_iterations / k_correspondences /
                                   transformation_epsilon, not max_correspondence_distance */
/* id 7 is left unassigned (an unknown method: b2r_config_default returns B2R_EINVAL for it) */
#define B2R_METHOD_GICP_OMP 8 /* pclomp::GeneralizedIterativeClosestPoint semantics (ndt_omp's copy of PCL's GICP, registrations.cpp:76-86,
                                 opted into as B200_GICP_OMP): B2R_METHOD_GICP_PCL's covariances, correspondences, BFGS and outer loop,
                                 reading the same fields, except the pose every functor evaluation (cost pass) uses: applyState(guess, x)
                                 = [R(x) R_guess | t_guess + t(x)] applied to the raw source point, where pcl GICP applies applyState(I, x)
                                 to guess * p.  With a translated guess the end pose differs from GICP's by about (R(x*) - I) t_guess.
                                 This pose rule is recalled, not read from the sources (DOUBT) */
#define B2R_METHOD_NDT_KDTREE 9 /* pclomp::NormalDistributionsTransform with reg_nn_search_method = KDTREE (registrations.cpp:112-113,
                                   opted into as B200_NDT_KDTREE): B2R_METHOD_NDT's voxel map, float32 term, float64 Hessian-only pass and
                                   Newton / More-Thuente driver over B2R_METHOD_NDT_PCL's neighbourhood (every voxel centroid within
                                   ndt_resolution, float32 d2 < (float)r^2, no nr_points check); reads ndt_resolution / ndt_step_size /
                                   ndt_outlier_ratio / ndt_mt_interval_flag / ndt_fixed_iterations, not ndt_search_method */

typedef struct b2r_handle b2r_handle;

/* Mirrors the per-method setters the factory feeds from rosparams (registrations.cpp:30-34,106-118; SURVEY App. B). */
typedef struct b2r_config {
  int32_t method;                     /* B2R_METHOD_* */
  int32_t device_id;                  /* CUDA device ordinal */
  int32_t max_iterations;             /* reg_maximum_iterations            (64)   */
  int32_t k_correspondences;          /* reg_correspondence_randomness     (20)   */
  double transformation_epsilon;      /* reg_transformation_epsilon        (0.01) */
  double rotation_epsilon;            /* fast_gicp rotation_epsilon_       (2e-3) */
  double max_correspondence_distance; /* reg_max_correspondence_distance   (2.5)  */
  double ndt_resolution;              /* reg_resolution                    (0.5 code default, 1.0 in launch files) */
  double ndt_step_size;               /* ndt_omp step_size_                (0.1)  */
  double ndt_outlier_ratio;           /* ndt_omp outlier_ratio_            (0.55) */
  int32_t ndt_search_method;          /* reg_nn_search_method: 1 = DIRECT1, 7 = DIRECT7 (default) */
  int32_t ndt_mt_interval_flag;       /* 0 = ndt_omp polarity (More-Thuente loop never entered), 1 = active line search */
  int32_t ndt_fixed_iterations;       /* >0: exactly this many iterations (BASELINE config 3), convergence test off */
  float grid_cell_min;                /* engine tuning: smallest search-grid cell, power of two (default 0.5 m) */
  int32_t max_optimizer_iterations;   /* reg_max_optimizer_iterations      (20)   pcl GICP max_inner_iterations_ (B2R_METHOD_GICP_PCL, _GICP_OMP) */
  int32_t use_reciprocal_correspondences; /* reg_use_reciprocal_correspondences (false): 0 or 1, read by B2R_METHOD_ICP_PCL only */
} b2r_config;

/* What the callers read back after align(): getFinalTransformation(), hasConverged(), and (loop closure)
 * getFitnessScore().  80 bytes — also the record all-gathered across GPUs by the batch path. */
typedef struct b2r_result {
  float T[16];        /* final_transformation_, column-major */
  double fitness;     /* getFitnessScore(max_range) when requested, else NaN */
  int32_t converged;  /* hasConverged() */
  int32_t iterations; /* outer iterations executed */
} b2r_result;

const char* b2r_last_error(void);
const char* b2r_version(void);

/* defaults of the reference factory for `method` */
int b2r_config_default(b2r_config* cfg, int method);

/* replaces select_registration_method(ros::NodeHandle&) (registrations.cpp:22-124): same parameter NAMES and defaults,
 * passed as string key/value pairs (the rosparam namespace of the nodelet).  "FAST_GICP"/"B200_GICP" -> GICP engine,
 * "NDT_OMP"/"B200_NDT" -> NDT engine, "NDT" -> pcl NDT engine (B2R_METHOD_NDT_PCL), "FAST_VGICP"/"B200_VGICP" -> VGICP engine
 * (B2R_METHOD_VGICP), "GICP"/"B200_GICP_PCL" and every other name that reaches the reference's GICP branch (contains "GICP" but not
 * "OMP") -> pcl GICP engine (B2R_METHOD_GICP_PCL), "B200_ICP" -> pcl ICP engine (B2R_METHOD_ICP_PCL; reg_use_reciprocal_correspondences
 * must be true / false / 1 / 0, else B2R_EINVAL), "B200_VGICP_CUDA" -> FastVGICPCuda engine (B2R_METHOD_VGICP_CUDA),
 * "B200_GICP_OMP" -> pclomp GICP engine (B2R_METHOD_GICP_OMP; the GICP branch's parameters and defaults), "B200_NDT_KDTREE" ->
 * NDT_OMP's KDTREE search (B2R_METHOD_NDT_KDTREE; reg_resolution, reg_transformation_epsilon, reg_maximum_iterations).
 * NDT_OMP / B200_NDT with reg_nn_search_method = KDTREE, ICP / GICP_OMP (and every other name containing GICP and OMP) / FAST_VGICP_CUDA and unknown names are not re-created: returns
 * B2R_EUNSUPPORTED so the caller keeps the reference's own branch.  (Built without USE_VGICP_CUDA the reference sends FAST_VGICP_CUDA to
 * its GICP branch; this factory refuses it all the same, so the caller decides.) */
int b2r_select_registration_method(const char* const* keys, const char* const* values, int n_params, int device_id,
                                   b2r_handle** out);

int b2r_create(const b2r_config* cfg, b2r_handle** out);
void b2r_destroy(b2r_handle* h);
int b2r_get_config(const b2r_handle* h, b2r_config* out);

/* replaces registration->setInputTarget(cloud) (scan_matching_odometry_nodelet.cpp:172,246; loop_detector.hpp:122).
 * Uploads, builds the search grid and (GICP) the k-NN covariances or (NDT) the voxel Gaussians. */
int b2r_set_target(b2r_handle* h, const void* points, size_t n, size_t stride_bytes);
/* replaces registration->setInputSource(cloud) (scan_matching_odometry_nodelet.cpp:177; loop_detector.hpp:136). */
int b2r_set_source(b2r_handle* h, const void* points, size_t n, size_t stride_bytes);
/* same, for clouds already resident in device memory (device pointers; used by the HBM-resident measurement and by
 * device-side pipelines such as b2r_voxelgrid_device -> registration). */
int b2r_set_target_device(b2r_handle* h, const void* d_points, size_t n, size_t stride_bytes);
int b2r_set_source_device(b2r_handle* h, const void* d_points, size_t n, size_t stride_bytes);
/* telemetry: bytes copied over PCIe, kernel launches and (when profiling is on) CUDA-event time per kernel class.
 * Used by bench.py for h2d/d2h_bytes_per_step, gpu_launches and the live roofline of the dominant kernel. */
typedef struct b2r_stats {
  uint64_t h2d_bytes, d2h_bytes;
  int32_t n_classes, reserved;
  uint64_t launches[16]; /* kernel launches per class */
  uint64_t calls[16];    /* timed spans per class */
  double ms[16];         /* CUDA-event milliseconds per class (profiling on) */
} b2r_stats;
int b2r_set_profiling(b2r_handle* h, int on);
int b2r_get_stats(b2r_handle* h, b2r_stats* out, int reset);
const char* b2r_kernel_class_name(int cls);
/* the CUDA stream (cudaStream_t) every kernel of this handle is launched on, so callers can bracket it with events */
int b2r_get_stream(b2r_handle* h, void** stream);
/* Software pipelining for replay / batch callers that already hold the NEXT source cloud: uploads it and builds its search
 * structure and covariances on a second stream while the current align() runs.  A following b2r_set_source[_device] with the
 * same pointer, size and stride adopts the prefetched cloud instead of repeating the work.  Results are unchanged. */
int b2r_prefetch_source(b2r_handle* h, const void* points, size_t n, size_t stride_bytes);
int b2r_prefetch_source_device(b2r_handle* h, const void* d_points, size_t n, size_t stride_bytes);
/* block until everything enqueued on the handle's stream (uploads, grid / covariance / voxel builds) has finished */
int b2r_synchronize(b2r_handle* h);
/* keyframe switch `keyframe = filtered; registration->setInputTarget(keyframe)` (scan_matching_odometry_nodelet.cpp:245-246):
 * the current source (points, grid, covariances) becomes the target without re-upload or recomputation.
 * Afterwards the handle has NO source until the next b2r_set_source* (or an adopted prefetch): b2r_align (which reports converged = 0
 * and the guess, like every failed align), b2r_fitness, b2r_get_aligned, a second b2r_promote_source_to_target and every parity tap
 * that reads the source (b2r_get_correspondences, b2r_get_covariances with which = 0, b2r_gicp_linearize_at, b2r_ndt_derivatives_at,
 * b2r_ndt_hessian_at, b2r_ndt_neighbors_at) return B2R_ESTATE.
 * The displaced target's records are never read again, so a target registered from device memory may be released by its owner. */
int b2r_promote_source_to_target(b2r_handle* h);

/* replaces registration->align(*aligned, guess) + hasConverged() + getFinalTransformation()
 * (scan_matching_odometry_nodelet.cpp:210,214,220; loop_detector.hpp:143,147,153). */
int b2r_align(b2r_handle* h, const float guess[16], b2r_result* out);

/* the `aligned` output cloud of align(): source transformed by the final pose.  Writes x,y,z (and 1.0f at offset 12 when
 * stride_bytes >= 16) of n records; other bytes are left untouched.  n must be the source's size (B2R_EINVAL otherwise).  The pose is
 * the last successful align's (identity before any; an align that returned an error leaves it as it was). */
int b2r_get_aligned(b2r_handle* h, void* out_points, size_t n, size_t stride_bytes);

/* replaces registration->getFitnessScore(max_range) (scan_matching_odometry_nodelet.cpp:307; loop_detector.hpp:146;
 * twin: information_matrix_calculator.cpp:49-80) and the inlier loop of scan_matching_odometry_nodelet.cpp:309-320.
 * T = NULL uses the last final transformation.  max_range is compared against the SQUARED distance, as in the reference. */
int b2r_fitness(b2r_handle* h, const float* T, double max_range, float inlier_thresh_sq, double* score, uint32_t* n_used,
                uint32_t* n_inliers);

/* replaces registration->getSearchMethodTarget()->nearestKSearch(pt, 1, ...) (scan_matching_odometry_nodelet.cpp:316):
 * exact 1-NN of n query points in the current target. */
int b2r_target_nearest(b2r_handle* h, const void* queries, size_t n, size_t stride_bytes, int32_t* idx_out, float* d2_out);

/* ---- parity / debug taps (not used by the reference's callers) ------------------------------------------------ */
/* correspondences_ of the last linearisation (target index per source point, -1 = rejected) */
int b2r_get_correspondences(b2r_handle* h, int32_t* out, size_t n);
/* which: 0 = source, 1 = target.  out: n x 9 doubles (3x3 row-major), original point order (GICP). */
int b2r_get_covariances(b2r_handle* h, int which, double* out, size_t n);
/* one update_correspondences + linearize at pose T (column-major double): H[36] row-major, b[6], *err = sum e^T M e */
int b2r_gicp_linearize_at(b2r_handle* h, const double T[16], double* H, double* b, double* err);
/* one compute_error at pose T with the correspondences of the last linearisation (GICP handle only: B2R_ESTATE on any other method) */
int b2r_gicp_error_at(b2r_handle* h, const double T[16], double* err);
/* NDT voxel table of the target (any NDT method): returns count through *n_voxels; arrays may be NULL.  keys ascending. */
int b2r_ndt_get_voxels(b2r_handle* h, size_t capacity, size_t* n_voxels, int64_t* keys, int32_t* npts, double* mean, double* icov,
                       int32_t min_b[3], int32_t div_b[3]);
/* one computeDerivatives pass at p = (tx,ty,tz,rx,ry,rz): score, g[6], H[36] row-major, number of (point,cell) pairs
 * (B2R_METHOD_NDT_PCL / _NDT_KDTREE: (point, radius neighbour) pairs) */
int b2r_ndt_derivatives_at(b2r_handle* h, const double p[6], double* score, double* g, double* H, uint64_t* n_pairs);
/* one float64 computeHessian pass at p (the pass the align runs after an active More-Thuente line search): H[36] row-major
 * (B2R_METHOD_NDT_KDTREE: over the radius neighbours) */
int b2r_ndt_hessian_at(b2r_handle* h, const double p[6], double* H);
/* B2R_METHOD_NDT_PCL / _NDT_KDTREE: the searchable centroid cloud of the target (VoxelGridCovariance::filter(true)): the leaf key and float32
 * centroid (xyz: 3 floats each) of every leaf with at least 6 points, keys ascending; *n_centroids = the count; arrays may be NULL */
int b2r_ndt_get_centroids(b2r_handle* h, size_t capacity, size_t* n_centroids, int64_t* keys, float* xyz);
/* B2R_METHOD_NDT_PCL / _NDT_KDTREE: the radiusSearch(T(p) x, resolution) of every source point, in the caller's point order: counts[i] (n source
 * entries, may be NULL) and one flat array of the neighbours' leaf keys, ascending within each point (CSR by counts; the first
 * `capacity` entries are written, keys may be NULL); *total = the number of (point, neighbour) pairs */
int b2r_ndt_neighbors_at(b2r_handle* h, const double p[6], uint32_t* counts, size_t capacity, int64_t* keys, size_t* total);
/* B2R_METHOD_VGICP / B2R_METHOD_VGICP_CUDA: the target's Gaussian voxel map (GaussianVoxelMap after finalize), cells ascending (x,
 * then y, then z): cells[3 V] = floor(p / resolution) per axis (VGICP_CUDA: floorf(p / resolution - 0.5f) in float32), counts[V] = num_points, mean[3 V], cov[9 V] (3x3 row-major); *n_voxels = V; the first
 * `capacity` voxels are written, every array may be NULL.  B2R_EUNSUPPORTED when a finite target point lies 2^20 cells or more from
 * the origin on an axis (the keys hold 21 bits per axis); points with a non-finite coordinate belong to no voxel. */
int b2r_vgicp_get_voxels(b2r_handle* h, size_t capacity, size_t* n_voxels, int32_t* cells, int32_t* counts, double* mean, double* cov);
/* B2R_METHOD_VGICP / B2R_METHOD_VGICP_CUDA: one update_correspondences (DIRECT1) + linearize at pose T (column-major double): H[36]
 * row-major, b[6], *cost = sum sqrt(num_points) e^T M e (VGICP_CUDA: float32 terms at T rounded to float32, summed in float64), *n_corr = source points with a voxel, voxel_of (n source entries in the caller's point order,
 * may be NULL) = the index of the point's voxel in b2r_vgicp_get_voxels' order, or -1 */
int b2r_vgicp_linearize_at(b2r_handle* h, const double T[16], double* H, double* b, double* cost, uint64_t* n_corr, int32_t* voxel_of, size_t n);

/* B2R_METHOD_GICP_PCL / B2R_METHOD_GICP_OMP (the same pass for both): one correspondence pass of pcl GICP's computeTransformation at the guess (applied to the source first,
 * transformPointCloud) and T_rel (transformation_), both column-major float: corr[n] (caller's point order, may be NULL) = the target
 * index of the exact 1-NN when its squared distance < max_correspondence_distance^2, else -1; M[9 n] (may be NULL) = the Mahalanobis
 * matrix (R C1 R^T + C2)^-1, 3x3 row-major, of every accepted point (NaN elsewhere); *n_corr = the accepted count.  The cost tap below
 * reads these correspondences. */
int b2r_gicp_pcl_correspondences_at(b2r_handle* h, const float guess[16], const float T_rel[16], int32_t* corr, double* M, uint64_t* n_corr);
/* B2R_METHOD_GICP_PCL / B2R_METHOD_GICP_OMP: one cost pass (OptimizationFunctorWithIndices) at the column-major float pose T over the
 * last correspondences: *f_sum = sum res^T M res, g_sum[3] = sum M res, dR_sum[9] = sum p_src (M res)^T (row-major), unscaled (the
 * functor divides by m), with p_src = guess * p.  GICP_PCL: res = T (guess * p) - q, T being applyState(I, x) in an align.  GICP_OMP:
 * res = T p - q on the raw source point p, T being applyState(guess, x) in an align, with the guess of the last correspondence pass */
int b2r_gicp_pcl_cost_at(b2r_handle* h, const float T[16], double* f_sum, double* g_sum, double* dR_sum);

/* B2R_METHOD_ICP_PCL: one correspondence pass with the source transformed once by the column-major float T (transformPointCloud),
 * forward or reciprocal as configured: corr[n] (caller's point order, may be NULL) = the target index of the accepted correspondence or
 * -1, d2[n] (may be NULL) = its squared distance (NaN where there is none), *count = the accepted number */
int b2r_icp_pcl_correspondences_at(b2r_handle* h, const float T[16], int32_t* corr, float* d2, uint64_t* count);
/* B2R_METHOD_ICP_PCL: the same pass, then TransformationEstimationSVD (pcl::umeyama) on it: transformation[16] column-major float and
 * sums[17] = count, sum d2, sum src (3), sum tgt (3) of the accepted pairs, then sum (tgt - tgt_mean)_i (src - src_mean)_j row-major (9).
 * B2R_ESTATE below 3 correspondences (the align stops there unconverged) */
int b2r_icp_pcl_estimate_at(b2r_handle* h, const float T[16], float* transformation, double* sums);

/* ---- companion: voxel-grid downsample ---------------------------------------------------------------------------
 * replaces pcl::VoxelGrid<PointXYZI>::filter with setLeafSize(leaf,leaf,leaf) (apps/prefiltering_nodelet.cpp:54-58,138-149;
 * apps/scan_matching_odometry_nodelet.cpp:86-90,147-157).  in/out records are `stride_bytes` long with intensity at byte
 * offset 16 when stride_bytes >= 20.  out must hold n records; *n_out receives the voxel count; out_keys/out_counts
 * (capacity n) may be NULL.  Returns 1 (and passes the input through) when the leaf is too small for int32 indices. */
int b2r_voxelgrid(b2r_handle* h, const void* in, size_t n, size_t stride_bytes, float leaf, void* out, size_t* n_out,
                  int32_t* out_keys, int32_t* out_counts);

/* the same filter with input and output resident in device memory: *d_out receives an engine-owned device buffer of *n_out records
 * (same record layout as the input; valid until the next voxel-grid call on this handle) that can go straight into
 * b2r_set_source_device / b2r_set_target_device / b2r_batch_add_cloud_device / b2r_odometry_matching_device — downsample ->
 * registration without leaving HBM.  Returns 1 with *d_out = d_in when the leaf is too small (pass-through). */
int b2r_voxelgrid_device(b2r_handle* h, const void* d_in, size_t n, size_t stride_bytes, float leaf, const void** d_out, size_t* n_out);

/* ---- companion: approximate voxel-grid downsample ------------------------------------------------------------------
 * replaces pcl::ApproximateVoxelGrid<PointXYZI>::filter with setLeafSize(leaf,leaf,leaf) and its 512-slot hash table
 * (apps/prefiltering_nodelet.cpp:61-63,138-149; downsample_method "APPROX_VOXELGRID").  Records as for b2r_voxelgrid; the outputs
 * come in PCL's order (flushes on hash collisions in input order, then the remaining slots 0..511), and one cell may appear more
 * than once.  out must hold n records; *n_out receives the output count; out_counts (capacity n, may be NULL) the points per output.
 * Non-finite points are not skipped (PCL has no check).  B2R_EINVAL for a leaf that is not finite and positive or a bad stride. */
int b2r_approximate_voxelgrid(b2r_handle* h, const void* in, size_t n, size_t stride_bytes, float leaf, void* out, size_t* n_out,
                              int32_t* out_counts);
/* the same filter with input and output resident in device memory: *d_out receives an engine-owned device buffer of *n_out records
 * (valid until the next voxel-grid or prefilter call on this handle) for b2r_set_source_device and the other device entry points. */
int b2r_approximate_voxelgrid_device(b2r_handle* h, const void* d_in, size_t n, size_t stride_bytes, float leaf, const void** d_out,
                                     size_t* n_out);

/* ---- "next" rows (SURVEY.md 8f-2): the rest of the prefilter chain.  Records are copied whole; kept points stay in input order.
 * PrefilteringNodelet::distance_filter (apps/prefiltering_nodelet.cpp:164-180): keep near < ||p|| < far (float32 norm). */
int b2r_distance_filter(b2r_handle* h, const void* in, size_t n, size_t stride_bytes, double near_thresh, double far_thresh, void* out, size_t* n_out);
/* pcl::RadiusOutlierRemoval with setRadiusSearch / setMinNeighborsInRadius (apps/prefiltering_nodelet.cpp:83-90,151-162) */
int b2r_radius_outlier_removal(b2r_handle* h, const void* in, size_t n, size_t stride_bytes, double radius, int min_neighbors, void* out, size_t* n_out);
/* pcl::StatisticalOutlierRemoval with setMeanK / setStddevMulThresh (apps/prefiltering_nodelet.cpp:73-81,151-162) */
int b2r_statistical_outlier_removal(b2r_handle* h, const void* in, size_t n, size_t stride_bytes, int mean_k, double stddev_mul, void* out, size_t* n_out);

/* PrefilteringNodelet::deskewing (apps/prefiltering_nodelet.cpp:182-243): point i rotated back by the gyro rate over its share of
 * the scan period (float32, Eigen's quaternion arithmetic; the quaternion (1, dt/2 w) is not normalised, as in the reference).
 * angular_velocity = the IMU message's angular_velocity (the engine negates it, :217).  out: n records. */
int b2r_deskew(b2r_handle* h, const void* in, size_t n, size_t stride_bytes, double scan_period, const float angular_velocity[3], void* out);

/* PrefilteringNodelet::cloud_callback (apps/prefiltering_nodelet.cpp:106-136) as ONE call with the cloud resident in HBM between the
 * stages: deskewing -> [base_link transform] -> distance_filter -> downsample -> outlier_removal.  Keep flags, the statistical
 * filter's mean / stddev and the compactions are computed on the device.  points: host records, or device records when
 * device_input != 0.  The result stays in an engine-owned device buffer (*d_out, valid until the next prefilter / voxel-grid call
 * on this handle; pass it to b2r_set_source_device / b2r_odometry_matching_device) and is also copied to out_host when that is
 * not NULL (capacity n records). */
#define B2R_DOWNSAMPLE_NONE 0
#define B2R_DOWNSAMPLE_VOXELGRID 1
#define B2R_DOWNSAMPLE_APPROX_VOXELGRID 2  /* :59-63; any other value passes the cloud through, as the reference does (:64-70) */
#define B2R_OUTLIER_NONE 0
#define B2R_OUTLIER_STATISTICAL 1
#define B2R_OUTLIER_RADIUS 2
typedef struct b2r_prefilter_params {
  int32_t deskewing;              /* "deskewing" (false)                                   prefiltering_nodelet.cpp:36  */
  int32_t use_base_link_transform;/* base_link_frame set                                    :114                         */
  double scan_period;             /* "scan_period" (0.1)                                    :234                         */
  float angular_velocity[3];      /* imu_msg->angular_velocity of the scan's stamp          :215                         */
  float base_link_transform[16];  /* column-major sensor -> base_link                       :121-126                     */
  int32_t use_distance_filter;    /* "use_distance_filter" (true)                           :96                          */
  double distance_near_thresh;    /* 1.0                                                    :97                          */
  double distance_far_thresh;     /* 100.0                                                  :98                          */
  int32_t downsample_method;      /* "downsample_method" VOXELGRID (or NONE, APPROX_VOXELGRID) :51                        */
  float downsample_resolution;    /* 0.1                                                    :52                          */
  int32_t outlier_removal_method; /* "outlier_removal_method" STATISTICAL                   :71                          */
  int32_t statistical_mean_k;     /* 20                                                     :73                          */
  double statistical_stddev;      /* 1.0                                                    :74                          */
  double radius_radius;           /* 0.8                                                    :83                          */
  int32_t radius_min_neighbors;   /* 2                                                      :84                          */
  int32_t reserved;
} b2r_prefilter_params;
int b2r_prefilter_params_default(b2r_prefilter_params* p);
int b2r_prefilter(b2r_handle* h, const void* points, size_t n, size_t stride_bytes, int device_input, const b2r_prefilter_params* p,
                  void* out_host, const void** d_out, size_t* n_out);

/* replaces FloorDetectionNodelet::detect (apps/floor_detection_nodelet.cpp:110-180) on the cloud of its cloud_callback (:72-103):
 * tilt, the height band of two plane clips, the k = 10 normal filter, the back-transform, the size gate, PCL 1.10's seeded RANSAC
 * plane fit (threshold 0.1) replayed hypothesis for hypothesis, the inlier gate, the verticality check and the upward flip.
 * points: host records, or device records when device_input != 0 (e.g. b2r_prefilter's *d_out); stride 12..48 bytes, x y z first,
 * every other field copied.  The call uses its own device buffers: no registration cloud, prefilter or voxel-grid output changes.
 *   filtered_host  (capacity n records, may be NULL) <- /floor_detection/floor_filtered_points (:127-130)
 *   inliers_host   (capacity n records, may be NULL) <- /floor_detection/floor_points (:168-177); filled whenever RANSAC found a
 *                  model (result->n_inliers records), which the reference publishes only when the floor is detected
 *   d_filtered / d_inliers (may be NULL) <- the same clouds in engine-owned device memory, valid until the next floor call on this
 *                  handle; NULL when empty.
 * Returns B2R_OK whenever the arguments are valid; result->detected says whether a FloorCoeffs message carries coefficients. */
#define B2R_FLOOR_OK 0
#define B2R_FLOOR_EMPTY_INPUT 1       /* no message at all (:76-78) */
#define B2R_FLOOR_TOO_FEW_FILTERED 2  /* filtered->size() < floor_pts_thresh (:133; size_t against int: a negative threshold always) */
#define B2R_FLOOR_NO_MODEL 3          /* RANSAC selected no sample (fewer than 3 points, or 1000 collinear draws) (:141) */
#define B2R_FLOOR_TOO_FEW_INLIERS 4   /* inliers->indices.size() < floor_pts_thresh (:147) */
#define B2R_FLOOR_NOT_VERTICAL 5      /* |coeffs.head<3>() . tilt^-1 UnitZ| < cos(floor_normal_thresh) (:152-161) */
typedef struct b2r_floor_params {
  double tilt_deg;                /* "tilt_deg" (0.0)                                     floor_detection_nodelet.cpp:57 */
  double sensor_height;           /* "sensor_height" (2.0)                                :58                            */
  double height_clip_range;       /* "height_clip_range" (1.0)                            :59                            */
  int32_t floor_pts_thresh;       /* "floor_pts_thresh" (512)                             :60                            */
  int32_t use_normal_filtering;   /* "use_normal_filtering" (true)                        :62                            */
  double floor_normal_thresh;     /* "floor_normal_thresh" (10.0 deg)                     :61                            */
  double normal_filter_thresh;    /* "normal_filter_thresh" (20.0 deg)                    :63                            */
} b2r_floor_params;
typedef struct b2r_floor_result {
  int32_t detected;               /* detect() returned coefficients                                                     */
  int32_t reason;                 /* B2R_FLOOR_*                                                                        */
  float coeffs[4];                /* the published plane (normal up, :164-166); RANSAC's model when not detected        */
  uint64_t n_filtered;            /* points after the band, normal filter and back-transform (:116-125)                */
  uint64_t n_inliers;             /* selectWithinDistance of the best model (:143-144)                                  */
  int32_t ransac_iterations;      /* RandomSampleConsensus::iterations_ at the end of computeModel (INT_MAX - 1 when the
                                     filtered cloud has fewer than 3 points: getSamples sets it so)                      */
  int32_t model_indices[3];       /* getModel(): the best sample's indices into the filtered cloud (-1: none)          */
  int32_t ransac_batches;         /* device round trips of the RANSAC replay                                           */
  int32_t ransac_hypotheses;      /* hypotheses drawn and counted on the device                                        */
  int32_t readbacks;              /* times the call waited for data from the device: kept counts, RANSAC batches, copies */
  int32_t reserved;
} b2r_floor_result;
int b2r_floor_params_default(b2r_floor_params* p);
int b2r_floor_detect(b2r_handle* h, const void* points, size_t n, size_t stride_bytes, int device_input, const b2r_floor_params* p,
                     b2r_floor_result* result, void* filtered_host, void* inliers_host, const void** d_filtered, const void** d_inliers);

/* replaces MapCloudGenerator::generate(keyframes, resolution) (src/hdl_graph_slam/map_cloud_generator.cpp:13-51; called at
 * apps/hdl_graph_slam_nodelet.cpp:528,989): every keyframe cloud transformed by its optimised pose (float32), all concatenated;
 * resolution <= 0 returns that cloud (intensity kept), otherwise the centres of the occupied voxels of a
 * pcl::octree::OctreePointCloud(resolution) — the same SET of centres as PCL's lattice (anchored at the first finite point),
 * emitted in ascending key order instead of octree traversal order; x,y,z,1 with intensity 0.
 * Returns 1 with *n_out = 0 when there is no keyframe ("warning: keyframes empty!!").  out: capacity out_capacity records.
 * Fails with B2R_EUNSUPPORTED when resolution > 0 and the octree needs more than 21 levels to hold every point (the voxel keys
 * hold 21 bits per axis: e.g. resolution 0.001 with points 3 km apart); PCL would grow a deeper octree. */
typedef struct b2r_keyframe_snapshot {
  const void* points;  /* KeyFrameSnapshot::cloud: n records of stride_bytes */
  size_t n;
  float pose[16];      /* KeyFrameSnapshot::pose.matrix().cast<float>(), column-major */
} b2r_keyframe_snapshot;
int b2r_map_cloud_generate(b2r_handle* h, const b2r_keyframe_snapshot* keyframes, size_t n_keyframes, size_t stride_bytes, double resolution,
                           void* out, size_t out_capacity, size_t* n_out);

/* ---- wire / disk formats at the seam (SURVEY.md 8f-4) ----------------------------------------------------------------
 * A sensor_msgs/PointCloud2 data[] blob (or a binary PCD body) goes to the device unconverted and is unpacked there into
 * pcl::PointXYZI records (32 bytes: x y z 1 | intensity 0 0 0) — the work of pcl::fromROSMsg at
 * apps/scan_matching_odometry_nodelet.cpp:118-119 and apps/hdl_graph_slam_nodelet.cpp:153-154, and of pcl::io::loadPCDFile at
 * src/hdl_graph_slam/keyframe.cpp:141.  *d_points is an engine-owned device buffer for b2r_set_source_device /
 * b2r_set_target_device / b2r_prefilter(device_input = 1) / b2r_batch_add_cloud_device / b2r_odometry_matching_ros(device = 1).  Two
 * such buffers are used in turn, so it stays valid until the SECOND ingest call after it on this handle: a frame ingested and matched
 * on the odometry's own handle is still intact while the next frame is ingested and matched against it.
 *   - Field mapping as PCL's fromPCLPointCloud2 does it for PointXYZI: intensity is read only when its datatype is FLOAT32; an
 *     intensity field of any other datatype is left unmapped and every point gets intensity 0 (PCL warns and does the same).
 *   - is_bigendian is honoured: x, y, z and intensity are byte-swapped.  (PCL copies the bytes as they are, so a big-endian
 *     message on a little-endian host decodes to garbage there; this is a deliberate deviation.)
 *   - b2r_ingest_pointcloud2 takes contiguous rows: n_points records of point_step bytes back to back, i.e. row_step == width *
 *     point_step.  An organized message with padded rows (row_step > width * point_step), which fromROSMsg also accepts, goes to
 *     b2r_ingest_pointcloud2_rows.
 *   - b2r_ingest_pointcloud2 is synchronous with respect to `data`: when it returns, the copy out of the caller's buffer has
 *     finished (pageable or pinned) and the buffer may be reused. */
typedef struct b2r_point_layout {
  uint32_t point_step;         /* PointCloud2.point_step */
  uint32_t off_x, off_y, off_z;/* byte offsets of the FLOAT32 fields "x", "y", "z" */
  uint32_t off_intensity;      /* byte offset of "intensity", 0xffffffff = absent (intensity 0) */
  uint32_t intensity_datatype; /* sensor_msgs/PointField datatype of "intensity" (1 INT8 2 UINT8 3 INT16 4 UINT16 5 INT32 6 UINT32 7 FLOAT32
                                  8 FLOAT64): validated against point_step, but only 7 is read; every other type gives intensity 0 */
  uint32_t is_bigendian;       /* PointCloud2.is_bigendian */
} b2r_point_layout;
int b2r_ingest_pointcloud2(b2r_handle* h, const void* data, size_t n_points, const b2r_point_layout* layout, const void** d_points);
/* the same unpacking for an organized message whose rows may be padded: `data` holds height * row_step bytes (all of them are
 * copied), and record i = r * width + c (row-major, width * height records, NaN records included) is read at byte
 * r * row_step + c * point_step.  Field mapping, byte order, intensity rules and the lifetime of *d_points are
 * b2r_ingest_pointcloud2's.  B2R_EINVAL when row_step < width * point_step (for a non-empty message); width * height = 0 succeeds
 * with *d_points = NULL. */
int b2r_ingest_pointcloud2_rows(b2r_handle* h, const void* data, uint32_t width, uint32_t height, uint32_t row_step,
                                const b2r_point_layout* layout, const void** d_points);
/* header of a binary PCD file (the cloud.pcd KeyFrame::save writes with pcl::io::savePCDFileBinary, keyframe.cpp:57): x, y, z must be
 * F 4 COUNT 1 (else B2R_EINVAL); "intensity" is reported (datatype 7) only when it is F 4 COUNT 1, otherwise off_intensity = 0xffffffff.
 * DATA ascii / binary_compressed: B2R_EUNSUPPORTED.  Without POINTS the count is WIDTH * HEIGHT. */
int b2r_pcd_read_header(const char* path, b2r_point_layout* layout, size_t* n_points, size_t* data_offset);
/* header parse + fread of the body straight into engine-owned pinned memory + H2D + device unpack (field mapping as above) */
int b2r_ingest_pcd(b2r_handle* h, const char* path, const void** d_points, size_t* n_points);

/* ---- host mirrors of the two callers (logic identical to the reference; only the handle is ours) ---------------- */
typedef struct b2r_odometry b2r_odometry;
typedef struct b2r_odometry_params {
  double keyframe_delta_trans;  /* scan_matching_odometry_nodelet.cpp:74 (0.25; 1.0 in hdl_graph_slam.launch:63) */
  double keyframe_delta_angle;  /* :75 */
  double keyframe_delta_time;   /* :76 */
  int32_t transform_thresholding; /* :79 */
  double max_acceptable_trans;  /* :80 */
  double max_acceptable_angle;  /* :81 */
  int32_t publish_status;       /* 1: also compute fitness + inlier fraction each frame (status topic subscribed, :298-335) */
  int32_t downsample_method;    /* "downsample_method" :83-103: B2R_DOWNSAMPLE_* (0 = NONE, the cloud as given; unknown values pass
                                   through).  Every shipped launch file sets NONE (the prefilter has already downsampled). */
  float downsample_resolution;  /* "downsample_resolution" :84 (0.1): leaf of VOXELGRID / APPROX_VOXELGRID */
} b2r_odometry_params;
typedef struct b2r_odometry_status {
  float odom[16];           /* keyframe_pose * trans, column-major (return value of matching(), :165-262) */
  float trans[16];          /* getFinalTransformation() of this frame */
  int32_t converged;
  int32_t iterations;
  int32_t keyframe_updated;
  int32_t frame_rejected;   /* not converged or thresholded (:214-233) */
  double matching_error;    /* getFitnessScore()          (status only) */
  float inlier_fraction;    /* (status only) */
  int32_t reserved;
} b2r_odometry_status;
/* p == NULL: the code defaults above, downsample NONE.  B2R_EINVAL when downsample_method is VOXELGRID and downsample_resolution is
 * not positive, or APPROX_VOXELGRID and it is not finite and positive (the checks of b2r_voxelgrid / b2r_approximate_voxelgrid). */
int b2r_odometry_create(b2r_handle* registration, const b2r_odometry_params* p, b2r_odometry** out);
void b2r_odometry_destroy(b2r_odometry* o);
/* ScanMatchingOdometryNodelet::matching(stamp, cloud) (apps/scan_matching_odometry_nodelet.cpp:165-262);
 * msf_delta may be NULL (identity).  With downsample_method VOXELGRID / APPROX_VOXELGRID the cloud is filtered first, on the device
 * and in buffers the odometry owns (never the handle's voxel-grid buffer, so b2r_prefilter's d_out may be passed on the same handle),
 * exactly as b2r_voxelgrid_device / b2r_approximate_voxelgrid_device would (including the "leaf too small" pass-through); the
 * filtered cloud is what is registered, becomes the keyframe, and is the denominator of inlier_fraction. */
int b2r_odometry_matching(b2r_odometry* o, double stamp, const void* cloud, size_t n, size_t stride_bytes, const float* msf_delta,
                          b2r_odometry_status* out);

/* same, for a cloud already resident in device memory (the HBM-resident measurement of bench.py) */
int b2r_odometry_matching_device(b2r_odometry* o, double stamp, const void* d_cloud, size_t n, size_t stride_bytes, const float* msf_delta,
                                 b2r_odometry_status* out);

/* matching(stamp, cloud) with the stamp as ros::Time holds it (sec, nsec) and the status chosen per call (want_status: status_pub has
 * subscribers, :299; the first frame computes none whatever it says).  device != 0: `cloud` is a device pointer, e.g. an ingest buffer of
 * the odometry's handle.  The keyframe test's delta_time is roscpp's exact (stamp - keyframe_stamp).toSec() (:243): seconds and
 * nanoseconds subtracted as integers, nanoseconds normalised into [0, 1e9), then sec + 1e-9 * nsec; the double entry points subtract
 * two doubles instead, which decides differently when the true difference lies within a few hundred nanoseconds of
 * keyframe_delta_time.  One odometry may mix both forms: the keyframe keeps the form of the call that made it, roscpp's rule applies
 * when both stamps are sec / nsec, and otherwise the doubles are subtracted, a sec / nsec stamp taken as ros::Time::toSec(). */
int b2r_odometry_matching_ros(b2r_odometry* o, uint32_t sec, uint32_t nsec, const void* cloud, size_t n, size_t stride_bytes, int device,
                              const float* msf_delta, int want_status, b2r_odometry_status* out);

/* aligned_points of the last matching call (:254-259): pcl::transformPointCloud(*cloud, *aligned, odom) of the RAW cloud that call was
 * given (before the odometry's downsample), computed on the device from the records matching left there (no second upload) and written
 * to `out` as n records of stride_bytes.  Each record is copied, then x, y, z become ((m0 x + m1 y) + m2 z) + m3 under odom (as
 * b2r_get_aligned) and the float at byte 12 becomes 1.0f (when stride_bytes >= 16).  is_dense == 0 (the input cloud's is_dense): a
 * record with a non-finite x, y or z stays as it was (PCL 1.10's non-dense branch).  B2R_ESTATE unless the last matching call
 * succeeded on an accepted frame (not the first, not rejected, :214-233 return before :254); B2R_EINVAL when n or stride_bytes
 * differs from that call's.  A device cloud given to that call is read again here: keep it unchanged until this returns. */
int b2r_odometry_aligned(b2r_odometry* o, int is_dense, void* out, size_t n, size_t stride_bytes);

/* announce the cloud of the NEXT matching() call: the following matching() prefetches it (b2r_prefetch_source) right after it
 * has set its own source, so the next frame's preprocessing overlaps this frame's align.  device != 0: device pointer.
 * With a downsample, the prefetch also filters the announced cloud on the prefetch stream; the next matching() uses that result only
 * if it is given the same raw cloud (pointer, n, stride and, for a host cloud, the same content), and filters afresh otherwise. */
int b2r_odometry_prefetch(b2r_odometry* o, const void* cloud, size_t n, size_t stride_bytes, int device);

/* LoopDetector::matching (include/hdl_graph_slam/loop_detector.hpp:117-171): align every candidate against the new
 * keyframe, keep the best converged fitness.  guesses: n_candidates x 16 floats, column-major (already z-zeroed by the
 * caller as in :141-142).  results (n_candidates, may be NULL) receives every candidate's record.
 * *best = index of the best candidate or -1 ("loop not found"). */
int b2r_loop_matching(b2r_handle* h, const void* new_keyframe, size_t n_new, size_t stride_bytes, const void* const* candidates,
                      const size_t* n_candidates_pts, size_t n_candidates, const float* guesses, double fitness_score_max_range,
                      double fitness_score_thresh, b2r_result* results, int32_t* best);


/* ---- batched, device-resident registration (north_star's multi-GPU split; loop_detector.hpp:135-154) --------------------
 * A b2r_batch lives on ONE GPU (cfg->device_id).  Keyframe clouds are registered once (b2r_batch_add_cloud: upload, search
 * structure, GICP covariances) and named by id; b2r_batch_align runs MANY (source, target, guess) registrations at once.
 * GICP config: one pair of kernel launches per LM iteration covers every pair still in flight, the LM step (6x6 solve, se3_exp,
 * rho test, convergence) runs on the device, and the host reads the 80-byte records back once per batch.  Results are bitwise
 * identical to running each pair alone through b2r_set_target / b2r_set_source / b2r_align (+ b2r_fitness-equivalent score).
 * NDT config (B2R_METHOD_NDT, the factory's default NDT_OMP): a cloud used as a target gets its voxel map at the first call
 * that uses it (a cloud added from device memory at the first call that names it); every pair runs the single handle's
 * Newton / More-Thuente driver and each round of derivative passes covers every pair in flight (one host wait per round).
 * Pose, flag, iteration count and fitness are bitwise those of b2r_set_target / b2r_set_source / b2r_align / b2r_fitness on
 * one NDT handle; b2r_batch_last_rounds counts batched rounds and, per pair, derivative / Hessian passes.
 * pcl GICP config (B2R_METHOD_GICP_PCL, and pclomp GICP, B2R_METHOD_GICP_OMP): every pair runs the single handle's computeTransformation / BFGS driver and each round has at
 * most one batched correspondence launch and one batched cost launch (one host wait per round); the records are bitwise the single
 * handle's, and b2r_batch_last_rounds counts, per pair, correspondence and cost passes.
 *
 * Host buffers passed to b2r_batch_add_cloud may be pageable (copied before the call returns) or pinned (DMA'd in place:
 * keep them unmodified until the next b2r_batch_align / b2r_batch_loop_detect / b2r_batch_synchronize returns). */
typedef struct b2r_batch b2r_batch;
typedef struct b2r_pair {
  int32_t source;  /* cloud id: setInputSource(candidate->cloud)   loop_detector.hpp:136 */
  int32_t target;  /* cloud id: setInputTarget(new_keyframe->cloud) loop_detector.hpp:122 */
  float guess[16]; /* column-major initial guess                     loop_detector.hpp:139-143 */
} b2r_pair;
int b2r_batch_create(const b2r_config* cfg, b2r_batch** out);
void b2r_batch_destroy(b2r_batch* b);
/* the engine handle behind the batch (telemetry / stream access: b2r_get_stats, b2r_set_profiling, b2r_get_stream) */
int b2r_batch_get_engine(b2r_batch* b, b2r_handle** out);
int b2r_batch_add_cloud(b2r_batch* b, const void* points, size_t n, size_t stride_bytes, int32_t* cloud_id);
int b2r_batch_add_cloud_device(b2r_batch* b, const void* d_points, size_t n, size_t stride_bytes, int32_t* cloud_id);
int b2r_batch_remove_cloud(b2r_batch* b, int32_t cloud_id);
int b2r_batch_cloud_count(const b2r_batch* b);
int b2r_batch_synchronize(b2r_batch* b);
/* align every pair; want_fitness != 0 also evaluates getFitnessScore(fitness_max_range) at each final pose (loop_detector.hpp:146;
 * max_range is compared with the SQUARED distance as in information_matrix_calculator.cpp:69), else fitness = NaN */
int b2r_batch_align(b2r_batch* b, const b2r_pair* pairs, size_t n_pairs, int want_fitness, double fitness_max_range, b2r_result* out);
/* replaces InformationMatrixCalculator::calc_fitness_score(cloud1, cloud2, relpose, max_range)
 * (src/hdl_graph_slam/information_matrix_calculator.cpp:49-80; called per odometry edge and per accepted loop,
 * apps/hdl_graph_slam_nodelet.cpp:235,569) for MANY edges at once on the keyframes' cached search structures:
 * pairs[i].target = cloud1 (the tree), pairs[i].source = cloud2 (transformed), pairs[i].guess = relpose.cast<float>() column-major.
 * scores[i] = mean squared NN distance over the neighbours with d2 <= max_range, DBL_MAX when there is none. */
int b2r_batch_calc_fitness_score(b2r_batch* b, const b2r_pair* pairs, size_t n_pairs, double max_range, double* scores);
/* MapCloudGenerator::generate over clouds of the b2r_batch keyframe cache: keyframe k = cloud ids[k] at poses[16k..16k+16)
 * (KeyFrameSnapshot::pose cast to float, column-major).  Same result as b2r_map_cloud_generate on the same clouds and poses,
 * with no point uploaded.  out_host (capacity out_capacity records of out_stride_bytes, may be NULL) and/or *d_out (engine-owned,
 * valid until the next map or prefilter call on the batch's engine handle, may be NULL; NULL when *n_out = 0).
 * Ids may come in any order and repeat; an unknown or removed id is B2R_EINVAL.  Returns 1 with *n_out = 0 when n_keyframes = 0.
 * resolution > 0 reads the clouds' search structures and builds the missing ones (the build the next b2r_batch_align would do; a
 * device-added cloud must be valid until then, as for an align).  resolution <= 0 copies the records the batch uploaded itself:
 * every cloud must come from b2r_batch_add_cloud with stride_bytes == out_stride_bytes, else B2R_EINVAL naming the id.
 * B2R_EUNSUPPORTED beyond 21 octree levels, as b2r_map_cloud_generate; the batch stays usable. */
int b2r_batch_map_cloud_generate(b2r_batch* b, const int32_t* ids, const float* poses, size_t n_keyframes, double resolution,
                                 size_t out_stride_bytes, void* out_host, size_t out_capacity, const void** d_out, size_t* n_out);
/* the rest of InformationMatrixCalculator::calc_information_matrix (information_matrix_calculator.cpp:25-47, weight() at
 * information_matrix_calculator.hpp:39-42): fitness score -> diagonal of the 6x6 information matrix (x,y,z, then rotation).
 * Defaults of the reference's rosparams: b2r_information_params_default. */
typedef struct b2r_information_params {
  int32_t use_const_inf_matrix; /* false */
  int32_t reserved;
  double const_stddev_x;        /* 0.5  */
  double const_stddev_q;        /* 0.1  */
  double var_gain_a;            /* 20.0 */
  double min_stddev_x;          /* 0.1  */
  double max_stddev_x;          /* 5.0  */
  double min_stddev_q;          /* 0.05 */
  double max_stddev_q;          /* 0.2  */
  double fitness_score_thresh;  /* 0.5 (information_matrix_calculator.cpp:21; 2.5 in the header's template load(), :31) */
} b2r_information_params;
int b2r_information_params_default(b2r_information_params* p);
int b2r_information_from_fitness(const b2r_information_params* p, double fitness_score, double inf_diag[6]);
/* rounds (launch pairs) and pair-rounds (sum over rounds of the pairs in flight) of the last batch: the work the roofline divides by */
int b2r_batch_last_rounds(const b2r_batch* b, uint64_t* rounds, uint64_t* pair_rounds);
/* the selection of LoopDetector::matching over one group's records (loop_detector.hpp:147,160-163): index of the best converged
 * candidate (a later candidate with an EQUAL score wins) or -1 when nothing converged or the best score exceeds the threshold */
int b2r_loop_argmin(const b2r_result* results, size_t n, double fitness_score_thresh, int32_t* best);

/* ---- LoopDetector's gating around the batch (include/hdl_graph_slam/loop_detector.hpp:39-46,57-68,81-109,137-142): host logic only ----
 * detect() walks the new keyframes one by one: find_candidates -> matching -> (loop found) last_edge_accum_distance = accum_distance.
 * The only coupling between two new keyframes is that scalar, so the walk splits into  plan  (every new keyframe's candidates and
 * guesses under the gate as it stands when the walk starts),  b2r_batch_loop_detect  (all pairs at once, sharded over the GPUs) and
 * replay  (the sequential walk on the results: a keyframe gated out at ITS turn reports no loop, an accepted loop moves the distance).
 * The outcome equals the reference's sequential detect(). */
typedef struct b2r_loop_params {
  double distance_thresh;          /* loop_detector.hpp:40  (5.0)  estimated xy distance between the two keyframes must not exceed it */
  double accum_distance_thresh;    /* :41 (8.0)  travelled distance between the two keyframes must reach it */
  double min_edge_interval;        /* :42 (5.0)  "distance_from_last_edge_thresh": travelled distance since the last registered loop edge */
  double fitness_score_max_range;  /* :44 (DBL_MAX) */
  double fitness_score_thresh;     /* :45 (0.5) */
} b2r_loop_params;
typedef struct b2r_keyframe_state {
  double accum_distance;           /* KeyFrame::accum_distance */
  double estimate[16];             /* KeyFrame::node->estimate().matrix(), column-major */
} b2r_keyframe_state;
int b2r_loop_params_default(b2r_loop_params* p);
/* LoopDetector::find_candidates (:81-109): indices into `keyframes` in their order; none if the new keyframe is closer than
 * min_edge_interval to the last registered loop edge.  *n_candidates = the number found (an error if it exceeds `capacity`). */
int b2r_loop_find_candidates(const b2r_loop_params* p, const b2r_keyframe_state* keyframes, size_t n_keyframes, const b2r_keyframe_state* new_keyframe,
                             double last_edge_accum_distance, int32_t* candidates, size_t capacity, size_t* n_candidates);
/* the initial guess of LoopDetector::matching (:137-142): rotations re-normalised through a quaternion, new^-1 * candidate,
 * cast to float, z translation zeroed; column-major in and out */
int b2r_loop_guess(const double* new_keyframe_estimate, const double* candidate_estimate, float* guess);
/* plan of one detect() walk: group g = new_keyframes[g]; pairs [group_first[g], group_first[g+1]) are its candidates
 * (candidate_index = index into `keyframes`, guesses = 16 floats per pair); group_first has n_new + 1 entries.  The caller turns
 * (candidate_index, g) into cloud ids of a b2r_batch and hands pairs + group_first to b2r_batch_loop_detect. */
int b2r_loop_detect_plan(const b2r_loop_params* p, const b2r_keyframe_state* keyframes, size_t n_keyframes, const b2r_keyframe_state* new_keyframes,
                         size_t n_new, double last_edge_accum_distance, int32_t* candidate_index, float* guesses, size_t capacity,
                         int64_t* group_first, size_t* n_pairs);
/* the sequential walk on the batch's answers: best[g] = b2r_batch_loop_detect's index inside group g or -1;
 * planned_last_edge_accum_distance = the value the plan was made with; *last_edge_accum_distance is read and updated (:166);
 * accepted[g] = index inside group g of the registered loop's start keyframe, or -1 */
int b2r_loop_detect_replay(const b2r_loop_params* p, const b2r_keyframe_state* new_keyframes, size_t n_new, const int64_t* group_first, const int32_t* best,
                           double planned_last_edge_accum_distance, double* last_edge_accum_distance, int32_t* accepted);

/* multi-GPU: one process per GPU; rank 0 creates the id, every rank receives it through the launcher's own channel
 * (bench.py: torch.distributed broadcast) and joins.  The library links NCCL itself. */
int b2r_nccl_unique_id(void* out128, size_t capacity);
int b2r_batch_comm_init(b2r_batch* b, const void* unique_id128, int rank, int world);
/* contiguous block of groups owned by `rank` (neighbouring groups share candidate keyframes: each is built on one GPU only) */
int b2r_shard_range(size_t n_groups, int world, int rank, size_t* g0, size_t* g1);
/* LoopDetector::matching for n_groups new keyframes at once.  pairs[group_first[g] .. group_first[g+1]) are the candidates of
 * group g in the reference's order.  Every rank passes the SAME pair list; cloud ids are only read for the rank's own groups
 * (b2r_shard_range).  Each rank aligns its share, ONE ncclAllGather moves the 80-byte records (padded to the largest share),
 * then every rank holds all_results[n_pairs] and best[n_groups] (index inside the group, or -1). */
int b2r_batch_loop_detect(b2r_batch* b, const b2r_pair* pairs, size_t n_pairs, const int64_t* group_first, size_t n_groups,
                          double fitness_score_max_range, double fitness_score_thresh, b2r_result* all_results, int32_t* best);

#ifdef __cplusplus
}
#endif
#endif
