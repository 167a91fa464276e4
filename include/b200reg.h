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
 * "NDT_OMP"/"B200_NDT" -> NDT engine.  ICP / GICP / GICP_OMP / NDT(pcl) / FAST_VGICP[_CUDA] are not re-created:
 * returns B2R_EUNSUPPORTED so the caller keeps the reference's own branch. */
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
 * the current source (points, grid, covariances) becomes the target without re-upload or recomputation. */
int b2r_promote_source_to_target(b2r_handle* h);

/* replaces registration->align(*aligned, guess) + hasConverged() + getFinalTransformation()
 * (scan_matching_odometry_nodelet.cpp:210,214,220; loop_detector.hpp:143,147,153). */
int b2r_align(b2r_handle* h, const float guess[16], b2r_result* out);

/* the `aligned` output cloud of align(): source transformed by the final pose.  Writes x,y,z (and 1.0f at offset 12 when
 * stride_bytes >= 16) of n records; other bytes are left untouched. */
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
/* one compute_error at pose T with the correspondences of the last linearisation */
int b2r_gicp_error_at(b2r_handle* h, const double T[16], double* err);
/* NDT voxel table of the target: returns count through *n_voxels; arrays may be NULL.  keys ascending. */
int b2r_ndt_get_voxels(b2r_handle* h, size_t capacity, size_t* n_voxels, int64_t* keys, int32_t* npts, double* mean, double* icov,
                       int32_t min_b[3], int32_t div_b[3]);
/* one computeDerivatives pass at p = (tx,ty,tz,rx,ry,rz): score, g[6], H[36] row-major, number of (point,cell) pairs */
int b2r_ndt_derivatives_at(b2r_handle* h, const double p[6], double* score, double* g, double* H, uint64_t* n_pairs);

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
  int32_t downsample_method;      /* "downsample_method" VOXELGRID                          :51                          */
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

/* replaces MapCloudGenerator::generate(keyframes, resolution) (src/hdl_graph_slam/map_cloud_generator.cpp:13-51; called at
 * apps/hdl_graph_slam_nodelet.cpp:528,989): every keyframe cloud transformed by its optimised pose (float32), all concatenated;
 * resolution <= 0 returns that cloud (intensity kept), otherwise the centres of the occupied voxels of a
 * pcl::octree::OctreePointCloud(resolution) — the same SET of centres as PCL's lattice (anchored at the first finite point),
 * emitted in ascending key order instead of octree traversal order; x,y,z,1 with intensity 0.
 * Returns 1 with *n_out = 0 when there is no keyframe ("warning: keyframes empty!!").  out: capacity out_capacity records. */
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
 * src/hdl_graph_slam/keyframe.cpp:141.  *d_points is an engine-owned device buffer (valid until the next ingest call on this
 * handle) for b2r_set_source_device / b2r_set_target_device / b2r_prefilter(device_input = 1) / b2r_batch_add_cloud_device. */
typedef struct b2r_point_layout {
  uint32_t point_step;         /* PointCloud2.point_step */
  uint32_t off_x, off_y, off_z;/* byte offsets of the FLOAT32 fields "x", "y", "z" */
  uint32_t off_intensity;      /* byte offset of "intensity", 0xffffffff = absent (intensity 0) */
  uint32_t intensity_datatype; /* sensor_msgs/PointField datatype of "intensity": 1 INT8 2 UINT8 3 INT16 4 UINT16 5 INT32 6 UINT32 7 FLOAT32 8 FLOAT64 */
  uint32_t is_bigendian;       /* PointCloud2.is_bigendian */
} b2r_point_layout;
int b2r_ingest_pointcloud2(b2r_handle* h, const void* data, size_t n_points, const b2r_point_layout* layout, const void** d_points);
/* header of a binary PCD file (the cloud.pcd KeyFrame::save writes with pcl::io::savePCDFileBinary, keyframe.cpp:57) */
int b2r_pcd_read_header(const char* path, b2r_point_layout* layout, size_t* n_points, size_t* data_offset);
/* header parse + fread of the body straight into pinned memory + H2D + device unpack */
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
int b2r_odometry_create(b2r_handle* registration, const b2r_odometry_params* p, b2r_odometry** out);
void b2r_odometry_destroy(b2r_odometry* o);
/* ScanMatchingOdometryNodelet::matching(stamp, cloud) (apps/scan_matching_odometry_nodelet.cpp:165-262);
 * msf_delta may be NULL (identity). */
int b2r_odometry_matching(b2r_odometry* o, double stamp, const void* cloud, size_t n, size_t stride_bytes, const float* msf_delta,
                          b2r_odometry_status* out);

/* same, for a cloud already resident in device memory (the HBM-resident measurement of bench.py) */
int b2r_odometry_matching_device(b2r_odometry* o, double stamp, const void* d_cloud, size_t n, size_t stride_bytes, const float* msf_delta,
                                 b2r_odometry_status* out);

/* announce the cloud of the NEXT matching() call: the following matching() prefetches it (b2r_prefetch_source) right after it
 * has set its own source, so the next frame's preprocessing overlaps this frame's align.  device != 0: device pointer */
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
 * structure, GICP covariances) and named by id; b2r_batch_align runs MANY (source, target, guess) registrations at once:
 * one pair of kernel launches per LM iteration covers every pair still in flight, the LM step (6x6 solve, se3_exp, rho test,
 * convergence) runs on the device, and the host reads the 80-byte records back once per batch.  Results are bitwise identical
 * to running each pair alone through b2r_set_target / b2r_set_source / b2r_align (+ b2r_fitness-equivalent score).
 * GICP engine only (the reference's loop closure uses FAST_GICP: launch/hdl_graph_slam.launch:127).
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
