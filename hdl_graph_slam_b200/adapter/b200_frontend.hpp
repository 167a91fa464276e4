// b200_frontend.hpp — drop-in replacements for the point work of the two front-end nodelets of koide3/hdl_graph_slam that run on
// every frame, each served by its own engine handle of libb200reg.so:
//   PrefilteringNodelet    apps/prefiltering_nodelet.cpp:50-243       -> B200Prefilter      (b2r_prefilter, row f-2)
//   FloorDetectionNodelet  apps/floor_detection_nodelet.cpp:56-238    -> B200FloorDetector  (b2r_floor_detect, row f-5)
// Both also take a sensor_msgs::PointCloud2 as it arrives and unpack it on the device (b2r_ingest_pointcloud2 /
// b2r_ingest_pointcloud2_rows, row f-4), so the raw scan is never converted on the host.  The nodelets keep their subscriptions,
// publishers, the IMU queue, the tf lookup and the colored_points debug cloud.  INTEGRATION.md §4c shows the two nodelet patches.
// Compiled only where ROS, PCL, Eigen and boost exist; tests/test_frontend_syntax.py checks it against the test-only stand-ins
// adapter/pcl_shim.hpp, adapter/backend_shim.hpp and adapter/frontend_shim.hpp.
//
// Threads: an instance is used by one thread at a time, as each nodelet's callback queue does (one callback at a time per
// nodelet).  Distinct instances own distinct handles and may run concurrently.
#pragma once
#include <b200reg.h>
#include <cstdint>
#include <iostream>
#include <memory>
#include <stdexcept>
#include <string>

namespace hdl_graph_slam {

namespace b200_frontend {

inline void check(int rc) {
  if (rc < 0) throw std::runtime_error(std::string("b200reg: ") + b2r_last_error());
}

// one engine handle on the device the rosparam "reg_device_id" names (default 0, as B200KeyframeCache reads it)
inline b2r_handle* create_handle(ros::NodeHandle& private_nh) {
  b2r_config cfg;
  check(b2r_config_default(&cfg, B2R_METHOD_GICP));
  cfg.device_id = private_nh.param<int>("reg_device_id", 0);
  b2r_handle* h = nullptr;
  check(b2r_create(&cfg, &h));
  return h;
}

// the fields pcl::fromROSMsg maps into pcl::PointXYZI: the first field of each name whose datatype and count match the point's
// (FLOAT32, count 1 or 0).  Without x, y and z there is nothing to unpack: std::invalid_argument, and the caller converts with
// fromROSMsg instead.  An intensity field of another type is left unmapped (intensity 0), as PCL leaves it.
inline b2r_point_layout pointcloud2_layout(const sensor_msgs::PointCloud2& msg) {
  b2r_point_layout L;
  L.point_step = msg.point_step;
  L.off_x = L.off_y = L.off_z = 0;
  L.off_intensity = 0xffffffffu;
  L.intensity_datatype = sensor_msgs::PointField::FLOAT32;
  L.is_bigendian = msg.is_bigendian ? 1u : 0u;
  const char* names[4] = {"x", "y", "z", "intensity"};
  uint32_t* offsets[4] = {&L.off_x, &L.off_y, &L.off_z, &L.off_intensity};
  bool found[4] = {false, false, false, false};
  for (int k = 0; k < 4; k++)
    for (const auto& f : msg.fields)
      if (f.name == names[k] && f.datatype == sensor_msgs::PointField::FLOAT32 && (f.count == 1 || f.count == 0)) {
        *offsets[k] = f.offset;
        found[k] = true;
        break;
      }
  if (!found[0] || !found[1] || !found[2]) throw std::invalid_argument("b200reg: the PointCloud2 has no FLOAT32 x, y and z fields");
  return L;
}

// msg.data -> width * height PointXYZI records in engine-owned device memory (NaN records of organized clouds included, as
// fromROSMsg keeps them); nullptr with *n = 0 for an empty message, whatever its fields.  Padded rows go to
// b2r_ingest_pointcloud2_rows.
inline const void* ingest_pointcloud2(b2r_handle* h, const sensor_msgs::PointCloud2& msg, size_t* n) {
  *n = (size_t)msg.width * msg.height;
  if (*n == 0) return nullptr;
  const b2r_point_layout L = pointcloud2_layout(msg);
  if (msg.data.size() < (size_t)msg.height * msg.row_step) throw std::invalid_argument("b200reg: PointCloud2 data is shorter than height * row_step");
  const void* d = nullptr;
  if ((uint64_t)msg.row_step == (uint64_t)msg.width * msg.point_step)
    check(b2r_ingest_pointcloud2(h, msg.data.data(), *n, &L, &d));
  else
    check(b2r_ingest_pointcloud2_rows(h, msg.data.data(), msg.width, msg.height, msg.row_step, &L, &d));
  return d;
}

}  // namespace b200_frontend

// PrefilteringNodelet::initialize_params + cloud_callback (prefiltering_nodelet.cpp:50-180) as one b2r_prefilter call:
// deskewing -> [base_link transform] -> distance filter -> downsample -> outlier removal, the cloud resident on the device between
// the stages.
class B200Prefilter {
public:
  using PointT = pcl::PointXYZI;

  // Reads what initialize_params reads (:50-99), with its console lines.  The NodeHandle is kept: "scan_period" is read again at
  // every call that deskews, as deskewing does (:229).  Throws std::runtime_error with the engine's message when no handle can be
  // created on "reg_device_id", so the nodelet can keep its reference filters.
  explicit B200Prefilter(ros::NodeHandle& private_nh) : private_nh_(private_nh) {
    b2r_prefilter_params_default(&params_);
    const std::string downsample_method = private_nh.param<std::string>("downsample_method", "VOXELGRID");
    const double downsample_resolution = private_nh.param<double>("downsample_resolution", 0.1);
    params_.downsample_resolution = static_cast<float>(downsample_resolution);  // setLeafSize takes floats (:57, :62)
    if (downsample_method == "VOXELGRID") {
      std::cout << "downsample: VOXELGRID " << downsample_resolution << std::endl;
      params_.downsample_method = B2R_DOWNSAMPLE_VOXELGRID;
    } else if (downsample_method == "APPROX_VOXELGRID") {
      std::cout << "downsample: APPROX_VOXELGRID " << downsample_resolution << std::endl;
      params_.downsample_method = B2R_DOWNSAMPLE_APPROX_VOXELGRID;
    } else {
      if (downsample_method != "NONE") {
        std::cerr << "warning: unknown downsampling type (" << downsample_method << ")" << std::endl;
        std::cerr << "       : use passthrough filter" << std::endl;
      }
      std::cout << "downsample: NONE" << std::endl;
      params_.downsample_method = B2R_DOWNSAMPLE_NONE;
    }

    const std::string outlier_removal_method = private_nh.param<std::string>("outlier_removal_method", "STATISTICAL");
    if (outlier_removal_method == "STATISTICAL") {
      params_.statistical_mean_k = private_nh.param<int>("statistical_mean_k", 20);
      params_.statistical_stddev = private_nh.param<double>("statistical_stddev", 1.0);
      std::cout << "outlier_removal: STATISTICAL " << params_.statistical_mean_k << " - " << params_.statistical_stddev << std::endl;
      params_.outlier_removal_method = B2R_OUTLIER_STATISTICAL;
    } else if (outlier_removal_method == "RADIUS") {
      params_.radius_radius = private_nh.param<double>("radius_radius", 0.8);
      params_.radius_min_neighbors = private_nh.param<int>("radius_min_neighbors", 2);
      std::cout << "outlier_removal: RADIUS " << params_.radius_radius << " - " << params_.radius_min_neighbors << std::endl;
      params_.outlier_removal_method = B2R_OUTLIER_RADIUS;
    } else {
      std::cout << "outlier_removal: NONE" << std::endl;
      params_.outlier_removal_method = B2R_OUTLIER_NONE;
    }

    // "use_distance_filter" is read at :95 but cloud_callback applies the distance filter unconditionally (:131)
    params_.use_distance_filter = 1;
    params_.distance_near_thresh = private_nh.param<double>("distance_near_thresh", 1.0);
    params_.distance_far_thresh = private_nh.param<double>("distance_far_thresh", 100.0);
    base_link_frame_ = private_nh.param<std::string>("base_link_frame", "");
    h_ = b200_frontend::create_handle(private_nh);
  }
  ~B200Prefilter() { b2r_destroy(h_); }
  B200Prefilter(const B200Prefilter&) = delete;
  B200Prefilter& operator=(const B200Prefilter&) = delete;

  // cloud_callback's point work on one scan.
  //   imu_angular_velocity: nullptr when the IMU queue is empty (deskewing returns the cloud, :184-186); otherwise the
  //                         angular_velocity of the IMU message deskewing picks (:207-217), as the message gives it (the engine
  //                         negates it, :219-220).
  //   to_base_link:         nullptr when base_link_frame is empty; otherwise pcl_ros::transformAsMatrix of the transform the
  //                         nodelet looked up (:120-125).
  // Returns nullptr for an empty input (cloud_callback returns without publishing, :108-110).  Otherwise the filtered cloud with
  // the input's header (:146, :159, :177), its frame_id replaced by base_link_frame after a base_link transform (:126),
  // width = size and height = 1 (:173-174).
  // is_dense (UPSTREAM-RECALL, PCL 1.10, not checkable here): the distance filter sets false (:175); pcl::VoxelGrid sets true;
  // pcl::ApproximateVoxelGrid sets false; the outlier filters copy their input's flag.  So the output is dense exactly when
  // downsample_method is VOXELGRID (a leaf too small for int32 voxel indices makes VoxelGrid copy its input instead, which this
  // rule does not follow).
  pcl::PointCloud<PointT>::ConstPtr filter(const pcl::PointCloud<PointT>::ConstPtr& cloud, const Eigen::Vector3f* imu_angular_velocity,
                                           const Eigen::Matrix4f* to_base_link) {
    if (!cloud || cloud->points.empty()) return nullptr;
    return run(cloud->points.data(), cloud->points.size(), 0, cloud->header, imu_angular_velocity, to_base_link);
  }

  // The same on a message as it arrives: the message is unpacked on the device (fields found by name as fromROSMsg finds them) and
  // filtered there; the header comes from msg.header.  Deskewing's i / size runs over all width * height records, NaN records of
  // an organized cloud included, as it does on fromROSMsg's cloud.  A non-empty message without FLOAT32 x, y and z throws
  // std::invalid_argument: convert it with fromROSMsg and call the first overload.
  pcl::PointCloud<PointT>::ConstPtr filter(const sensor_msgs::PointCloud2& msg, const Eigen::Vector3f* imu_angular_velocity,
                                           const Eigen::Matrix4f* to_base_link) {
    size_t n = 0;
    const void* d = b200_frontend::ingest_pointcloud2(h_, msg, &n);
    if (n == 0) return nullptr;
    pcl::PCLHeader header;
    pcl_conversions::toPCL(msg.header, header);
    return run(d, n, 1, header, imu_angular_velocity, to_base_link);
  }

  const std::string& base_link_frame() const { return base_link_frame_; }
  // the parameters the next call starts from (deskewing, scan_period and the transform are filled per call)
  const b2r_prefilter_params& params() const { return params_; }

private:
  pcl::PointCloud<PointT>::ConstPtr run(const void* points, size_t n, int device_input, const pcl::PCLHeader& header,
                                        const Eigen::Vector3f* imu_angular_velocity, const Eigen::Matrix4f* to_base_link) {
    b2r_prefilter_params p = params_;
    p.deskewing = imu_angular_velocity ? 1 : 0;
    if (imu_angular_velocity) {
      p.scan_period = private_nh_.param<double>("scan_period", 0.1);
      for (int i = 0; i < 3; i++) p.angular_velocity[i] = (*imu_angular_velocity)[i];
    }
    p.use_base_link_transform = to_base_link ? 1 : 0;
    if (to_base_link)
      for (int i = 0; i < 16; i++) p.base_link_transform[i] = to_base_link->data()[i];  // both column-major
    pcl::PointCloud<PointT>::Ptr out(new pcl::PointCloud<PointT>());
    out->points.resize(n);
    size_t m = 0;
    b200_frontend::check(b2r_prefilter(h_, points, n, sizeof(PointT), device_input, &p, out->points.data(), nullptr, &m));
    out->points.resize(m);
    out->header = header;
    if (to_base_link) out->header.frame_id = base_link_frame_;
    out->width = static_cast<uint32_t>(m);
    out->height = 1;
    out->is_dense = params_.downsample_method == B2R_DOWNSAMPLE_VOXELGRID;
    return out;
  }

  ros::NodeHandle private_nh_;
  b2r_prefilter_params params_;
  std::string base_link_frame_;
  b2r_handle* h_ = nullptr;
};

// FloorDetectionNodelet::initialize_params + detect (floor_detection_nodelet.cpp:56-63, :110-180) as one b2r_floor_detect call.
class B200FloorDetector {
public:
  using PointT = pcl::PointXYZI;

  // Reads what initialize_params reads (:57-63).  Throws std::runtime_error with the engine's message when no handle can be
  // created on "reg_device_id".
  explicit B200FloorDetector(ros::NodeHandle& private_nh) {
    b2r_floor_params_default(&params_);
    params_.tilt_deg = private_nh.param<double>("tilt_deg", 0.0);
    params_.sensor_height = private_nh.param<double>("sensor_height", 2.0);
    params_.height_clip_range = private_nh.param<double>("height_clip_range", 1.0);
    params_.floor_pts_thresh = private_nh.param<int>("floor_pts_thresh", 512);
    params_.floor_normal_thresh = private_nh.param<double>("floor_normal_thresh", 10.0);
    params_.use_normal_filtering = private_nh.param<bool>("use_normal_filtering", true) ? 1 : 0;
    params_.normal_filter_thresh = private_nh.param<double>("normal_filter_thresh", 20.0);
    h_ = b200_frontend::create_handle(private_nh);
  }
  ~B200FloorDetector() { b2r_destroy(h_); }
  B200FloorDetector(const B200FloorDetector&) = delete;
  B200FloorDetector& operator=(const B200FloorDetector&) = delete;

  // What detect(cloud) returns (:110-180).  want_filtered / want_inliers: floor_filtered_pub / floor_points_pub have subscribers.
  // filtered() then holds floor_filtered_points whenever it was asked for, a floor found or not (:127-130); inliers() holds
  // floor_points only when coefficients are returned (:168-177).  Both take cloud->header (:128, :174), width = size, height = 1.
  // is_dense (UPSTREAM-RECALL, PCL 1.10): normal_filtering sets false (:235); without it the plane clips' ExtractIndices copy the
  // input's flag; the inlier extraction copies the filtered cloud's.
  boost::optional<Eigen::Vector4f> detect(const pcl::PointCloud<PointT>::Ptr& cloud, bool want_filtered, bool want_inliers) {
    return run(cloud->points.data(), cloud->points.size(), 0, cloud->header, cloud->is_dense, want_filtered, want_inliers);
  }

  // The same on a message as it arrives, unpacked on the device (see B200Prefilter::filter(msg)).  An empty message is reported as
  // B2R_FLOOR_EMPTY_INPUT without detecting and without a filtered cloud: cloud_callback returns before detect (:76-78).
  boost::optional<Eigen::Vector4f> detect(const sensor_msgs::PointCloud2& msg, bool want_filtered, bool want_inliers) {
    size_t n = 0;
    const void* d = b200_frontend::ingest_pointcloud2(h_, msg, &n);
    if (n == 0) {
      reset();
      result_.reason = B2R_FLOOR_EMPTY_INPUT;
      return boost::none;
    }
    pcl::PCLHeader header;
    pcl_conversions::toPCL(msg.header, header);
    return run(d, n, 1, header, msg.is_dense != 0, want_filtered, want_inliers);  // fromROSMsg copies is_dense
  }

  // the clouds of the last detect, nullptr where the rules above give none
  pcl::PointCloud<PointT>::Ptr filtered() const { return filtered_; }
  pcl::PointCloud<PointT>::Ptr inliers() const { return inliers_; }
  // the engine's account of the last detect: reason, RANSAC iterations, model indices, device readbacks
  const b2r_floor_result& last_result() const { return result_; }

private:
  void reset() {
    filtered_.reset();
    inliers_.reset();
    b2r_floor_result r = {};
    r.model_indices[0] = r.model_indices[1] = r.model_indices[2] = -1;
    result_ = r;
  }

  boost::optional<Eigen::Vector4f> run(const void* points, size_t n, int device_input, const pcl::PCLHeader& header, bool input_is_dense,
                                       bool want_filtered, bool want_inliers) {
    reset();
    pcl::PointCloud<PointT>::Ptr filtered, inliers;
    if (want_filtered) {
      filtered.reset(new pcl::PointCloud<PointT>());
      filtered->points.resize(n);
    }
    if (want_inliers) {
      inliers.reset(new pcl::PointCloud<PointT>());
      inliers->points.resize(n);
    }
    b200_frontend::check(b2r_floor_detect(h_, points, n, sizeof(PointT), device_input, &params_, &result_,
                                          filtered ? filtered->points.data() : nullptr, inliers ? inliers->points.data() : nullptr, nullptr, nullptr));
    const bool dense = params_.use_normal_filtering ? false : input_is_dense;
    auto finish = [&](pcl::PointCloud<PointT>& c, size_t m) {
      c.points.resize(m);
      c.header = header;
      c.width = static_cast<uint32_t>(m);
      c.height = 1;
      c.is_dense = dense;
    };
    if (filtered) {
      finish(*filtered, result_.n_filtered);
      filtered_ = filtered;
    }
    if (!result_.detected) return boost::none;
    if (inliers) {
      finish(*inliers, result_.n_inliers);
      inliers_ = inliers;
    }
    return Eigen::Vector4f(result_.coeffs[0], result_.coeffs[1], result_.coeffs[2], result_.coeffs[3]);
  }

  b2r_floor_params params_;
  b2r_floor_result result_ = {};
  pcl::PointCloud<PointT>::Ptr filtered_, inliers_;
  b2r_handle* h_ = nullptr;
};

}  // namespace hdl_graph_slam
