// b200_odometry.hpp — drop-in replacement for the point work of ScanMatchingOdometryNodelet of koide3/hdl_graph_slam, served by one
// engine handle of libb200reg.so and its odometry mirror:
//   initialize_params' odometry half (apps/scan_matching_odometry_nodelet.cpp:65-107),
//   downsample (:140-157), matching (:165-262),
//   the point work of publish_scan_matching_status (:298-335)      -> B200ScanMatchingOdometry
// It also takes the sensor_msgs::PointCloud2 as it arrives and unpacks it on the device (b200_frontend::ingest_pointcloud2), so the scan
// is never converted on the host.  The nodelet keeps its subscriptions, the msf / tf lookups that make msf_delta (:182-207),
// publish_odometry, the tf broadcasters, the status message itself (its prediction error is host Eigen on final_transformation()) and
// read_until.  INTEGRATION.md §4d shows the nodelet patch.  Compiled only where ROS, PCL, Eigen and boost exist;
// tests/test_odometry_syntax.py checks it against the test-only stand-ins adapter/pcl_shim.hpp, backend_shim.hpp and frontend_shim.hpp.
//
// Threads: an instance is used by one thread at a time, as the nodelet's callback queue does.  Distinct instances own distinct handles
// and may run concurrently.
#pragma once
#include <b200reg.h>
#include "b200_frontend.hpp"
#include "b200_select.hpp"
#include <cstdint>
#include <cstring>
#include <iostream>
#include <memory>
#include <stdexcept>
#include <string>

namespace hdl_graph_slam {

class B200ScanMatchingOdometry {
public:
  using PointT = pcl::PointXYZI;

  // Reads what initialize_params reads for the odometry (:65-107), with its console and warning lines: an unknown downsample_method
  // means NONE.  The registration handle is select_registration_method(private_nh) (:106) on "reg_device_id".  A registration_method
  // the engine does not re-create (B2R_EUNSUPPORTED), or no device, throws std::runtime_error with the engine's message, so the
  // nodelet can keep its reference code.
  explicit B200ScanMatchingOdometry(ros::NodeHandle& private_nh) {
    odom_frame_id_ = private_nh.param<std::string>("odom_frame_id", "odom");
    b2r_odometry_params p = {};
    p.keyframe_delta_trans = private_nh.param<double>("keyframe_delta_trans", 0.25);
    p.keyframe_delta_angle = private_nh.param<double>("keyframe_delta_angle", 0.15);
    p.keyframe_delta_time = private_nh.param<double>("keyframe_delta_time", 1.0);
    p.transform_thresholding = private_nh.param<bool>("transform_thresholding", false) ? 1 : 0;
    p.max_acceptable_trans = private_nh.param<double>("max_acceptable_trans", 1.0);
    p.max_acceptable_angle = private_nh.param<double>("max_acceptable_angle", 1.0);
    p.publish_status = 0;  // chosen per frame: matching(..., want_status, ...)
    const std::string downsample_method = private_nh.param<std::string>("downsample_method", "VOXELGRID");
    const double downsample_resolution = private_nh.param<double>("downsample_resolution", 0.1);
    p.downsample_resolution = static_cast<float>(downsample_resolution);  // setLeafSize takes floats (:88, :93)
    if (downsample_method == "VOXELGRID") {
      std::cout << "downsample: VOXELGRID " << downsample_resolution << std::endl;
      p.downsample_method = B2R_DOWNSAMPLE_VOXELGRID;
    } else if (downsample_method == "APPROX_VOXELGRID") {
      std::cout << "downsample: APPROX_VOXELGRID " << downsample_resolution << std::endl;
      p.downsample_method = B2R_DOWNSAMPLE_APPROX_VOXELGRID;
    } else {
      if (downsample_method != "NONE") {
        std::cerr << "warning: unknown downsampling type (" << downsample_method << ")" << std::endl;
        std::cerr << "       : use passthrough filter" << std::endl;
      }
      std::cout << "downsample: NONE" << std::endl;
      p.downsample_method = B2R_DOWNSAMPLE_NONE;
    }
    h_ = b200_select::select_registration_method(private_nh);
    const int rc = b2r_odometry_create(h_, &p, &o_);
    if (rc < 0) {
      const std::string msg = std::string("b200reg: ") + b2r_last_error();
      b2r_destroy(h_);
      throw std::runtime_error(msg);
    }
    keyframe_pose_ = broadcast_pose_ = Eigen::Matrix4f::Identity();
  }
  ~B200ScanMatchingOdometry() {
    b2r_odometry_destroy(o_);
    b2r_destroy(h_);
  }
  B200ScanMatchingOdometry(const B200ScanMatchingOdometry&) = delete;
  B200ScanMatchingOdometry& operator=(const B200ScanMatchingOdometry&) = delete;

  // matching(stamp, cloud) (:165-262): the pose it returns.
  //   msf_delta:    nullptr for identity (neither the IMU nor the robot odometry gave a guess, :180); otherwise msf_delta.matrix().
  //   want_status:  status_pub has subscribers (:299): converged(), final_transformation(), matching_error() and inlier_fraction()
  //                 are then valid for this frame unless it is the first (:166-174 publishes no status).
  //   want_aligned: aligned_points_pub has subscribers (:254): aligned() then holds the cloud unless the frame is the first or rejected.
  // The keyframe test's delta_time is roscpp's exact (stamp - keyframe_stamp).toSec() (b2r_odometry_matching_ros).
  Eigen::Matrix4f matching(const ros::Time& stamp, const pcl::PointCloud<PointT>::ConstPtr& cloud, const Eigen::Matrix4f* msf_delta,
                           bool want_status, bool want_aligned) {
    return run(stamp, cloud->points.data(), cloud->points.size(), 0, cloud->header, cloud->width, cloud->height, cloud->is_dense, msf_delta,
               want_status, want_aligned);
  }

  // The same on the message as cloud_callback receives it (:112-116): the stamp is msg.header.stamp, the cloud's header comes from
  // msg.header, and the message is unpacked on the device as fromROSMsg would unpack it (all width * height records, NaN records and
  // padded rows included).  A non-empty message without FLOAT32 x, y and z throws std::invalid_argument: convert it with fromROSMsg
  // and call the first overload.
  Eigen::Matrix4f matching(const sensor_msgs::PointCloud2& msg, const Eigen::Matrix4f* msf_delta, bool want_status, bool want_aligned) {
    size_t n = 0;
    const void* d = b200_frontend::ingest_pointcloud2(h_, msg, &n);
    pcl::PCLHeader header;
    pcl_conversions::toPCL(msg.header, header);
    return run(msg.header.stamp, d, n, 1, header, msg.width, msg.height, msg.is_dense != 0, msf_delta, want_status, want_aligned);
  }

  // the status of the last frame (valid where matching's want_status says)
  bool converged() const { return status_.converged != 0; }
  Eigen::Matrix4f final_transformation() const { return from_colmajor(status_.trans); }
  double matching_error() const { return status_.matching_error; }
  float inlier_fraction() const { return status_.inlier_fraction; }
  // the keyframe pose as :238 broadcasts it on an accepted frame, i.e. before this frame's keyframe switch
  const Eigen::Matrix4f& keyframe_pose() const { return broadcast_pose_; }
  bool keyframe_updated() const { return status_.keyframe_updated != 0; }
  bool frame_rejected() const { return status_.frame_rejected != 0; }
  // aligned_points (:254-259): the raw input cloud under the returned pose, with the input's header, width, height and is_dense and
  // frame_id = odom_frame_id; nullptr unless it was asked for and the frame was accepted
  pcl::PointCloud<PointT>::ConstPtr aligned() const { return aligned_; }
  const std::string& odom_frame_id() const { return odom_frame_id_; }

private:
  static Eigen::Matrix4f from_colmajor(const float* m) {
    Eigen::Matrix4f T;
    std::memcpy(T.data(), m, 16 * sizeof(float));  // both column-major
    return T;
  }

  Eigen::Matrix4f run(const ros::Time& stamp, const void* points, size_t n, int device_input, const pcl::PCLHeader& header, uint32_t width,
                      uint32_t height, bool is_dense, const Eigen::Matrix4f* msf_delta, bool want_status, bool want_aligned) {
    aligned_.reset();
    b2r_odometry_status st;
    b200_select::check(b2r_odometry_matching_ros(o_, stamp.sec, stamp.nsec, points, n, sizeof(PointT), device_input,
                                                 msf_delta ? msf_delta->data() : nullptr, want_status ? 1 : 0, &st));
    const bool first = !has_keyframe_;
    has_keyframe_ = true;
    status_ = st;
    const Eigen::Matrix4f odom = from_colmajor(st.odom);
    broadcast_pose_ = keyframe_pose_;
    if (st.keyframe_updated) keyframe_pose_ = odom;  // :248 (the first frame's keyframe pose is the identity it returns)
    if (want_aligned && !first && !st.frame_rejected) {
      pcl::PointCloud<PointT>::Ptr a(new pcl::PointCloud<PointT>());
      a->points.resize(n);
      b200_select::check(b2r_odometry_aligned(o_, is_dense ? 1 : 0, a->points.data(), n, sizeof(PointT)));
      a->header = header;
      a->header.frame_id = odom_frame_id_;
      a->width = width;
      a->height = height;
      a->is_dense = is_dense;
      aligned_ = a;
    }
    return odom;
  }

  std::string odom_frame_id_;
  b2r_handle* h_ = nullptr;
  b2r_odometry* o_ = nullptr;
  bool has_keyframe_ = false;
  b2r_odometry_status status_ = {};
  Eigen::Matrix4f keyframe_pose_, broadcast_pose_;
  pcl::PointCloud<PointT>::Ptr aligned_;
};

}  // namespace hdl_graph_slam
