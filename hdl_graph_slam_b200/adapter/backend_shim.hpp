// backend_shim.hpp — TEST-ONLY stand-in for the few ROS / Eigen / g2o / hdl_graph_slam declarations b200_backend.hpp touches (with
// pcl_shim.hpp for PCL), so the back-end drop-in can be compiled and run in an image without them (tests/test_backend_syntax.py,
// tests/backend_harness.cpp).  Names and signatures follow ROS noetic's roscpp, Eigen 3.3, g2o and the reference's keyframe.hpp /
// loop_detector.hpp.  Nothing here is shipped or linked.
#pragma once
#include "pcl_shim.hpp"
#include <map>
#include <memory>
#include <sstream>
#include <string>
#include <vector>

namespace Eigen {
struct Matrix4d {  // column-major, like Eigen's default
  double m[16];
  double* data() { return m; }
  const double* data() const { return m; }
};
struct Isometry3d {
  Matrix4d mat;
  Matrix4d& matrix() { return mat; }
  const Matrix4d& matrix() const { return mat; }
};
struct MatrixXd {
  int r = 0, c = 0;
  std::vector<double> v;  // column-major
  static MatrixXd Identity(int rows, int cols) {
    MatrixXd I;
    I.r = rows;
    I.c = cols;
    I.v.assign((size_t)rows * cols, 0.0);
    for (int i = 0; i < rows && i < cols; i++) I(i, i) = 1.0;
    return I;
  }
  double& operator()(int i, int j) { return v[(size_t)j * r + i]; }
  double operator()(int i, int j) const { return v[(size_t)j * r + i]; }
  int rows() const { return r; }
  int cols() const { return c; }
};
}  // namespace Eigen

namespace ros {
// the private namespace of a nodelet: values kept as strings, converted on read as the parameter server would.  Copies share one
// store, as copies of a roscpp NodeHandle reach the same parameter server.
class NodeHandle {
public:
  void setParam(const std::string& key, const std::string& value) { (*p_)[key] = value; }
  bool hasParam(const std::string& key) const { return p_->count(key) != 0; }
  template <typename T>
  T param(const std::string& key, const T& default_val) const {
    auto it = p_->find(key);
    if (it == p_->end()) return default_val;
    return convert(it->second, default_val);
  }

private:
  template <typename T>
  static T convert(const std::string& s, const T&) {
    std::istringstream in(s);
    T v{};
    in >> v;
    return v;
  }
  static std::string convert(const std::string& s, const std::string&) { return s; }
  static bool convert(const std::string& s, const bool&) { return s == "true" || s == "1"; }
  std::shared_ptr<std::map<std::string, std::string>> p_ = std::make_shared<std::map<std::string, std::string>>();
};
}  // namespace ros

namespace g2o {
class VertexSE3 {
public:
  const Eigen::Isometry3d& estimate() const { return est_; }
  void setEstimate(const Eigen::Isometry3d& e) { est_ = e; }

private:
  Eigen::Isometry3d est_;
};
}  // namespace g2o

namespace hdl_graph_slam {
struct KeyFrame {
  using PointT = pcl::PointXYZI;
  using Ptr = std::shared_ptr<KeyFrame>;
  double accum_distance = 0.0;
  pcl::PointCloud<PointT>::ConstPtr cloud;
  g2o::VertexSE3* node = nullptr;
};

struct KeyFrameSnapshot {
  using PointT = KeyFrame::PointT;
  using Ptr = std::shared_ptr<KeyFrameSnapshot>;
  KeyFrameSnapshot(const Eigen::Isometry3d& pose, const pcl::PointCloud<PointT>::ConstPtr& cloud) : pose(pose), cloud(cloud) {}
  Eigen::Isometry3d pose;
  pcl::PointCloud<PointT>::ConstPtr cloud;
};

struct Loop {
  using Ptr = std::shared_ptr<Loop>;
  Loop(const KeyFrame::Ptr& key1, const KeyFrame::Ptr& key2, const Eigen::Matrix4f& relpose) : key1(key1), key2(key2), relative_pose(relpose) {}
  KeyFrame::Ptr key1;
  KeyFrame::Ptr key2;
  Eigen::Matrix4f relative_pose;
};

class GraphSLAM {};
}  // namespace hdl_graph_slam
