// frontend_shim.hpp — TEST-ONLY stand-in for the few ROS / PCL / Eigen / boost declarations b200_frontend.hpp touches beyond
// pcl_shim.hpp and backend_shim.hpp (whose ros::NodeHandle it reuses), so the front-end drop-in can be compiled and run in an image
// without them (tests/test_frontend_syntax.py, tests/frontend_harness.cpp).  Names and signatures follow ROS noetic's
// sensor_msgs / std_msgs / pcl_conversions, Eigen 3.3 and boost 1.71.  Nothing here is shipped or linked.
#pragma once
#include "backend_shim.hpp"
#include <cstdint>
#include <string>
#include <utility>
#include <vector>

namespace Eigen {
struct Vector3f {
  float v[3];
  Vector3f() : v{0.f, 0.f, 0.f} {}
  Vector3f(float x, float y, float z) : v{x, y, z} {}
  float& operator[](int i) { return v[i]; }
  float operator[](int i) const { return v[i]; }
  float* data() { return v; }
  const float* data() const { return v; }
};
struct Vector4f {
  float v[4];
  Vector4f() : v{0.f, 0.f, 0.f, 0.f} {}
  Vector4f(float a, float b, float c, float d) : v{a, b, c, d} {}
  float& operator[](int i) { return v[i]; }
  float operator[](int i) const { return v[i]; }
  float* data() { return v; }
  const float* data() const { return v; }
};
}  // namespace Eigen

namespace boost {
struct none_t {};
const none_t none = none_t();
// the part of boost::optional the nodelets use: engaged test, dereference, boost::none
template <typename T>
class optional {
public:
  optional() : has_(false), v_() {}
  optional(none_t) : has_(false), v_() {}
  optional(const T& v) : has_(true), v_(v) {}
  explicit operator bool() const { return has_; }
  bool is_initialized() const { return has_; }
  const T& operator*() const { return v_; }
  T& operator*() { return v_; }
  const T* operator->() const { return &v_; }
  const T& get() const { return v_; }

private:
  bool has_;
  T v_;
};
}  // namespace boost

namespace ros {
struct Time {
  uint32_t sec = 0, nsec = 0;
  uint64_t toNSec() const { return (uint64_t)sec * 1000000000ull + nsec; }
};
}  // namespace ros

namespace std_msgs {
struct Header {
  uint32_t seq = 0;
  ros::Time stamp;
  std::string frame_id;
};
}  // namespace std_msgs

namespace sensor_msgs {
struct PointField {
  enum : uint8_t { INT8 = 1, UINT8 = 2, INT16 = 3, UINT16 = 4, INT32 = 5, UINT32 = 6, FLOAT32 = 7, FLOAT64 = 8 };
  std::string name;
  uint32_t offset = 0;
  uint8_t datatype = 0;
  uint32_t count = 0;
};
struct PointCloud2 {
  std_msgs::Header header;
  uint32_t height = 0, width = 0;
  std::vector<PointField> fields;
  uint8_t is_bigendian = 0;
  uint32_t point_step = 0, row_step = 0;
  std::vector<uint8_t> data;
  uint8_t is_dense = 0;
};
}  // namespace sensor_msgs

namespace pcl_conversions {
// pcl_conversions::toPCL(const std_msgs::Header&, pcl::PCLHeader&): the stamp goes to microseconds
inline void toPCL(const std_msgs::Header& header, pcl::PCLHeader& pcl_header) {
  pcl_header.stamp = header.stamp.toNSec() / 1000ull;
  pcl_header.seq = header.seq;
  pcl_header.frame_id = header.frame_id;
}
}  // namespace pcl_conversions
