// b200_select.hpp — select_registration_method(pnh) (src/hdl_graph_slam/registrations.cpp:22-124) for the drop-ins that need a
// registration handle configured from a nodelet's reg_* rosparams: B200KeyframeCache (b200_backend.hpp) and B200ScanMatchingOdometry
// (b200_odometry.hpp).  Include it after the ROS headers (it uses ros::NodeHandle).
#pragma once
#include <b200reg.h>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

namespace hdl_graph_slam {
namespace b200_select {

inline void check(int rc) {
  if (rc < 0) throw std::runtime_error(std::string("b200reg: ") + b2r_last_error());
}

// b2r_select_registration_method with the parameters of pnh that are set, on the device "reg_device_id" names (default 0).  The engine
// applies each branch's own defaults to the others.  A registration_method the engine does not re-create (B2R_EUNSUPPORTED), or no
// device, throws std::runtime_error with the engine's message, so the caller can keep the reference classes.
inline b2r_handle* select_registration_method(ros::NodeHandle& pnh) {
  std::vector<std::string> keys, values;
  auto put = [&](const char* k, const std::string& v) { keys.push_back(k); values.push_back(v); };
  auto num = [](double v) { char s[32]; std::snprintf(s, sizeof s, "%.17g", v); return std::string(s); };
  for (const char* k : {"registration_method", "reg_nn_search_method"})
    if (pnh.hasParam(k)) put(k, pnh.param<std::string>(k, ""));
  for (const char* k : {"reg_resolution", "reg_transformation_epsilon", "reg_max_correspondence_distance"})
    if (pnh.hasParam(k)) put(k, num(pnh.param<double>(k, 0.0)));
  for (const char* k : {"reg_maximum_iterations", "reg_correspondence_randomness", "reg_max_optimizer_iterations"})
    if (pnh.hasParam(k)) put(k, std::to_string(pnh.param<int>(k, 0)));
  if (pnh.hasParam("reg_use_reciprocal_correspondences"))
    put("reg_use_reciprocal_correspondences", pnh.param<bool>("reg_use_reciprocal_correspondences", false) ? "true" : "false");
  std::vector<const char*> k, v;
  for (size_t i = 0; i < keys.size(); i++) { k.push_back(keys[i].c_str()); v.push_back(values[i].c_str()); }
  b2r_handle* h = nullptr;
  check(b2r_select_registration_method(k.data(), v.data(), (int)k.size(), pnh.param<int>("reg_device_id", 0), &h));
  return h;
}

}  // namespace b200_select
}  // namespace hdl_graph_slam
