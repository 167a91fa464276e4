// odometry_gate.cuh — the pose arithmetic and the two decisions of ScanMatchingOdometryNodelet::matching (host code only, no CUDA:
// tests/odo_gate_harness.cpp compiles it with the host compiler alone).
//
// Mirrors hdl_graph_slam's apps/scan_matching_odometry_nodelet.cpp:
//   not converged                  -> return keyframe_pose * prev_trans                                  :214-218
//   odom = keyframe_pose * trans                                                                          :220-221
//   transform_thresholding         -> delta = prev_trans.inverse() * trans, dx, da, reject               :223-233
//   keyframe switch                -> delta_trans, delta_angle, delta_time                               :241-252
//                                     (delta_time of two ros::Time stamps: ros_delta_time; of two doubles: their difference)
// Arithmetic (DESIGN.md §2 "Documented oracle choices"): everything the reference computes on Eigen::Matrix4f is float32 here too.
//   4x4 products    float32, each entry ((a0 b0 + a1 b1) + a2 b2) + a3 b3 with separate multiplies and adds (the translation unit
//                   is compiled with -ffp-contract=off, build.py);
//   norms           `double dx = v.norm()` is a float32 norm widened afterwards: sqrtf((x x + y y) + z z), the association this
//                   project uses for Vector3f::norm() everywhere (prefilter.cuh, oracle/gicp.cpp); Eigen is not available to check
//                   it against: if its unrolled reduction associates x x + (y y + z z), a norm differs by at most one float32 ulp;
//   angles          `double da = std::acos(Quaternionf(R).w())` is the float overload: acosf of the float32 w, widened afterwards.
//                   w > 1 (a trace that rounds above 3) gives NaN, and every comparison with NaN is false, as in the reference;
//   inverse         prev_trans.inverse() is Eigen's general float32 4x4 inverse, which cannot be restated bit for bit without
//                   Eigen.  The engine inverts the 3x3 block by cofactors in float64, forms -A^-1 t in float64 and rounds each entry
//                   to float32 once; the last row is 0 0 0 1.  Only `delta` (hence dx, da of the thresholding block) is unpinned by
//                   this; it is within a float32 ulp or two of any correctly rounded inverse of a rigid transform.
// All matrices are ROW-major float[16].
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include "../../include/b200reg.h"

namespace b2r {

inline void mat4_mul(const float* a, const float* b, float* o) {
  float t[16];
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) {
      float s = a[r * 4 + 0] * b[0 * 4 + c];
      s += a[r * 4 + 1] * b[1 * 4 + c];
      s += a[r * 4 + 2] * b[2 * 4 + c];
      s += a[r * 4 + 3] * b[3 * 4 + c];
      t[r * 4 + c] = s;
    }
  std::memcpy(o, t, sizeof(t));
}

// inverse of [A t; 0 1] with a general 3x3 A (see "inverse" above)
inline void mat4_inv_rigid_general(const float* m, float* o) {
  const double a[9] = {m[0], m[1], m[2], m[4], m[5], m[6], m[8], m[9], m[10]};
  const double c00 = a[4] * a[8] - a[5] * a[7], c01 = a[5] * a[6] - a[3] * a[8], c02 = a[3] * a[7] - a[4] * a[6];
  const double id = 1.0 / (a[0] * c00 + a[1] * c01 + a[2] * c02);
  const double Ai[9] = {c00 * id, (a[2] * a[7] - a[1] * a[8]) * id, (a[1] * a[5] - a[2] * a[4]) * id,
                        c01 * id, (a[0] * a[8] - a[2] * a[6]) * id, (a[2] * a[3] - a[0] * a[5]) * id,
                        c02 * id, (a[1] * a[6] - a[0] * a[7]) * id, (a[0] * a[4] - a[1] * a[3]) * id};
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) o[r * 4 + c] = (float)Ai[r * 3 + c];
    o[r * 4 + 3] = (float)(-(Ai[r * 3 + 0] * m[3] + Ai[r * 3 + 1] * m[7] + Ai[r * 3 + 2] * m[11]));
  }
  o[12] = o[13] = o[14] = 0.f; o[15] = 1.f;
}

// w of Eigen::Quaternionf(R) for the rotation block of m (Eigen 3.3's quaternionbase_assign_impl<..., 3, 3>, all four branches)
inline float quat_w_from_R(const float* m) {
  float t = m[0] + m[5] + m[10];
  if (t > 0.f) {
    t = std::sqrt(t + 1.0f);
    return 0.5f * t;
  }
  int i = 0;
  if (m[5] > m[0]) i = 1;
  if (m[10] > m[i * 4 + i]) i = 2;
  const int j = (i + 1) % 3, k = (j + 1) % 3;
  t = std::sqrt(m[i * 4 + i] - m[j * 4 + j] - m[k * 4 + k] + 1.0f);
  t = 0.5f / t;
  return (m[k * 4 + j] - m[j * 4 + k]) * t;
}

// `double d = m.block<3, 1>(0, 3).norm()`
inline double translation_norm(const float* m) { return (double)std::sqrt((m[3] * m[3] + m[7] * m[7]) + m[11] * m[11]); }
// `double a = std::acos(Eigen::Quaternionf(m.block<3, 3>(0, 0)).w())`
inline double rotation_angle(const float* m) { return (double)std::acos(quat_w_from_R(m)); }

// :223-233 — is the step from prev_trans to trans too large?  (*dx, *da: the two quantities compared, for the tests)
inline bool odometry_step_too_large(const b2r_odometry_params& p, const float* prev_trans, const float* trans, double* dx_out = nullptr,
                                    double* da_out = nullptr) {
  float inv[16], delta[16];
  mat4_inv_rigid_general(prev_trans, inv);
  mat4_mul(inv, trans, delta);
  const double dx = translation_norm(delta);
  const double da = rotation_angle(delta);
  if (dx_out) *dx_out = dx;
  if (da_out) *da_out = da;
  return dx > p.max_acceptable_trans || da > p.max_acceptable_angle;
}

// :243 `double delta_time = (stamp - keyframe_stamp).toSec()` on two ros::Time stamps (UPSTREAM-RECALL: roscpp_core's
// TimeBase::operator- and DurationBase::toSec, not in this tree): seconds and nanoseconds are subtracted as integers, the nanoseconds
// normalised into [0, 1e9) by borrowing from the seconds, and toSec() = (double)sec + 1e-9 * (double)nsec.  Exact up to that last
// rounding, unlike the difference of two epoch stamps widened to double, which keeps only about 0.24 us of an epoch stamp.
inline double ros_delta_time(uint32_t sec, uint32_t nsec, uint32_t ref_sec, uint32_t ref_nsec) {
  int64_t s = (int64_t)sec - (int64_t)ref_sec;
  int64_t ns = (int64_t)nsec - (int64_t)ref_nsec;
  s += ns / 1000000000LL;
  ns %= 1000000000LL;
  if (ns < 0) {
    ns += 1000000000LL;
    s -= 1;
  }
  return (double)s + 1e-9 * (double)ns;
}

// :241-244 — does this accepted frame become the keyframe?  delta_time: the frame's stamp minus the keyframe's, in seconds
inline bool odometry_wants_keyframe_dt(const b2r_odometry_params& p, const float* trans, double delta_time) {
  const double delta_trans = translation_norm(trans);
  const double delta_angle = rotation_angle(trans);
  return delta_trans > p.keyframe_delta_trans || delta_angle > p.keyframe_delta_angle || delta_time > p.keyframe_delta_time;
}
// the same with the two stamps as double seconds, subtracted as doubles
inline bool odometry_wants_keyframe(const b2r_odometry_params& p, const float* trans, double stamp, double keyframe_stamp) {
  return odometry_wants_keyframe_dt(p, trans, stamp - keyframe_stamp);
}

enum OdometryDecision { ODOM_REJECTED = 0, ODOM_ACCEPTED = 1, ODOM_KEYFRAME = 2 };

// :214-252 after the align: the decision on this frame and the pose matching() returns (odom, row-major).
//   ODOM_REJECTED  not converged or thresholded: odom = keyframe_pose * prev_trans, no state changes
//   ODOM_ACCEPTED  odom = keyframe_pose * trans; the caller sets prev_trans = trans, prev_time = stamp
//   ODOM_KEYFRAME  as ACCEPTED, and the frame becomes the keyframe: keyframe_pose = odom, keyframe_stamp = stamp, prev_trans = I
//   delta_time     the frame's stamp minus the keyframe's (ros_delta_time, or a difference of doubles)
inline OdometryDecision odometry_gate_dt(const b2r_odometry_params& p, const float* keyframe_pose, const float* prev_trans, const float* trans,
                                         bool converged, double delta_time, float* odom) {
  if (!converged || (p.transform_thresholding && odometry_step_too_large(p, prev_trans, trans))) {
    mat4_mul(keyframe_pose, prev_trans, odom);
    return ODOM_REJECTED;
  }
  mat4_mul(keyframe_pose, trans, odom);
  return odometry_wants_keyframe_dt(p, trans, delta_time) ? ODOM_KEYFRAME : ODOM_ACCEPTED;
}
inline OdometryDecision odometry_gate(const b2r_odometry_params& p, const float* keyframe_pose, const float* prev_trans, const float* trans,
                                      bool converged, double stamp, double keyframe_stamp, float* odom) {
  return odometry_gate_dt(p, keyframe_pose, prev_trans, trans, converged, stamp - keyframe_stamp, odom);
}

}  // namespace b2r
