// odo_gate_harness.cpp — drives csrc/odometry_gate.cuh (host code only) on records a test writes, for tests/test_odometry_gate.py.
//
//   odo_gate_harness <in.f64> <out.f64>
// in : records of 57 doubles: keyframe_pose[16], prev_trans[16], trans[16] (row-major float32 values), converged, stamp,
//      keyframe_stamp, keyframe_delta_trans, keyframe_delta_angle, keyframe_delta_time, transform_thresholding, max_acceptable_trans,
//      max_acceptable_angle
// out: records of 57 doubles: decision (0 rejected, 1 accepted, 2 keyframe), odom[16], dx, da, delta_trans, delta_angle,
//      w(delta), w(trans), too_large, wants_keyframe, inverse(prev_trans)[16], delta[16]
// Compile with -ffp-contract=off, like the engine's host code and the oracle.
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../hdl_graph_slam_b200/csrc/odometry_gate.cuh"

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  std::vector<double> in;
  double buf[57];
  while (std::fread(buf, sizeof(double), 57, f) == 57) in.insert(in.end(), buf, buf + 57);
  std::fclose(f);
  const size_t n = in.size() / 57;
  std::vector<double> out(n * 57);
  for (size_t i = 0; i < n; i++) {
    const double* r = &in[i * 57];
    float kp[16], pt[16], tr[16];
    for (int k = 0; k < 16; k++) { kp[k] = (float)r[k]; pt[k] = (float)r[16 + k]; tr[k] = (float)r[32 + k]; }
    b2r_odometry_params p = {};
    p.keyframe_delta_trans = r[51]; p.keyframe_delta_angle = r[52]; p.keyframe_delta_time = r[53];
    p.transform_thresholding = (int32_t)r[54]; p.max_acceptable_trans = r[55]; p.max_acceptable_angle = r[56];
    double* o = &out[i * 57];
    float odom[16], inv[16], delta[16];
    o[0] = (double)b2r::odometry_gate(p, kp, pt, tr, r[48] != 0.0, r[49], r[50], odom);
    for (int k = 0; k < 16; k++) o[1 + k] = odom[k];
    o[23] = b2r::odometry_step_too_large(p, pt, tr, &o[17], &o[18]) ? 1.0 : 0.0;
    o[19] = b2r::translation_norm(tr);
    o[20] = b2r::rotation_angle(tr);
    b2r::mat4_inv_rigid_general(pt, inv);
    b2r::mat4_mul(inv, tr, delta);
    o[21] = b2r::quat_w_from_R(delta);
    o[22] = b2r::quat_w_from_R(tr);
    o[24] = b2r::odometry_wants_keyframe(p, tr, r[49], r[50]) ? 1.0 : 0.0;
    for (int k = 0; k < 16; k++) { o[25 + k] = inv[k]; o[41 + k] = delta[k]; }
  }
  f = std::fopen(argv[2], "wb");
  if (!f) return 4;
  const bool ok = std::fwrite(out.data(), sizeof(double), out.size(), f) == out.size();
  std::fclose(f);
  return ok ? 0 : 5;
}
