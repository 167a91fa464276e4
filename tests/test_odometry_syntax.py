"""CPU-only: the odometry drop-in (hdl_graph_slam_b200/adapter/b200_odometry.hpp) compiles with -Wall -Werror against the C ABI header and
the test-only stand-ins, links to the library, and without a GPU its constructor throws with the engine's B2R_ENODEVICE message after
printing the reference's parameter lines (an unknown downsample name warns and means NONE).

The keyframe test's delta_time on ros::Time stamps (csrc/odometry_gate.cuh: ros_delta_time, odometry_wants_keyframe_dt), driven through
a small harness, against roscpp's rule restated with Python integers: (stamp - keyframe_stamp) subtracts seconds and nanoseconds,
normalises the nanoseconds into [0, 1e9), and toSec() = sec + 1e-9 * nsec in double."""
import os
import struct
import subprocess
from fractions import Fraction
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
ADAPTER = os.path.join(ROOT, "hdl_graph_slam_b200", "adapter")
LIB = os.path.join(ROOT, "hdl_graph_slam_b200", "_lib")

PROG = r'''
#include "frontend_shim.hpp"
#include "b200_odometry.hpp"
#include <cstdio>
using namespace hdl_graph_slam;
int main() {
  ros::NodeHandle pnh;
  pnh.setParam("downsample_method", "DOWNSAMPLE");
  pnh.setParam("registration_method", "FAST_GICP");
  pnh.setParam("reg_max_correspondence_distance", "2.5");
  try {
    B200ScanMatchingOdometry odom(pnh);
    pcl::PointCloud<pcl::PointXYZI>::ConstPtr empty(new pcl::PointCloud<pcl::PointXYZI>());
    ros::Time t;
    Eigen::Matrix4f delta = Eigen::Matrix4f::Identity();
    Eigen::Matrix4f pose = odom.matching(t, empty, &delta, true, true);
    sensor_msgs::PointCloud2 msg;
    pose = odom.matching(msg, nullptr, false, false);
    std::printf("constructed %d %d %g\n", odom.keyframe_updated() ? 1 : 0, odom.aligned() ? 1 : 0, (double)pose.data()[0]);
  } catch (const std::invalid_argument& e) {
    std::printf("invalid: %s\n", e.what());
  } catch (const std::runtime_error& e) {
    std::printf("no device: %s\n", e.what());
  }
  return 0;
}
'''


def compile_and_run(tmp_path, downsample):
    from hdl_graph_slam_b200 import build
    build.build_engine()
    src = tmp_path / "odometry_main.cpp"
    src.write_text(PROG.replace("DOWNSAMPLE", downsample))
    exe = tmp_path / "odometry_main"
    subprocess.check_call([CXX, "-std=c++14", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-I", ADAPTER, "-o", str(exe),
                           str(src), "-L", LIB, "-lb200reg", "-Wl,-rpath," + LIB, "-pthread"])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    return out


def test_odometry_adapter_compiles_links_and_refuses_without_a_device(tmp_path):
    out = compile_and_run(tmp_path, "APPROX_VOXELGRID")
    assert "downsample: APPROX_VOXELGRID 0.1" in out.stdout, out.stdout
    assert "warning" not in out.stderr
    if "constructed" in out.stdout:  # a CUDA device is present
        return
    assert "no device: b200reg: " in out.stdout, out.stdout
    assert "CUDA" in out.stdout.split("no device: ", 1)[1], out.stdout


def test_unknown_downsample_name_warns_like_the_reference(tmp_path):
    """scan_matching_odometry_nodelet.cpp:95-101: an unknown name warns on stderr, prints NONE and filters nothing"""
    out = compile_and_run(tmp_path, "OCTREE")
    assert "warning: unknown downsampling type (OCTREE)\n       : use passthrough filter\n" in out.stderr
    assert "downsample: NONE" in out.stdout


# ---- the delta-time rule
HARNESS = r'''
#include "../hdl_graph_slam_b200/csrc/odometry_gate.cuh"
#include <cstdio>
// stdin: records (uint32 sec, nsec, ref_sec, ref_nsec, float64 threshold); stdout: (float64 ros_delta_time, int32 keyframe by the ROS
// rule, int32 keyframe by the difference of the two toSec() doubles)
int main() {
  uint32_t s[4];
  double thr;
  while (std::fread(s, sizeof s, 1, stdin) == 1 && std::fread(&thr, sizeof thr, 1, stdin) == 1) {
    b2r_odometry_params p = {};
    p.keyframe_delta_trans = 1e30;
    p.keyframe_delta_angle = 1e30;
    p.keyframe_delta_time = thr;
    const float I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    const double dt = b2r::ros_delta_time(s[0], s[1], s[2], s[3]);
    const int32_t ros = b2r::odometry_wants_keyframe_dt(p, I, dt) ? 1 : 0;
    const double t = (double)s[0] + 1e-9 * (double)s[1], k = (double)s[2] + 1e-9 * (double)s[3];
    const int32_t dbl = b2r::odometry_wants_keyframe(p, I, t, k) ? 1 : 0;
    std::fwrite(&dt, sizeof dt, 1, stdout);
    std::fwrite(&ros, sizeof ros, 1, stdout);
    std::fwrite(&dbl, sizeof dbl, 1, stdout);
  }
  return 0;
}
'''


@pytest.fixture(scope="module")
def delta_harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("delta_time")
    src = d / "delta_time.cpp"
    src.write_text(HARNESS.replace("../hdl_graph_slam_b200/csrc/odometry_gate.cuh", os.path.join(ROOT, "hdl_graph_slam_b200", "csrc", "odometry_gate.cuh")))
    exe = d / "delta_time"
    # -ffp-contract=off, as the engine's host code is built (hdl_graph_slam_b200/build.py)
    subprocess.check_call([CXX, "-std=c++14", "-O2", "-Wall", "-Werror", "-ffp-contract=off", "-o", str(exe), str(src)])

    def run(cases):
        blob = b"".join(struct.pack("<4Id", *c) for c in cases)
        out = subprocess.run([str(exe)], input=blob, capture_output=True, timeout=60, check=True).stdout
        rec = np.frombuffer(out, dtype=[("dt", "<f8"), ("ros", "<i4"), ("dbl", "<i4")])
        assert rec.shape[0] == len(cases)
        return rec
    return run


def ros_to_sec(sec, nsec, ref_sec, ref_nsec):
    """roscpp: TimeBase::operator- -> DurationBase(sec, nsec) normalised with nsec in [0, 1e9) -> toSec()"""
    s, ns = sec - ref_sec, nsec - ref_nsec
    s += ns // 1_000_000_000  # Python's floor division borrows into [0, 1e9) directly
    ns %= 1_000_000_000
    return float(s) + 1e-9 * float(ns)


def exact(sec, nsec, ref_sec, ref_nsec):
    return Fraction((sec - ref_sec) * 1_000_000_000 + nsec - ref_nsec, 1_000_000_000)


def check(delta_harness, cases):
    rec = delta_harness(cases)
    for (s, ns, rs, rns, thr), r in zip(cases, rec):
        want = ros_to_sec(s, ns, rs, rns)
        assert np.float64(r["dt"]).tobytes() == np.float64(want).tobytes(), (s, ns, rs, rns, r["dt"], want)
        assert r["ros"] == int(want > thr)
        dbl = (float(s) + 1e-9 * float(ns)) - (float(rs) + 1e-9 * float(rns))
        assert r["dbl"] == int(dbl > thr)
    return rec


def test_issue_example_switches_by_ros_rule_only(delta_harness):
    """1436939143.126614242 -> 1436939144.126614449 is 1.000000207 s after the keyframe: more than keyframe_delta_time = 1.0.  The two
    stamps as doubles differ by exactly 1.0, so the double rule does not switch"""
    (r,) = check(delta_harness, [(1436939144, 126614449, 1436939143, 126614242, 1.0)])
    assert r["ros"] == 1 and r["dbl"] == 0
    assert (1436939144 + 1e-9 * 126614449) - (1436939143 + 1e-9 * 126614242) == 1.0


@pytest.mark.parametrize("thr", [1.0, 10000.0, 0.15, 0.25])
def test_one_nanosecond_either_side_of_the_threshold(delta_harness, thr):
    """keyframe_delta_time is 1.0 by default and 10000.0 in every shipped launch file: 1 ns above switches and 1 ns below does not, as
    the exact difference decides.  At exactly the threshold the answer is whatever roscpp's toSec() rounds to (checked in `check`)."""
    thr_ns = int(Fraction(str(thr)) * 1_000_000_000)
    rng = np.random.default_rng(int(thr * 1000))
    cases = []
    for _ in range(200):
        ref_sec, ref_nsec = int(rng.integers(1_300_000_000, 1_800_000_000)), int(rng.integers(0, 1_000_000_000))
        for off in (-1, 0, 1):
            t = ref_sec * 1_000_000_000 + ref_nsec + thr_ns + off
            cases.append((t // 1_000_000_000, t % 1_000_000_000, ref_sec, ref_nsec, thr))
    rec = check(delta_harness, cases)
    for c, r in zip(cases, rec):
        if exact(*c[:4]) != Fraction(str(thr)):
            assert r["ros"] == int(exact(*c[:4]) > Fraction(str(thr))), c
    assert rec["ros"][2::3].all() and not rec["ros"][0::3].any()


def test_nanosecond_borrow_and_equal_stamps(delta_harness):
    cases = [
        (101, 5, 100, 999_999_999, 1.0),          # 6 ns: the nanoseconds borrow a second
        (101, 0, 100, 999_999_999, 0.0),          # 1 ns > 0
        (100, 999_999_999, 101, 0, 0.0),          # -1 ns: sec -1, nsec 999999999
        (100, 0, 101, 999_999_999, -1.5),         # -1.999999999 s
        (1436939143, 126614242, 1436939143, 126614242, 0.0),  # equal stamps: 0.0, not > 0
        (1436939143, 126614242, 1436939143, 126614242, 1.0),
        (2_000_000_000, 999_999_999, 0, 0, 1e9),  # a difference of 63 years still fits roscpp's int32 seconds
    ]
    rec = check(delta_harness, cases)
    assert rec["dt"][0] == ros_to_sec(101, 5, 100, 999_999_999) and rec["ros"][0] == 0
    assert rec["ros"][1] == 1 and rec["ros"][2] == 0 and rec["ros"][3] == 0
    assert rec["dt"][4] == 0.0 and rec["ros"][4] == 0 and rec["ros"][5] == 0
    assert rec["ros"][6] == 1


def test_random_stamps_near_the_threshold_follow_roscpp(delta_harness):
    """60 000 epoch stamp pairs within +-300 ns of the threshold: every delta is roscpp's, and the double rule decides a share of
    them differently"""
    rng = np.random.default_rng(7)
    cases = []
    for thr in (0.15, 1.0, 10000.0):
        thr_ns = int(Fraction(thr) * 1_000_000_000)
        for _ in range(20000):
            ref = int(rng.integers(1_300_000_000, 1_800_000_000)) * 1_000_000_000 + int(rng.integers(0, 1_000_000_000))
            t = ref + thr_ns + int(rng.integers(-300, 301))
            cases.append((t // 1_000_000_000, t % 1_000_000_000, ref // 1_000_000_000, ref % 1_000_000_000, thr))
    rec = check(delta_harness, cases)
    assert np.mean(rec["ros"] != rec["dbl"]) > 0.05
