"""CPU-only: the front-end drop-in (hdl_graph_slam_b200/adapter/b200_frontend.hpp) compiles with -Wall against the C ABI header and the
test-only stand-ins for the ROS / PCL / Eigen / boost declarations it uses, and links to the library; constructing either class without
a GPU throws with the engine's B2R_ENODEVICE message.  The numpy restatement of fromROSMsg on padded rows (tests/frontend_ref.py),
which the GPU tests hold the device unpacking to, passes its known answers."""
import os
import subprocess
import numpy as np
from ingest_ref import FLOAT32, NO_FIELD, ONE_BITS, UINT8
from frontend_ref import decode_rows, layout_of, message

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROG = r'''
#include "frontend_shim.hpp"
#include "b200_frontend.hpp"
#include <cstdio>
using namespace hdl_graph_slam;
int main() {
  ros::NodeHandle pnh;
  pnh.setParam("downsample_method", "APPROX_VOXELGRID");
  pnh.setParam("outlier_removal_method", "RADIUS");
  try {
    B200Prefilter prefilter(pnh);
    pcl::PointCloud<pcl::PointXYZI>::ConstPtr empty(new pcl::PointCloud<pcl::PointXYZI>());
    Eigen::Vector3f w(0.f, 0.f, 0.1f);
    Eigen::Matrix4f T = Eigen::Matrix4f::Identity();
    auto out = prefilter.filter(empty, &w, &T);
    sensor_msgs::PointCloud2 msg;
    auto out2 = prefilter.filter(msg, nullptr, nullptr);
    std::printf("prefilter constructed %d %d\n", out ? 1 : 0, out2 ? 1 : 0);
  } catch (const std::invalid_argument& e) {
    std::printf("prefilter invalid: %s\n", e.what());
  } catch (const std::runtime_error& e) {
    std::printf("prefilter no device: %s\n", e.what());
  }
  try {
    B200FloorDetector floor(pnh);
    pcl::PointCloud<pcl::PointXYZI>::Ptr empty(new pcl::PointCloud<pcl::PointXYZI>());
    boost::optional<Eigen::Vector4f> c = floor.detect(empty, true, true);
    std::printf("floor constructed %d %d\n", c ? 1 : 0, floor.last_result().reason);
  } catch (const std::runtime_error& e) {
    std::printf("floor no device: %s\n", e.what());
  }
  return 0;
}
'''


def test_frontend_adapter_compiles_links_and_refuses_without_a_device(tmp_path):
    from hdl_graph_slam_b200 import build
    build.build_engine()
    src = tmp_path / "frontend_main.cpp"
    src.write_text(PROG)
    exe = tmp_path / "frontend_main"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    lib = os.path.join(ROOT, "hdl_graph_slam_b200", "_lib")
    subprocess.check_call([cxx, "-std=c++14", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "hdl_graph_slam_b200", "adapter"), "-o", str(exe), str(src), "-L", lib, "-lb200reg",
                           "-Wl,-rpath," + lib, "-pthread"])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    # the constructor reads the rosparams first (with the reference's console lines), then creates the handle
    assert "downsample: APPROX_VOXELGRID 0.1" in out.stdout and "outlier_removal: RADIUS 0.8 - 2" in out.stdout, out.stdout
    if "constructed" in out.stdout:  # a CUDA device is present: empty inputs give nullptr / no floor
        assert "prefilter constructed 0 0" in out.stdout and "floor constructed 0 1" in out.stdout, out.stdout
        return
    assert "prefilter no device: b200reg: no CUDA device" in out.stdout, out.stdout
    assert "floor no device: b200reg: no CUDA device" in out.stdout, out.stdout


def test_unknown_downsample_name_warns_like_the_reference(tmp_path):
    """an unknown downsample_method is read as NONE with the reference's two warning lines (prefiltering_nodelet.cpp:64-70)"""
    from hdl_graph_slam_b200 import build
    build.build_engine()
    src = tmp_path / "names.cpp"
    src.write_text(r'''
#include "frontend_shim.hpp"
#include "b200_frontend.hpp"
int main() {
  ros::NodeHandle pnh;
  pnh.setParam("downsample_method", "OCTREE");
  pnh.setParam("outlier_removal_method", "MEDIAN");
  try { hdl_graph_slam::B200Prefilter p(pnh); } catch (const std::exception&) {}
  return 0;
}
''')
    exe = tmp_path / "names"
    lib = os.path.join(ROOT, "hdl_graph_slam_b200", "_lib")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++14", "-Wall", "-Werror",
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "hdl_graph_slam_b200", "adapter"), "-o", str(exe),
                           str(src), "-L", lib, "-lb200reg", "-Wl,-rpath," + lib, "-pthread"])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    assert "warning: unknown downsampling type (OCTREE)\n       : use passthrough filter\n" in out.stderr
    assert "downsample: NONE" in out.stdout and "outlier_removal: NONE" in out.stdout


def f32(words):
    return np.array(words, np.float32).view(np.uint32)


def test_padded_rows_known_answer():
    """2 rows x 3 records of point_step 16 (x y z intensity), rows padded to 56 bytes with 0xAB: the padding is skipped"""
    pts = np.arange(24, dtype=np.float32).reshape(6, 4) + 0.5
    data = np.full((2, 56), 0xAB, np.uint8)
    data[:, :48] = pts.reshape(2, 12).view(np.uint8).reshape(2, 48)
    lay = layout_of([("x", 0, FLOAT32, 1), ("y", 4, FLOAT32, 1), ("z", 8, FLOAT32, 1), ("intensity", 12, FLOAT32, 1)], 16)
    got = decode_rows(data.tobytes(), 3, 2, 56, lay)
    want = np.zeros((6, 8), np.uint32)
    want[:, :3] = f32(pts[:, :3])
    want[:, 3] = ONE_BITS
    want[:, 4] = f32(pts[:, 3])
    assert np.array_equal(got, want)
    assert not np.any(got == 0xABABABAB)


def test_padded_rows_big_endian_and_field_order_known_answer():
    """z y x order, big-endian, intensity UINT8 (left unmapped: 0), rows padded by 3 bytes"""
    pts = np.array([[1.0, -2.0, 3.5], [np.nan, 0.0, -0.0], [1e-40, np.inf, 7.25], [4.0, 5.0, 6.0]], np.float32)
    rows, width, step, pad = 2, 2, 13, 3
    rec = np.zeros((4, step), np.uint8)
    for j, off in ((2, 0), (1, 4), (0, 8)):
        rec[:, off:off + 4] = pts[:, j].astype(">f4").view(np.uint8).reshape(4, 4)
    rec[:, 12] = 200
    data = np.full((rows, width * step + pad), 0x7F, np.uint8)
    data[:, :width * step] = rec.reshape(rows, width * step)
    fields = [("z", 0, FLOAT32, 1), ("y", 4, FLOAT32, 0), ("x", 8, FLOAT32, 1), ("intensity", 12, UINT8, 1)]
    lay = layout_of(fields, step, is_bigendian=True)
    assert lay["off_intensity"] == NO_FIELD
    got = decode_rows(data.tobytes(), width, rows, width * step + pad, lay)
    assert np.array_equal(got[:, :3], pts.view(np.uint32))
    assert np.all(got[:, 3] == ONE_BITS) and np.all(got[:, 4:] == 0)


def test_layout_needs_float32_xyz_and_takes_the_first_match():
    assert layout_of([("x", 0, FLOAT32, 1), ("y", 4, FLOAT32, 1), ("z", 8, 8, 1)], 16) is None  # FLOAT64 z: no match
    assert layout_of([("x", 0, FLOAT32, 1), ("y", 4, FLOAT32, 1)], 16) is None
    assert layout_of([("x", 0, FLOAT32, 2), ("y", 4, FLOAT32, 1), ("z", 8, FLOAT32, 1)], 16) is None  # count 2
    lay = layout_of([("x", 0, FLOAT32, 1), ("x", 12, FLOAT32, 1), ("y", 4, FLOAT32, 1), ("z", 8, FLOAT32, 1)], 16)
    assert lay["off_x"] == 0


def test_message_builder_round_trips():
    rng = np.random.default_rng(3)
    cloud = rng.normal(size=(12, 4)).astype(np.float32)
    for kind in ("velodyne", "ouster"):
        for big in (False, True):
            m = message(cloud, kind=kind, width=4, height=3, pad=5, big=big)
            lay = layout_of(m["fields"], m["point_step"], m["is_bigendian"])
            got = decode_rows(m["data"], m["width"], m["height"], m["row_step"], lay)
            assert np.array_equal(got[:, :3], cloud[:, :3].view(np.uint32)) and np.array_equal(got[:, 4], cloud[:, 3].view(np.uint32))
