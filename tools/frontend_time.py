"""Per-frame wall clock of the front-end drop-in (hdl_graph_slam_b200/adapter/b200_frontend.hpp) on one GPU, against the CPU
restatements on the same host.

    python tools/frontend_time.py [--frames 10] [--reps 3] [--out record.json]

Workloads: raw VLP-16 (65 536 points), HDL-32E (131 072) and KITTI-shaped (120 000) scans, each under the prefilter rosparams of
launch/hdl_graph_slam{,_400,_501,_kitti}.launch (base_link transform given, no IMU).  A small C++ program built here against the
test-only stand-ins calls the header as the nodelets would and times, with std::chrono around each call:
  - B200Prefilter::filter from a pcl cloud (host records, uploaded by the call);
  - B200Prefilter::filter from a velodyne-style PointCloud2 (x y z intensity ring time, point_step 22), unpacked on the device;
  - B200FloorDetector::detect on the filter's output, with the floor parameters of that launch file (hdl: the 400 file's), no
    filtered or inlier cloud requested.
The CPU columns are single-thread restatements, not PCL: the oracle's distance filter, voxel grid and outlier filters (oracle/) for
the prefilter (without the base_link transform, a per-point affine map), and tests/floor_ref.cpp (-O2) for the floor detector.  nproc and the card's name and power limit are recorded."""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SCANS = {"vlp16": "vlp16", "hdl32e": "hdl32e", "kitti": "kitti"}
FLOOR_OF = {"hdl": "hdl", "400": "hdl", "501": "501", "kitti": "kitti"}
TF = np.array([[1, 0, 0, 0.1], [0, 1, 0, 0.0], [0, 0, 1, 0.0], [0, 0, 0, 1]], np.float32)  # sensor -> base_link: a 0.1 m offset that keeps the synthetic ground in the floor band

PROG = r'''
#include "frontend_shim.hpp"
#include "b200_frontend.hpp"
#include <chrono>
#include <cstdio>
using namespace hdl_graph_slam;
using Cloud = pcl::PointCloud<pcl::PointXYZI>;
static double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
// argv: scans.bin reps; stdin-free: scans.bin holds the rosparams, the transform and the frames
int main(int argc, char** argv) {
  FILE* f = std::fopen(argv[1], "rb");
  const int reps = std::atoi(argv[2]);
  auto geti = [&]() { int32_t v = 0; if (std::fread(&v, 4, 1, f) != 1) std::exit(2); return v; };
  auto gets = [&]() { std::string s(geti(), '\0'); if (!s.empty() && std::fread(&s[0], 1, s.size(), f) != s.size()) std::exit(2); return s; };
  ros::NodeHandle pnh, fnh;
  for (int i = 0, n = geti(); i < n; i++) { std::string k = gets(); pnh.setParam(k, gets()); }
  for (int i = 0, n = geti(); i < n; i++) { std::string k = gets(); fnh.setParam(k, gets()); }
  Eigen::Matrix4f T;
  if (std::fread(T.m, 4, 16, f) != 16) return 2;
  std::vector<Cloud::Ptr> clouds;
  std::vector<sensor_msgs::PointCloud2> msgs;
  for (int i = 0, n = geti(); i < n; i++) {
    Cloud::Ptr c(new Cloud());
    c->points.resize(geti());
    if (std::fread(c->points.data(), 32, c->points.size(), f) != c->points.size()) return 2;
    c->width = c->points.size(); c->height = 1; c->header.frame_id = "velodyne";
    sensor_msgs::PointCloud2 m;
    m.header.frame_id = "velodyne"; m.width = c->points.size(); m.height = 1; m.point_step = 22; m.row_step = 22 * m.width;
    const char* names[6] = {"x", "y", "z", "intensity", "ring", "time"};
    const uint32_t offs[6] = {0, 4, 8, 12, 16, 18};
    const uint8_t types[6] = {7, 7, 7, 7, 4, 7};
    for (int k = 0; k < 6; k++) { sensor_msgs::PointField pf; pf.name = names[k]; pf.offset = offs[k]; pf.datatype = types[k]; pf.count = 1; m.fields.push_back(pf); }
    m.data.assign((size_t)m.row_step, 0);
    for (size_t j = 0; j < c->points.size(); j++) {
      const auto& p = c->points[j];
      std::memcpy(&m.data[22 * j], &p.x, 12);
      std::memcpy(&m.data[22 * j + 12], &p.intensity, 4);
    }
    clouds.push_back(c); msgs.push_back(std::move(m));
  }
  std::fclose(f);
  B200Prefilter prefilter(pnh);
  B200FloorDetector floor(fnh);
  std::vector<double> t_pcl, t_msg, t_floor;
  size_t kept = 0;
  int detected = 0;
  for (int r = -1; r < reps; r++) {  // r = -1: warm-up
    for (size_t i = 0; i < clouds.size(); i++) {
      double a = now_ms();
      Cloud::ConstPtr out = prefilter.filter(Cloud::ConstPtr(clouds[i]), nullptr, &T);
      double b = now_ms();
      Cloud::ConstPtr out2 = prefilter.filter(msgs[i], nullptr, &T);
      double c = now_ms();
      Cloud::Ptr in(new Cloud(*out));
      double d = now_ms();
      auto coeffs = floor.detect(in, false, false);
      double e = now_ms();
      if (r < 0) continue;
      t_pcl.push_back(b - a); t_msg.push_back(c - b); t_floor.push_back(e - d);
      kept += out->points.size();
      detected += coeffs ? 1 : 0;
      if (out2->points.size() != out->points.size()) return 4;
    }
  }
  std::printf("{\"kept_mean\": %g, \"detected\": %d, \"pcl_ms\": [", (double)kept / t_pcl.size(), detected);
  for (size_t i = 0; i < t_pcl.size(); i++) std::printf("%s%.4f", i ? ", " : "", t_pcl[i]);
  std::printf("], \"msg_ms\": [");
  for (size_t i = 0; i < t_msg.size(); i++) std::printf("%s%.4f", i ? ", " : "", t_msg[i]);
  std::printf("], \"floor_ms\": [");
  for (size_t i = 0; i < t_floor.size(); i++) std::printf("%s%.4f", i ? ", " : "", t_floor[i]);
  std::printf("]}\n");
  return 0;
}
'''


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def build(tmp):
    from hdl_graph_slam_b200 import build as b
    b.build_engine()
    src = os.path.join(tmp, "frontend_time.cpp")
    with open(src, "w") as f:
        f.write(PROG)
    exe = os.path.join(tmp, "frontend_time")
    lib = os.path.join(ROOT, "hdl_graph_slam_b200", "_lib")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++14", "-O2", "-include", "cstring",
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "hdl_graph_slam_b200", "adapter"), "-o", exe, src,
                           "-L", lib, "-lb200reg", "-Wl,-rpath," + lib, "-pthread"])
    return exe


def kv(d):
    return struct.pack("<i", len(d)) + b"".join(struct.pack("<i", len(k)) + k.encode() + struct.pack("<i", len(str(v))) + str(v).encode()
                                                   for k, v in d.items())


def cpu_prefilter(orc, c, ros):
    """the oracle's stage-wise chain under the launch parameters (single thread)"""
    x = c[orc.distance_filter(c, float(ros["distance_near_thresh"]), float(ros["distance_far_thresh"]))]
    if ros["downsample_method"] == "VOXELGRID":
        v = orc.voxelgrid(x, float(ros["downsample_resolution"]))[0]
        x = np.zeros((v.shape[0], 8), np.float32)
        x[:, :3], x[:, 3], x[:, 4] = v[:, :3], 1.0, v[:, 3]
    if ros["outlier_removal_method"] == "RADIUS":
        x = x[orc.radius_outlier(x, float(ros["radius_radius"]), int(ros["radius_min_neighbors"]), threads=1)]
    elif ros["outlier_removal_method"] == "STATISTICAL":
        x = x[orc.statistical_outlier(x, int(ros["statistical_mean_k"]), float(ros["statistical_stddev"]), threads=1)[0]]
    return x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    from hdl_graph_slam_b200 import build as b
    b.build_synth()
    from hdl_graph_slam_b200 import synth
    from oracle import oracle as orc
    orc.build()
    orc.lib()
    from floor_ref import LAUNCH as FLOOR_LAUNCH, Reference
    from test_frontend_adapter_gpu import PREFILTER_LAUNCH
    tmp = tempfile.mkdtemp(prefix="frontend_time_")
    exe = build(tmp)
    ref = Reference(tmp)
    rec = {"tool": "frontend_time", "card": card(), "nproc": os.cpu_count(), "frames": a.frames, "reps": a.reps,
           "timer": "std::chrono around each header call (wall clock, includes H2D / D2H)",
           "cpu_note": "single-thread restatements on the same host (oracle prefilter chain, tests/floor_ref.cpp), not PCL", "workloads": {}}
    for scan, sensor in SCANS.items():
        clouds = [synth.scan(sensor, frame=f, stride=8) for f in range(a.frames)]
        for launch in ("hdl", "400", "501", "kitti"):
            ros = PREFILTER_LAUNCH[launch]
            fros = {k: ("true" if v else "false") if k == "use_normal_filtering" else str(v) for k, v in FLOOR_LAUNCH[FLOOR_OF[launch]].items()}
            body = kv(ros) + kv(fros) + TF.T.astype(np.float32).tobytes() + struct.pack("<i", len(clouds))
            body += b"".join(struct.pack("<i", c.shape[0]) + np.ascontiguousarray(c, np.float32).tobytes() for c in clouds)
            path = os.path.join(tmp, "scans.bin")
            with open(path, "wb") as f:
                f.write(body)
            p = subprocess.run([exe, path, str(a.reps)], capture_output=True, text=True, timeout=1800)
            if p.returncode != 0:
                raise SystemExit(f"{scan}/{launch}: exit {p.returncode}\n{p.stderr}")
            g = json.loads(p.stdout.strip().splitlines()[-1])
            cpu_pf, cpu_fd = [], []
            for c in clouds:
                t0 = time.perf_counter()
                x = cpu_prefilter(orc, c, ros)
                t1 = time.perf_counter()
                ref.detect(x, **FLOOR_LAUNCH[FLOOR_OF[launch]])
                t2 = time.perf_counter()
                cpu_pf.append((t1 - t0) * 1e3)
                cpu_fd.append((t2 - t1) * 1e3)
            rec["workloads"][f"{scan}/{launch}"] = dict(
                points=int(clouds[0].shape[0]), kept_mean=g["kept_mean"], detected=g["detected"],
                filter_pcl_ms_median=float(np.median(g["pcl_ms"])), filter_pcl_ms_min=float(np.min(g["pcl_ms"])),
                filter_msg_ms_median=float(np.median(g["msg_ms"])), filter_msg_ms_min=float(np.min(g["msg_ms"])),
                detect_ms_median=float(np.median(g["floor_ms"])), detect_ms_min=float(np.min(g["floor_ms"])),
                cpu_restatement_prefilter_ms_median=float(np.median(cpu_pf)), cpu_restatement_floor_ms_median=float(np.median(cpu_fd)))
            print(scan, launch, json.dumps(rec["workloads"][f"{scan}/{launch}"]), flush=True)
    s = json.dumps(rec)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
