"""Per-frame wall clock of the odometry drop-in (hdl_graph_slam_b200/adapter/b200_odometry.hpp) on one GPU, against the raw mirror on
the same frames.

    python tools/odometry_adapter_time.py [--frames 120] [--warmup 10] [--rounds 3] [--out record.json]

Workload: a walk of raw VLP-16 scans (65 536 points, 0.3 m apart) under launch/hdl_graph_slam.launch's odometry rosparams (FAST_GICP,
downsample NONE).  tests/odometry_harness.cpp, built here against the test-only stand-ins, calls B200ScanMatchingOdometry::matching as
the nodelet would and times each call with std::chrono (H2D and D2H copies included):
  - pcl:      from a pcl cloud (host records, uploaded by the call);
  - msg:      from a velodyne-style PointCloud2 (x y z intensity ring time, point_step 22), unpacked on the device;
  - each with want_status and want_aligned off, and both on (the status and the aligned cloud copied back every frame).
  - raw:      b2r_odometry_matching through the Python mirror on the same frames (publish_status off), a perf_counter around each call.
The arms alternate, round by round; each round is a fresh odometry over the whole walk, and its first `warmup` frames are not
recorded.  The card's name, power limit and max SM clock are recorded from nvidia-smi in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

ROS = dict(registration_method="FAST_GICP", reg_num_threads="0", reg_maximum_iterations="64", reg_max_optimizer_iterations="20",
           reg_use_reciprocal_correspondences="false", reg_correspondence_randomness="20", reg_resolution="1.0", reg_nn_search_method="DIRECT7",
           odom_frame_id="odom", keyframe_delta_trans="1.0", keyframe_delta_angle="1.0", keyframe_delta_time="10000.0",
           transform_thresholding="false", max_acceptable_trans="1.0", max_acceptable_angle="1.0", downsample_method="NONE",
           downsample_resolution="0.1", reg_transformation_epsilon="0.01", reg_max_correspondence_distance="2.5")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stats(ns):
    ms = np.asarray(ns, np.float64) / 1e6
    return dict(median_ms=float(np.median(ms)), p10_ms=float(np.percentile(ms, 10)), p90_ms=float(np.percentile(ms, 90)), n=int(ms.size))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    import hdl_graph_slam_b200 as pkg
    from hdl_graph_slam_b200 import build, synth
    from frontend_ref import message
    from odometry_adapter_io import ODOMETRY, build_harness, encode_call, msg_input, pcl_input, run_jobs
    build.build_all()
    tmp = Path(tempfile.mkdtemp(prefix="odometry_adapter_time_"))
    harness = build_harness(tmp / "odometry_harness")
    frames = [synth.scan("vlp16", frame=k, step=0.3, stride=8) for k in range(a.frames)]
    msgs = [message(f[:, [0, 1, 2, 4]], kind="velodyne", seed=k) for k, f in enumerate(frames)]
    stamps = [((1436939143_000_000_000 + k * 100_000_000) // 10**9, (1436939143_000_000_000 + k * 100_000_000) % 10**9) for k in range(a.frames)]
    arms = {}
    for inp in ("pcl", "msg"):
        for extra in (False, True):
            name = f"{inp}_{'status_aligned' if extra else 'plain'}"
            src = (lambda k: pcl_input(frames[k])) if inp == "pcl" else (lambda k: msg_input(msgs[k], True))
            arms[name] = [encode_call(ODOMETRY, src(k), stamps[k], want_status=extra, want_aligned=extra) for k in range(a.frames)]
    times = {n: [] for n in list(arms) + ["raw"]}
    poses = {}
    for r in range(a.rounds):
        for name, calls in arms.items():
            (ans,), _, (t,) = run_jobs(harness, tmp, [(ODOMETRY, ROS, calls)], times=True)
            times[name] += t[a.warmup:].tolist()
            poses[name] = np.stack([x["odom"] for x in ans])
        reg = pkg.select_registration_method({k: v for k, v in ROS.items() if k == "registration_method" or k.startswith("reg_")})
        odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=1.0, keyframe_delta_angle=1.0, keyframe_delta_time=10000.0)
        raw = []
        for k, f in enumerate(frames):
            t0 = time.perf_counter_ns()
            st = odo.matching(float(stamps[k][0]) + 1e-9 * float(stamps[k][1]), f)
            if k >= a.warmup:
                times["raw"].append(time.perf_counter_ns() - t0)
            raw.append(st["odom"])
        odo.close()
        reg.close()
        poses["raw"] = np.stack(raw)
    same = {n: bool(np.array_equal(poses[n].view(np.uint32), poses["raw"].view(np.uint32))) for n in poses}
    rec = dict(tool="odometry_adapter_time", card=card(), nproc=os.cpu_count(), frames=a.frames, warmup=a.warmup, rounds=a.rounds,
               points_per_frame=int(frames[0].shape[0]), arms={n: stats(t) for n, t in times.items()}, poses_equal_raw=same)
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
