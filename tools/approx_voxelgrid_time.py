"""Time b2r_approximate_voxelgrid_device against b2r_voxelgrid_device, and b2r_prefilter under both downsample methods, on the same
seeded inputs resident in HBM (development aid, not part of bench.py):

    python tools/approx_voxelgrid_time.py [--steps 300] [--warmup 30] [--rounds 5] [--out record.json]

Each call ends with the engine's one host round trip (the output count), so a call's time is CUDA-event time on the handle's stream
(b2r_get_stream) over `steps` back-to-back calls.  The two methods alternate in `rounds` blocks; the median block is reported.  The
card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import hdl_graph_slam_b200 as pkg  # noqa: E402
from hdl_graph_slam_b200 import synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,driver_version", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable: " + torch.cuda.get_device_name(0)


def workloads():
    kitti = synth.scan("kitti", frame=0, stride=8)
    vlp = synth.scan("vlp16", frame=0, stride=8)
    parts = []
    for f in range(10):
        c = synth.scan("kitti", frame=f, stride=8)
        T = synth.pose_matrix(f).astype(np.float32)
        c[:, :3] = (c[:, :3] @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
        parts.append(c)
    return [("kitti_raw_120k", kitti, 0.25), ("vlp16_64k", vlp, 0.1), ("map_1.2M", np.concatenate(parts), 0.25)]


def time_calls(stream, fn, steps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        s.record(stream)
        for _ in range(steps):
            fn()
        e.record(stream)
    e.synchronize()
    return s.elapsed_time(e) * 1e3 / steps  # us per call


def ab(stream, fns, steps, warmup, rounds):
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    t = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            t[k].append(time_calls(stream, fn, steps))
    return {k: dict(median_us=float(np.median(v)), min_us=float(np.min(v)), max_us=float(np.max(v))) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to time")
    rec = dict(card=card(), steps=a.steps, warmup=a.warmup, rounds=a.rounds, filters={}, prefilter={})
    reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    stream = torch.cuda.ExternalStream(reg.getStream())
    for name, cloud, leaf in workloads():
        d = torch.from_numpy(cloud).cuda()
        torch.cuda.synchronize()
        p, n, sb = d.data_ptr(), d.shape[0], d.shape[1] * 4
        m_vg = reg.voxelGridFilterDevice(p, n, sb, leaf)[1]
        m_avg = reg.approximateVoxelGridFilterDevice(p, n, sb, leaf)[1]
        r = ab(stream, {"voxelgrid": lambda: reg.voxelGridFilterDevice(p, n, sb, leaf),
                        "approx_voxelgrid": lambda: reg.approximateVoxelGridFilterDevice(p, n, sb, leaf)}, a.steps, a.warmup, a.rounds)
        r.update(points=n, leaf=leaf, outputs_voxelgrid=m_vg, outputs_approx_voxelgrid=m_avg)
        rec["filters"][name] = r
        print(name, json.dumps(r), flush=True)
    # the KITTI per-scan prefilter (bench.py's kitti_pipeline parameters) under both downsample methods
    raw = torch.from_numpy(workloads()[0][1]).cuda()
    torch.cuda.synchronize()
    pre = dict(use_distance_filter=1, distance_near_thresh=0.1, distance_far_thresh=100.0, downsample_resolution=0.25, outlier_removal_method=2,
               radius_radius=0.5, radius_min_neighbors=2)
    fns = {}
    for method, key in ((pkg.B2R_DOWNSAMPLE_VOXELGRID, "voxelgrid"), (pkg.B2R_DOWNSAMPLE_APPROX_VOXELGRID, "approx_voxelgrid")):
        fns[key] = (lambda mth: lambda: reg.prefilter_raw(raw.data_ptr(), raw.shape[0], raw.shape[1] * 4, device=True, downsample_method=mth, **pre))(method)
    r = ab(stream, fns, max(a.steps // 3, 1), a.warmup, a.rounds)
    r.update(points=raw.shape[0], outputs_voxelgrid=fns["voxelgrid"]()[2], outputs_approx_voxelgrid=fns["approx_voxelgrid"]()[2])
    rec["prefilter"]["kitti_raw_120k"] = r
    print("prefilter", json.dumps(r), flush=True)
    reg.close()
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
