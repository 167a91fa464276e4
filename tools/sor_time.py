"""Time the statistical outlier filter (b2r_prefilter with only that stage, mean_k 20, stddev_mul 1.0) on clouds resident in HBM,
and the k_sor_stats kernel alone (development aid, not part of bench.py).  The "_wide" clouds take the kernel's index-order path:

    python tools/sor_time.py [--steps 100] [--warmup 10] [--rounds 5] [--out record.json]

A call's time is CUDA-event time on the handle's stream (b2r_get_stream) over `steps` back-to-back calls, each ending with the
engine's one host round trip (the output count); the median of `rounds` blocks is reported.  The kernel's own time comes from a
separate torch.profiler pass.  The card's name and power limit are read in the same run.  B2R_LIB selects another build of the
library, so two builds are compared by running this once per build."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import hdl_graph_slam_b200 as pkg  # noqa: E402
from hdl_graph_slam_b200 import _capi, synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,driver_version", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable: " + torch.cuda.get_device_name(0)


def workloads():
    vlp = synth.scan("vlp16", frame=0, stride=8)
    parts = []
    for f in range(10):
        c = synth.scan("kitti", frame=f, stride=8)
        T = synth.pose_matrix(f).astype(np.float32)
        c[:, :3] = (c[:, :3] @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
        parts.append(c)
    kmap = np.concatenate(parts)
    # the same clouds with 300 points spread over a 4 km cube and a 1 mm cluster of 200: mean distances over so many binades that
    # k_sor_stats' exactness bound fails and it sums on one thread in index order (its slow path)
    rng = np.random.default_rng(17)
    extra = np.zeros((500, 8), np.float32)
    extra[:300, :3] = rng.uniform(-2000, 2000, (300, 3))
    extra[300:, :3] = np.array([5.0, -7.0, 1.0]) + rng.uniform(0, 1e-3, (200, 3))
    extra[:, 3] = 1.0
    return [("vlp16_25k", vlp[:25000].copy()), ("vlp16_40k", vlp[:40000].copy()), ("kitti_map_1.2M", kmap),
            ("vlp16_25k_wide", np.concatenate([vlp[:24500], extra])), ("kitti_map_1.2M_wide", np.concatenate([kmap[:-500], extra]))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to time")
    rec = dict(card=card(), library=os.path.relpath(_capi.LIB_PATH, os.path.dirname(os.path.dirname(os.path.abspath(__file__)))),
               steps=a.steps, warmup=a.warmup, rounds=a.rounds, clouds={})
    reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    stream = torch.cuda.ExternalStream(reg.getStream())
    pre = dict(use_distance_filter=0, downsample_method=0, outlier_removal_method=1, statistical_mean_k=20, statistical_stddev=1.0)
    for name, cloud in workloads():
        d = torch.from_numpy(cloud).cuda()
        torch.cuda.synchronize()

        def call():
            return reg.prefilter_raw(d.data_ptr(), d.shape[0], d.shape[1] * 4, device=True, **pre)

        kept = call()[2]
        for _ in range(a.warmup):
            call()
        blocks = []
        for _ in range(a.rounds):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(stream):
                s.record(stream)
                for _ in range(a.steps):
                    call()
                e.record(stream)
            e.synchronize()
            blocks.append(s.elapsed_time(e) * 1e3 / a.steps)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                call()
            torch.cuda.synchronize()
        kern = {ev.key: ev.device_time_total / ev.count for ev in prof.key_averages() if "k_sor_stats" in ev.key or "k_knn_stat" in ev.key}
        r = dict(points=int(cloud.shape[0]), kept=int(kept), call_median_us=float(np.median(blocks)), call_min_us=float(np.min(blocks)),
                 call_max_us=float(np.max(blocks)), kernel_us={k.split("(")[0]: float(v) for k, v in kern.items()})
        rec["clouds"][name] = r
        print(name, json.dumps(r), flush=True)
    reg.close()
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
