"""FloorDetectionNodelet::detect on the device (b2r_floor_detect) timed on clouds resident in HBM (one GPU).

    python tools/floor_time.py [--frames 20] [--reps 3] [--out record.json] [--hypotheses 16,64,256]

Workloads: VLP-16 and HDL-32E scans through b2r_prefilter's defaults, and the KITTI-shaped 120 000-point scan through the 0.25 m voxel
grid; each under the hdl / 501 / kitti launch parameter sets (the kitti set, sensor_height 3.0, on scans lowered by 1.2 m so that its
band holds the ground).  Per workload: the median ms per call over --frames frames (CUDA events around the call; the prefiltered cloud
is already on the device), hypotheses, RANSAC iterations, RANSAC round trips and all readbacks (host waits on device data) per call, and the single-thread CPU time of the
sequential reference (tests/floor_ref.cpp, -O2) on the same host.  Each batch size B2R_FLOOR_HYPOTHESES of --hypotheses runs in a
child process (the switch is read once per process); the card's name and power limit are read in the same call."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SCANS = {"vlp16": ("vlp16", 0.1), "hdl32e": ("hdl32e", 0.1), "kitti": ("kitti", 0.25)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def child(frames, reps):
    import torch
    import hdl_graph_slam_b200 as pkg
    from hdl_graph_slam_b200 import synth
    from floor_ref import LAUNCH, Reference
    ref = Reference(tempfile.mkdtemp())
    reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    out = {}
    for scan, (sensor, leaf) in SCANS.items():
        for launch, kw in LAUNCH.items():
            clouds = []
            for f in range(frames):
                c = synth.scan(sensor, frame=f, stride=8)
                if launch == "kitti":
                    c[:, 2] -= np.float32(1.2)
                host, dptr, m = reg.prefilter(c, want_host=True, downsample_resolution=leaf)
                clouds.append((torch.from_numpy(host).cuda(), m, host))
            torch.cuda.synchronize()
            for t, m, _ in clouds[:3]:  # warm-up
                reg.floor_detect(ptr=t.data_ptr(), n=m, stride_bytes=32, device=True, want_host=False, **kw)
            ms, hyp, it, rt, rb, det = [], [], [], [], [], 0
            for _ in range(reps):
                for t, m, _ in clouds:
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    r = reg.floor_detect(ptr=t.data_ptr(), n=m, stride_bytes=32, device=True, want_host=False, **kw)
                    b.record()
                    b.synchronize()
                    ms.append(a.elapsed_time(b))
                    hyp.append(r["ransac_hypotheses"]); it.append(r["ransac_iterations"]); rt.append(r["ransac_batches"]); rb.append(r["readbacks"])
                    det += r["detected"]
            t0 = time.perf_counter()
            for _, _, host in clouds:
                ref.detect(host, **kw)
            cpu_ms = (time.perf_counter() - t0) * 1e3 / len(clouds)
            out[f"{scan}/{launch}"] = dict(points=int(np.median([m for _, m, _ in clouds])), ms_median=float(np.median(ms)), ms_min=float(np.min(ms)),
                                           hypotheses_median=float(np.median(hyp)), iterations_median=float(np.median(it)),
                                           ransac_round_trips_median=float(np.median(rt)), readbacks_median=float(np.median(rb)), detected_share=det / len(ms), cpu_ref_ms=cpu_ms)
    reg.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--hypotheses", default="16,64,256")
    ap.add_argument("--out")
    ap.add_argument("--child", action="store_true")
    a = ap.parse_args()
    if a.child:
        print(json.dumps(child(a.frames, a.reps)))
        return
    rec = {"tool": "floor_time", "card": card(), "frames": a.frames, "reps": a.reps, "by_hypotheses": {}}
    for b in a.hypotheses.split(","):
        env = dict(os.environ, B2R_FLOOR_HYPOTHESES=b)
        p = subprocess.run([sys.executable, __file__, "--child", "--frames", str(a.frames), "--reps", str(a.reps)], env=env,
                           capture_output=True, text=True, check=True)
        rec["by_hypotheses"][b] = json.loads(p.stdout.strip().splitlines()[-1])
    s = json.dumps(rec)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
