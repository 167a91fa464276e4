"""The factory's `GICP_OMP` branch (B2R_METHOD_GICP_OMP, pclomp::GeneralizedIterativeClosestPoint, `B200_GICP_OMP`) timed beside `GICP`
(pcl::GeneralizedIterativeClosestPoint) and FAST_GICP on one GPU.

    python tools/gicp_omp_time.py [--frames 20] [--groups 8] [--reps 3] [--out profiles/h100/gicp_omp_time_1.json]

  odometry   ScanMatchingOdometry over --frames VLP-16 frames of 65 536 points, the three methods alternated rep by rep, from host clouds
             and from clouds resident in device memory (HBM); median ms per frame, and for GICP_OMP and GICP the outer iterations,
             correspondence passes and cost passes per registration (each pass is one host round trip: the BFGS runs on the host)
  loop       LoopDetector::matching (b2r_loop_matching) over --groups new keyframes x 8 candidates (VLP-16, 65 536 points): each
             keyframe's candidates as one device batch; median seconds, pairs/s
Prints one JSON record; the card's name, power limit and clocks are read in the same call.  No speed-up is assumed."""
import argparse
import json
import os
import subprocess
import sys
import time
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
import hdl_graph_slam_b200 as pkg  # noqa: E402
from hdl_graph_slam_b200 import synth  # noqa: E402

METHODS = {"GICP_OMP": {"registration_method": "B200_GICP_OMP"}, "GICP": {"registration_method": "GICP"},
           "FAST_GICP": {"registration_method": "FAST_GICP"}}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem,driver_version", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def odometry(frames, dframes, name):
    reg = pkg.select_registration_method(METHODS[name])
    odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=0.25)
    n = frames[0].shape[0]

    def match(k):
        if dframes is None:
            return odo.matching(0.1 * k, frames[k])
        return odo.matching_raw(0.1 * k, dframes[k].data_ptr(), n, 16, device=True)
    match(0)
    reg.getStats(reset=True)
    t, iters = [], []
    for k in range(1, len(frames)):
        t0 = time.perf_counter()
        st = match(k)
        t.append(time.perf_counter() - t0)
        iters.append(st["iterations"])
    launches = reg.getStats()["launches"]
    odo.close()
    reg.close()
    m = len(frames) - 1
    work = {"outer_iterations_per_registration": float(np.mean(iters))}
    if name != "FAST_GICP":
        work.update({"correspondence_passes_per_registration": launches["gicp_pcl_correspondences"] / m,
                     "cost_passes_per_registration": launches["gicp_pcl_cost"] / m})
    return float(np.median(t)) * 1e3, work


def loop(name, groups):
    reg = pkg.select_registration_method(METHODS[name])
    det = pkg.LoopDetector(reg, fitness_score_max_range=2.5)
    t0 = time.perf_counter()
    conv = 0
    for tgt, cands, guesses in groups:
        _, res = det.matching(cands, tgt, guesses)
        conv += sum(r["converged"] for r in res)
    dt = time.perf_counter() - t0
    reg.close()
    return dt, conv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--groups", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    rec = {"tool": "gicp_omp_time", "card": card()}
    frames = [np.ascontiguousarray(synth.scan("vlp16", frame=k), np.float32) for k in range(a.frames)]
    dframes = [torch.from_numpy(f).cuda() for f in frames]
    torch.cuda.synchronize()
    odo = {f"{m}_{src}": [] for m in METHODS for src in ("host", "hbm")}
    work = {}
    for _ in range(a.reps):
        for m in METHODS:
            for src in ("host", "hbm"):
                ms, w = odometry(frames, dframes if src == "hbm" else None, m)
                odo[f"{m}_{src}"].append(ms)
                work[m] = w
    rec["odometry"] = {"points_per_frame": int(frames[0].shape[0]), "frames": a.frames,
                       **{f"{k}_ms_per_frame": float(np.median(v)) for k, v in odo.items()}, "all_ms": odo, "work": work}
    # loop candidates: new keyframe f, candidates f - 8 .. f - 1 with the identity guess (neighbouring frames of the same drive)
    groups = []
    for g in range(a.groups):
        f = 8 + 9 * g
        groups.append((synth.scan("vlp16", frame=f), [synth.scan("vlp16", frame=f - 1 - c) for c in range(8)], [np.eye(4, dtype=np.float32)] * 8))
    for m in METHODS:
        loop(m, groups[:1])  # warm-up
    tl = {m: [] for m in METHODS}
    conv = {}
    for _ in range(a.reps):
        for m in METHODS:
            dt, conv[m] = loop(m, groups)
            tl[m].append(dt)
    pairs = 8 * a.groups
    rec["loop"] = {"pairs": pairs, "group": 8, "sensor": "vlp16", "points_per_cloud": int(groups[0][0].shape[0]),
                   **{m: {"s": float(np.median(tl[m])), "all_s": tl[m], "pairs_per_s": pairs / float(np.median(tl[m])), "converged": int(conv[m])}
                      for m in METHODS}}
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
