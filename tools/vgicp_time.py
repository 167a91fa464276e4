"""The factory's `FAST_VGICP` branch (B2R_METHOD_VGICP) timed beside FAST_GICP on one GPU.

    python tools/vgicp_time.py [--frames 40] [--groups 256] [--reps 3] [--out profiles/h100/vgicp_1.json]

  odometry   ScanMatchingOdometry over --frames VLP-16 frames of 65 536 points (the bench.py workload's sensor and size), FAST_VGICP at
             reg_resolution 1.0 and FAST_GICP alternated rep by rep, each end to end from host clouds and HBM-resident (device clouds,
             b2r_odometry_matching_device); median ms per frame, then one profiled pass per method: per-kernel-class ms per frame
             (b2r_set_profiling, CUDA events)
  loop       --groups x 8 loop candidates (hdl_graph_slam_b200.batch.loop_workload, VLP-16; 2048 pairs by default): b2r_batch_align
             with fitness for both methods after one untimed pass over every pair, reps alternated between the methods; median seconds,
             pairs/s, and per-kernel-class ms of one further profiled pass
Prints one JSON record; the card's name, power limit and clocks are read in the same call.  No speed-up is assumed: the record
holds both methods' numbers as measured."""
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
from hdl_graph_slam_b200.batch import loop_workload  # noqa: E402

METHODS = {"FAST_VGICP": {"registration_method": "FAST_VGICP", "reg_resolution": "1.0"}, "FAST_GICP": {"registration_method": "FAST_GICP"}}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem,driver_version", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def odometry(frames, dev, name, device, profile=False):
    reg = pkg.select_registration_method(METHODS[name])
    odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=0.25)
    stride = frames[0].shape[1] * 4
    run = (lambda k, t: odo.matching_raw(t, dev[k].data_ptr(), frames[k].shape[0], stride, device=True)) if device else \
        (lambda k, t: odo.matching(t, frames[k]))
    run(0, 0.0)
    if profile:
        reg.getStats(reset=True)
        reg.setProfiling(True)
    t = []
    for k in range(1, len(frames)):
        t0 = time.perf_counter()
        run(k, 0.1 * k)
        t.append(time.perf_counter() - t0)
    stats = reg.getStats() if profile else None
    odo.close()
    reg.close()
    if profile:
        n = len(frames) - 1
        return {c: ms / n for c, ms in stats["ms"].items() if ms > 0}
    return float(np.median(t)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--groups", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-range", type=float, default=2.5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    rec = {"tool": "vgicp_time", "card": card()}
    frames = [synth.scan("vlp16", frame=k) for k in range(a.frames)]
    dev = [torch.from_numpy(f).cuda() for f in frames]
    torch.cuda.synchronize()
    odo = {f"{m}_{w}": [] for m in METHODS for w in ("host", "hbm")}
    for _ in range(a.reps):
        for m in METHODS:
            odo[f"{m}_host"].append(odometry(frames, dev, m, False))
            odo[f"{m}_hbm"].append(odometry(frames, dev, m, True))
    rec["odometry"] = {"points_per_frame": int(frames[0].shape[0]), "frames": a.frames,
                       **{f"{k}_ms_per_frame": float(np.median(v)) for k, v in odo.items()}, "all_ms": odo,
                       "kernel_ms_per_frame_hbm": {m: odometry(frames, dev, m, True, profile=True) for m in METHODS}}
    groups, guesses, group_first = loop_workload(a.groups, "vlp16")
    lf = sorted({f for tf, sfs in groups for f in [tf] + list(sfs)})
    clouds = {f: synth.scan("vlp16", frame=f, stride=8) for f in lf}
    pairs = [(sf, tf) for tf, sfs in groups for sf in sfs]
    # both batches hold every cloud; a full untimed pass builds every structure (and every VGICP target's voxel map), then the timed
    # reps alternate between the methods
    lbs, pls, tb, res, fit_ms = {}, {}, {m: [] for m in METHODS}, {}, {}
    for m in METHODS:
        lbs[m] = pkg.RegistrationBatch(params=METHODS[m])
        ids = {f: lbs[m].addCloud(c) for f, c in clouds.items()}
        pls[m] = [(ids[s], ids[t], guesses[i]) for i, (s, t) in enumerate(pairs)]
        lbs[m].align(pls[m], True, a.max_range)
    for _ in range(a.reps):
        for m in METHODS:
            t0 = time.perf_counter()
            res[m] = lbs[m].align(pls[m], True, a.max_range)
            tb[m].append(time.perf_counter() - t0)
    for m in METHODS:  # one profiled pass (CUDA events per kernel class), apart from the timed ones
        eng = lbs[m].engine
        eng.setProfiling(True)
        eng.getStats(reset=True)
        lbs[m].align(pls[m], True, a.max_range)
        fit_ms[m] = {c: v for c, v in eng.getStats()["ms"].items() if v > 0}
        eng.setProfiling(False)
    loop = {}
    for m in METHODS:
        lbs[m].close()
        loop[m] = {"batch_s": float(np.median(tb[m])), "all_s": tb[m], "pairs_per_s": len(pairs) / float(np.median(tb[m])),
                   "converged": int(sum(bool(r["converged"]) for r in res[m])), "kernel_ms_per_pass": fit_ms[m]}
    rec["loop"] = {"pairs": len(pairs), "group": 8, "sensor": "vlp16", "points_per_cloud": int(clouds[lf[0]].shape[0]), **loop}
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
