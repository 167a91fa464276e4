"""NDT loop-closure candidates through the device batch vs the sequential single-handle loop (one GPU).

    python tools/ndt_batch_time.py [--groups 32] [--sensor vlp16] [--res 1.0] [--reps 3] [--out record.json]

Workload: loop_workload(groups) of hdl_graph_slam_b200.batch (GROUP = 8 candidates per new keyframe, VLP-16 scans), NDT_OMP at
the given resolution, DIRECT7.  Arms, alternated rep by rep on the same pairs:
  batch       b2r_batch_align(want_fitness) over all pairs (clouds added once, outside the timed window)
  sequential  the reference's LoopDetector::matching walk on one handle: setInputTarget per group, then setInputSource / align /
              getFitnessScore per candidate (clouds uploaded inside the window, as the walk does)
Prints one JSON record: per-arm median seconds, pairs/s, batched rounds, and whether every pair is bitwise equal across arms.
The card's name, power limit and clocks are read in the same call."""
import argparse
import json
import os
import subprocess
import sys
import time
import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import hdl_graph_slam_b200 as pkg  # noqa: E402
from hdl_graph_slam_b200 import synth  # noqa: E402
from hdl_graph_slam_b200.batch import loop_workload  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem,driver_version", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=32)
    ap.add_argument("--sensor", default="vlp16")
    ap.add_argument("--res", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-range", type=float, default=2.5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    groups, guesses, group_first = loop_workload(a.groups, a.sensor)
    frames = sorted({f for tf, sfs in groups for f in [tf] + list(sfs)})
    clouds = {f: synth.scan(a.sensor, frame=f, stride=8) for f in frames}
    pairs = [(sf, tf) for tf, sfs in groups for sf in sfs]
    cfg = pkg.default_config(pkg.B2R_METHOD_NDT)
    cfg.ndt_resolution = a.res
    cfg.ndt_search_method = 7
    lb = pkg.RegistrationBatch(cfg=cfg)
    ids = {f: lb.addCloud(c) for f, c in clouds.items()}
    pl = [(ids[s], ids[t], guesses[i]) for i, (s, t) in enumerate(pairs)]
    reg = pkg.Registration(cfg)

    def run_batch():
        t0 = time.perf_counter()
        res = lb.align(pl, True, a.max_range)
        return time.perf_counter() - t0, res

    def run_seq():
        out = []
        t0 = time.perf_counter()
        for tf, sfs in groups:
            reg.setInputTarget(clouds[tf])
            for sf in sfs:
                i = len(out)
                reg.setInputSource(clouds[sf])
                reg.align(guesses[i])
                out.append({"T": reg.getFinalTransformation(), "converged": reg.hasConverged(), "iterations": reg.nr_iterations,
                            "fitness": reg.getFitnessScore(a.max_range)})
        return time.perf_counter() - t0, out

    run_batch(); run_seq()  # warm-up: voxel maps, workspaces, module loads
    tb, ts = [], []
    equal = True
    for _ in range(a.reps):
        t, rb = run_batch(); tb.append(t)
        rounds, pair_passes = lb.lastRounds()
        t, rs = run_seq(); ts.append(t)
        for x, y in zip(rb, rs):
            equal &= bool(np.array_equal(np.asarray(x["T"]).view(np.uint32), np.asarray(y["T"]).view(np.uint32)) and
                          bool(x["converged"]) == bool(y["converged"]) and x["iterations"] == y["iterations"] and
                          np.float64(x["fitness"]).tobytes() == np.float64(y["fitness"]).tobytes())
    n = len(pairs)
    rec = {"tool": "ndt_batch_time", "card": card(), "pairs": n, "group": 8, "sensor": a.sensor, "points_per_cloud": int(clouds[frames[0]].shape[0]),
           "resolution": a.res, "search": "DIRECT7", "reps": a.reps,
           "batch_s": float(np.median(tb)), "sequential_s": float(np.median(ts)), "batch_all_s": tb, "sequential_all_s": ts,
           "batch_pairs_per_s": n / float(np.median(tb)), "sequential_pairs_per_s": n / float(np.median(ts)),
           "speedup": float(np.median(ts) / np.median(tb)), "batched_rounds": int(rounds), "pair_passes": int(pair_passes),
           "bitwise_equal": bool(equal)}
    reg.close()
    lb.close()
    line = json.dumps(rec)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
