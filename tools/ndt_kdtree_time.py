"""NDT_OMP's KDTREE search (B2R_METHOD_NDT_KDTREE, `B200_NDT_KDTREE`) timed beside NDT_OMP DIRECT7 and the factory's `NDT` (one GPU).

    python tools/ndt_kdtree_time.py [--frames 20] [--groups 32] [--reps 3] [--out record.json]

  odometry   ScanMatchingOdometry over --frames HDL-32E frames of 131 072 points, resolution 1.0, exactly 30 iterations per frame
             (ndt_fixed_iterations), keyframe every 1 m; B200_NDT_KDTREE, NDT_OMP DIRECT7 and NDT alternated rep by rep; median ms per frame
  loop       --groups x 8 B200_NDT_KDTREE loop candidates (hdl_graph_slam_b200.batch.loop_workload, VLP-16): b2r_batch_align against the
             sequential single-handle LoopDetector::matching walk; median seconds, pairs/s and whether every pair is bitwise equal
Prints one JSON record; the card's name, power limit and clocks are read in the same call."""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem,driver_version", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def cfg_of(method, res, fixed=0):
    c = pkg.default_config(method)
    c.ndt_resolution = res
    c.ndt_search_method = 7
    c.ndt_fixed_iterations = fixed
    return c


def odometry(frames, method):
    reg = pkg.Registration(cfg_of(method, 1.0, 30))
    odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=1.0, keyframe_delta_angle=1.0, keyframe_delta_time=10000.0)
    odo.matching(0.0, frames[0])
    t = []
    for k in range(1, len(frames)):
        t0 = time.perf_counter()
        st = odo.matching(0.1 * k, frames[k])
        t.append(time.perf_counter() - t0)
        assert st["iterations"] == 30
    odo.close()
    reg.close()
    return float(np.median(t)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--groups", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-range", type=float, default=2.5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rec = {"tool": "ndt_kdtree_time", "card": card()}
    # ---- odometry
    frames = [synth.scan("hdl32e", frame=k, stride=8) for k in range(a.frames)]
    odo = {"KDTREE": [], "NDT_OMP": [], "NDT": []}
    for _ in range(a.reps):
        odo["KDTREE"].append(odometry(frames, pkg.B2R_METHOD_NDT_KDTREE))
        odo["NDT_OMP"].append(odometry(frames, pkg.B2R_METHOD_NDT))
        odo["NDT"].append(odometry(frames, pkg.B2R_METHOD_NDT_PCL))
    rec["odometry"] = {"points_per_frame": int(frames[0].shape[0]), "resolution": 1.0, "iterations_per_frame": 30, "frames": a.frames,
                       "ndt_kdtree_ms_per_frame": float(np.median(odo["KDTREE"])), "ndt_omp_direct7_ms_per_frame": float(np.median(odo["NDT_OMP"])),
                       "ndt_ms_per_frame": float(np.median(odo["NDT"])), "ndt_kdtree_all_ms": odo["KDTREE"], "ndt_omp_all_ms": odo["NDT_OMP"],
                       "ndt_all_ms": odo["NDT"]}
    # ---- loop batch
    groups, guesses, group_first = loop_workload(a.groups, "vlp16")
    lf = sorted({f for tf, sfs in groups for f in [tf] + list(sfs)})
    clouds = {f: synth.scan("vlp16", frame=f, stride=8) for f in lf}
    pairs = [(sf, tf) for tf, sfs in groups for sf in sfs]
    cfg = cfg_of(pkg.B2R_METHOD_NDT_KDTREE, 1.0)
    lb = pkg.RegistrationBatch(cfg=cfg)
    ids = {f: lb.addCloud(c) for f, c in clouds.items()}
    pl = [(ids[s], ids[t], guesses[i]) for i, (s, t) in enumerate(pairs)]
    reg = pkg.Registration(cfg)
    tb, ts = [], []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        res_b = lb.align(pl, True, a.max_range)
        tb.append(time.perf_counter() - t0)
        out = []
        t0 = time.perf_counter()
        for g in range(len(groups)):
            reg.setInputTarget(clouds[groups[g][0]])
            for i in range(group_first[g], group_first[g + 1]):
                reg.setInputSource(clouds[pairs[i][0]])
                reg.align(guesses[i])
                out.append((reg.getFinalTransformation(), reg.hasConverged(), reg.nr_iterations, reg.getFitnessScore(a.max_range)))
        ts.append(time.perf_counter() - t0)
    same = all(np.array_equal(np.asarray(r["T"]).view(np.uint32), T.view(np.uint32)) and bool(r["converged"]) == c and r["iterations"] == it
               and np.float64(r["fitness"]).tobytes() == np.float64(f).tobytes() for r, (T, c, it, f) in zip(res_b, out))
    rounds, pair_rounds = lb.lastRounds()
    lb.close()
    reg.close()
    rec["loop"] = {"pairs": len(pairs), "group": 8, "sensor": "vlp16", "points_per_cloud": int(clouds[lf[0]].shape[0]), "resolution": 1.0,
                   "batch_s": float(np.median(tb)), "sequential_s": float(np.median(ts)), "batch_all_s": tb, "sequential_all_s": ts,
                   "batch_pairs_per_s": len(pairs) / float(np.median(tb)), "sequential_pairs_per_s": len(pairs) / float(np.median(ts)),
                   "speedup": float(np.median(ts)) / float(np.median(tb)), "batched_rounds": rounds, "pair_passes": pair_rounds,
                   "bitwise_equal": bool(same)}
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
