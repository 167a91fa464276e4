"""Time one hdl_graph_slam back-end session with the shared-keyframe-cache drop-in (adapter/b200_backend.hpp) against today's path,
the reference LoopDetector walk over the pcl::Registration adapter (development aid, not part of bench.py):

    python tools/backend_time.py [--methods FAST_GICP NDT_OMP] [--keyframes 252] [--per-tick 4] [--res 0.05] [--rounds 3] [--out record.json]

Session: keyframes every 2 m along two laps of the synthetic circuit (16 384-point vlp16_16k scans, 32-byte pcl::PointXYZI records,
graph estimates = trajectory poses with a seeded drift), `per-tick` new keyframes per optimisation tick.  Each tick, as
hdl_graph_slam_nodelet does it: detect(keyframes, new_keyframes) with the rosparam defaults and fitness_score_max_range 2.5, one
information matrix per odometry edge of the new keyframes and one per registered loop, then one map at `res` over every keyframe.
Arms (the same ABI calls each class makes, issued from Python with their arguments built in the timed region):
  dropin  B200LoopDetector: b2r_loop_detect_plan -> b2r_batch_loop_detect -> b2r_loop_detect_replay on one b2r_batch;
          B200InformationMatrixCalculator: b2r_batch_calc_fitness_score of one pair + b2r_information_from_fitness;
          B200MapCloudGenerator: b2r_batch_map_cloud_generate.  Each keyframe cloud is added to the batch at its first use.
  today   LoopDetector::matching on one registration handle, one candidate at a time: setInputTarget, then per candidate
          setInputSource (upload + search structure + covariances), align, getFitnessScore (b2r_fitness).  The information matrices
          and the map have no device path today (a CPU kd-tree per edge, a CPU octree per map); this arm times the engine's
          uncached single-handle calls in their place (b2r_set_target / b2r_set_source / b2r_fitness per edge, b2r_map_cloud_generate
          uploading every keyframe per map), so it is a lower bound on today's back-end time, not the reference's CPU time.
Every call returns after its results are on the host, so a host clock around a stage is the caller's time.  The arms alternate in
`rounds` full sessions after one warm-up session each; the record keeps each stage's per-session totals and the median per tick, the
registered loops of both arms (equal, relative poses bitwise), whether the information matrices and maps are bitwise equal, and the
card's name, power limit and clocks, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import hdl_graph_slam_b200 as pkg  # noqa: E402
from hdl_graph_slam_b200 import synth  # noqa: E402

DBL_MAX = np.finfo(np.float64).max
MAX_RANGE, THRESH = 2.5, 0.5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem,driver_version", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable: " + torch.cuda.get_device_name(0)


def workload(n_keyframes, spacing=2):
    frames = [spacing * k for k in range(n_keyframes)]
    rng = np.random.default_rng(77)
    clouds = [synth.scan("vlp16_16k", frame=f, stride=8) for f in frames]
    est = []
    for f in frames:
        T = synth.pose_matrix(f)
        a = np.deg2rad(rng.uniform(-1.0, 1.0))
        D = np.eye(4)
        D[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
        D[:3, 3] = rng.uniform(-0.2, 0.2, 3)
        est.append(T @ D)
    return [float(f) for f in frames], clouds, est


class DropIn:
    def __init__(self, params, clouds):
        self.lb = pkg.RegistrationBatch(params=params)
        self.gate = pkg.LoopClosureGate(fitness_score_max_range=MAX_RANGE, fitness_score_thresh=THRESH)
        self.clouds, self.ids = clouds, {}

    def cid(self, k):
        if k not in self.ids:
            self.ids[k] = self.lb.addCloud(self.clouds[k])
        return self.ids[k]

    def detect(self, kfs, new):
        """kfs / new: lists of (keyframe index, accum, estimate) -> [(new index, candidate index, T)]"""
        planned = self.gate.last_edge_accum_distance
        cand, guesses, gf = self.gate.plan([k[1:] for k in kfs], [k[1:] for k in new])
        best = [-1] * len(new)
        results = []
        if gf[-1]:
            pairs = [(self.cid(kfs[cand[j]][0]), self.cid(new[g][0]), guesses[j]) for g in range(len(new)) for j in range(gf[g], gf[g + 1])]
            best, results = self.lb.loopDetect(pairs, gf, MAX_RANGE, THRESH)
        accepted = self.gate.replay([k[1:] for k in new], gf, best, planned)
        return [(new[g][0], kfs[cand[gf[g] + a]][0], results[gf[g] + a]["T"]) for g, a in enumerate(accepted) if a >= 0]

    def information(self, k1, k2, rel):
        return pkg.information_from_fitness(self.lb.calcFitnessScore([(self.cid(k1), self.cid(k2), rel.astype(np.float32))], DBL_MAX)[0])

    def map(self, ks, poses, res):
        return self.lb.mapCloudGenerate([self.cid(k) for k in ks], poses, res)

    def close(self):
        self.lb.close()


class Today:
    def __init__(self, params, clouds):
        self.reg = pkg.select_registration_method(params)
        self.inf = pkg.select_registration_method(params)
        self.gate = pkg.LoopClosureGate(fitness_score_max_range=MAX_RANGE, fitness_score_thresh=THRESH)
        self.clouds = clouds

    def detect(self, kfs, new):
        loops = []
        for nk in new:
            cands = self.gate.find_candidates([k[1:] for k in kfs], nk[1:])  # reads last_edge_accum_distance
            if not cands:
                continue
            self.reg.setInputTarget(self.clouds[nk[0]])
            best_score, best = DBL_MAX, None
            for c in cands:
                self.reg.setInputSource(self.clouds[kfs[c][0]])
                self.reg.align(self.gate.guess(nk[2], kfs[c][2]))
                score = self.reg.getFitnessScore(MAX_RANGE)
                if not self.reg.hasConverged() or score > best_score:
                    continue
                best_score, best = score, (kfs[c][0], self.reg.getFinalTransformation())
            if best is not None and best_score <= THRESH:
                loops.append((nk[0], best[0], best[1]))
                self.gate.last_edge_accum_distance = nk[1]
        return loops

    def information(self, k1, k2, rel):
        self.inf.setInputTarget(self.clouds[k1])
        self.inf.setInputSource(self.clouds[k2])
        return pkg.information_from_fitness(self.inf.getFitnessScore(DBL_MAX, T=rel.astype(np.float32)))

    def map(self, ks, poses, res):
        return self.reg.mapCloudGenerate([(self.clouds[k], p) for k, p in zip(ks, poses)], res)

    def close(self):
        self.reg.close()
        self.inf.close()


def session(arm, params, accum, clouds, est, per_tick, res):
    """one back-end session -> (per-tick stage seconds, loops, information matrices, last map)"""
    a = (DropIn if arm == "dropin" else Today)(params, clouds)
    t = {"detect": [], "information": [], "map": []}
    loops_all, infos, m = [], [], None
    n = len(clouds)
    for first in range(0, n, per_tick):
        kfs = [(k, accum[k], est[k]) for k in range(first)]
        new = [(k, accum[k], est[k]) for k in range(first, min(first + per_tick, n))]
        t0 = time.perf_counter()
        loops = a.detect(kfs, new)
        t1 = time.perf_counter()
        edges = [(k, k - 1, np.linalg.inv(est[k - 1]) @ est[k]) for k, _, _ in new if k > 0]
        edges += [(k1, k2, T.astype(np.float64)) for k1, k2, T in loops]
        infos += [a.information(k1, k2, rel) for k1, k2, rel in edges]
        t2 = time.perf_counter()
        last = new[-1][0] + 1
        m = a.map(list(range(last)), [est[k] for k in range(last)], res)
        t3 = time.perf_counter()
        t["detect"].append(t1 - t0)
        t["information"].append(t2 - t1)
        t["map"].append(t3 - t2)
        loops_all += loops
    a.close()
    return t, loops_all, infos, m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--methods", nargs="+", default=["FAST_GICP", "NDT_OMP"])
    ap.add_argument("--keyframes", type=int, default=252)
    ap.add_argument("--per-tick", type=int, default=4)
    ap.add_argument("--res", type=float, default=0.05)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to time")
    accum, clouds, est = workload(a.keyframes)
    results = []
    for method in a.methods:
        params = {"registration_method": method, "reg_resolution": 1.0}
        for arm in ("dropin", "today"):  # warm-up: module loads, first allocations
            session(arm, params, accum[:2 * a.per_tick], clouds[:2 * a.per_tick], est[:2 * a.per_tick], a.per_tick, a.res)
        runs = {"dropin": [], "today": []}
        out = {}
        for _ in range(a.rounds):
            for arm in ("dropin", "today"):
                t, loops, infos, m = session(arm, params, accum, clouds, est, a.per_tick, a.res)
                runs[arm].append(t)
                out[arm] = (loops, infos, m)
        (la, ia, ma), (lb_, ib, mb) = out["dropin"], out["today"]
        loops_equal = [(x[0], x[1]) for x in la] == [(x[0], x[1]) for x in lb_] and all(np.array_equal(x[2], y[2]) for x, y in zip(la, lb_))
        stages = {}
        for arm, rs in runs.items():
            stages[arm] = {}
            for st in ("detect", "information", "map"):
                tot = [1e3 * sum(r[st]) for r in rs]
                stages[arm][st] = dict(session_ms=[round(x, 3) for x in tot], median_session_ms=float(np.median(tot)),
                                       median_tick_ms=float(np.median([1e3 * x for r in rs for x in r[st]])))
            tot = [1e3 * sum(sum(r[st]) for st in r) for r in rs]
            stages[arm]["total"] = dict(session_ms=[round(x, 3) for x in tot], median_session_ms=float(np.median(tot)))
        results.append(dict(method=method, keyframes=a.keyframes, ticks=len(runs["dropin"][0]["detect"]), loops=len(la),
                            information_matrices=len(ia), loops_equal=bool(loops_equal),
                            information_bitwise_equal=bool(len(ia) == len(ib) and all(np.array_equal(x, y) for x, y in zip(ia, ib))),
                            last_map_points=int(ma.shape[0]), map_bitwise_equal=bool(np.array_equal(ma, mb)), ms=stages))
        print(json.dumps(results[-1]), flush=True)
    rec = dict(card=card(), workload=f"{a.keyframes} keyframes every 2 m over the synthetic circuit, 16 384-point vlp16_16k scans, "
               f"{a.per_tick} new keyframes per tick; per tick detect, the information matrices of its odometry edges and loops, one map at {a.res}",
               rounds=a.rounds, params="reg_resolution 1.0, distance_thresh 5, accum_distance_thresh 8, min_edge_interval 5, "
               "fitness_score_max_range 2.5, fitness_score_thresh 0.5",
               arms={"dropin": "b200_backend.hpp's ABI calls on one shared b2r_batch, each keyframe uploaded once",
                     "today": "LoopDetector walk over one registration handle, one candidate at a time; information matrices and maps "
                              "as uncached single-handle engine calls (a lower bound: the reference computes them on the CPU)"},
               results=results)
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
