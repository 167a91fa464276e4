"""Loop-closure candidate batch across GPUs (SURVEY.md §8e; BASELINE.json configs[3]) — workload generator, CPU-testable
mirror of the sharding / gather layout, and the bench leg.  All compute and the collective are in libb200reg.so
(b2r_batch_* in include/b200reg.h; csrc/pair_engine.cuh, csrc/batch.cuh); nothing here computes.

The reference validates loop candidates one after another inside LoopDetector::matching
(/root/reference/include/hdl_graph_slam/loop_detector.hpp:117-171): one shared target (the new keyframe, :122) and C
independent align() + getFitnessScore() calls (:135-154) that only couple through the running `best_score`, i.e. a post-hoc
argmin.  So the batch shards naturally:

  * groups (= all candidates of one new keyframe) are dealt to ranks in CONTIGUOUS blocks (b2r_shard_range): neighbouring
    groups share candidate keyframes, so each keyframe's search structure / covariances are built once, on one GPU;
  * clouds reach a GPU only over PCIe (b2r_batch_add_cloud); nothing point-sized ever crosses NVLink;
  * on each GPU every LM iteration of every pair in flight is ONE pair of kernel launches, the LM step runs on the device;
  * ONE collective ends the batch: ncclAllGather (issued by the library) of fixed 80-byte records {T[16] f32, fitness f64,
    converged i32, iterations i32} padded to the largest per-rank share;
  * every rank then holds all records and runs the reference's argmin per group (b2r_loop_argmin; tie rule of :147).
"""
import ctypes as C
import json
import os
import sys
import math
import time
import numpy as np

RECORD_BYTES = 80
RECORD_DTYPE = np.dtype([("T", np.float32, (16,)), ("fitness", np.float64), ("converged", np.int32), ("iterations", np.int32)])
assert RECORD_DTYPE.itemsize == RECORD_BYTES


# ------------------------------------------------------------------------------------------------ layout mirror (CPU-testable)
def shard_range(n_groups, world, rank):
    """Python mirror of b2r_shard_range: contiguous block [g0, g1) of groups owned by `rank`"""
    return n_groups * rank // world, n_groups * (rank + 1) // world


def layout(group_first, world):
    """(padded per-rank record count M, per-rank pair ranges [(p0, p1)]) exactly as b2r_batch_loop_detect computes them"""
    n_groups = len(group_first) - 1
    ranges = []
    for r in range(world):
        g0, g1 = shard_range(n_groups, world, r)
        ranges.append((int(group_first[g0]), int(group_first[g1])))
    return max((p1 - p0 for p0, p1 in ranges), default=0), ranges


def unpack_gathered(gathered, group_first, world):
    """gathered: (world, M) record array as the all-gather leaves it -> flat record array in pair order"""
    M, ranges = layout(group_first, world)
    out = np.zeros(int(group_first[-1]), RECORD_DTYPE)
    for r, (p0, p1) in enumerate(ranges):
        out[p0:p1] = gathered[r][: p1 - p0]
    return out


def argmin_per_group(records, group_first, fitness_score_thresh):
    """LoopDetector::matching's selection (loop_detector.hpp:147-163) per group -> index inside the group or -1 (mirror of b2r_loop_argmin)"""
    best = []
    for g in range(len(group_first) - 1):
        best_score, best_c = np.finfo(np.float64).max, -1
        for c, rec in enumerate(records[int(group_first[g]): int(group_first[g + 1])]):
            score = float(rec["fitness"])
            if not rec["converged"] or score > best_score:
                continue
            best_score, best_c = score, c
        if best_score > fitness_score_thresh:
            best_c = -1
        best.append(best_c)
    return best


def gather_records_torch(local_records, M, world, device=None):
    """the same fixed-size all-gather through torch.distributed (gloo on CPU): stand-in for the library's ncclAllGather in CPU tests"""
    import torch
    import torch.distributed as dist
    buf = np.zeros(max(M, 1), RECORD_DTYPE)
    buf[: len(local_records)] = local_records
    t = torch.from_numpy(buf.view(np.uint8).reshape(-1).copy())
    if device is not None:
        t = t.to(device)
    out = torch.empty(world * t.numel(), dtype=torch.uint8, device=t.device)
    if world > 1:
        dist.all_gather_into_tensor(out, t)
    else:
        out.copy_(t)
    return out.cpu().numpy().reshape(world, -1).view(RECORD_DTYPE)


# ------------------------------------------------------------------------------------------------ workload (configs[3])
LAP = 251  # frames per lap of the synthetic circuit: frame f + LAP revisits the place of frame f
GROUP = 8


def loop_workload(n_groups, sensor="vlp16", seed=1234, period=None):
    """n_groups new keyframes, each with GROUP candidates one lap later, a few metres around the new keyframe's pose; initial
    guess = true relative pose o perturbation U(+-0.5 m, +-3 deg), z zeroed as loop_detector.hpp:141-142.
    period: the workload repeats after `period` groups (group g is the same keyframes and guesses as group g - period), so that
    contiguous shards of `period` groups are IDENTICAL work — weak scaling with exactly fixed per-GPU work.
    Returns (frames needed per group [(target frame, [source frames])], guesses (n_pairs, 4, 4) float32, group_first)."""
    from . import synth
    if period and n_groups > period:
        base_groups, base_guesses, _ = loop_workload(period, sensor, seed)
        groups = [base_groups[g % period] for g in range(n_groups)]
        guesses = np.concatenate([base_guesses[(g % period) * GROUP:(g % period + 1) * GROUP] for g in range(n_groups)])
        return groups, guesses, [GROUP * g for g in range(n_groups + 1)]
    rng = np.random.default_rng(seed)
    groups, guesses, group_first = [], [], [0]
    for g in range(n_groups):
        tf = 3 * g
        sfs = []
        for c in range(GROUP):
            sf = tf + LAP + c - GROUP // 2
            dt, da = rng.uniform(-0.5, 0.5, 3), np.deg2rad(rng.uniform(-3, 3))
            rel = np.linalg.inv(synth.pose_matrix(tf)) @ synth.pose_matrix(sf)
            P = np.eye(4)
            P[:3, 3] = dt
            P[0, 0], P[0, 1], P[1, 0], P[1, 1] = np.cos(da), -np.sin(da), np.sin(da), np.cos(da)
            guess = (rel @ P).astype(np.float32)
            guess[2, 3] = 0.0  # loop_detector.hpp:142
            guesses.append(guess)
            sfs.append(sf)
        groups.append((tf, sfs))
        group_first.append(group_first[-1] + GROUP)
    return groups, np.stack(guesses), group_first


# ------------------------------------------------------------------------------------------------ bench leg
def _clock_sampler(local_rank):
    import bench
    return bench.ClockSampler(local_rank)


def run_loop_batch(args, rank, world, local_rank, quiet=False):
    """K timed passes of the whole loop-closure batch (every pass registers the keyframe clouds afresh, aligns all pairs, gathers).
    Returns the JSON-able line (rank 0) or None."""
    import torch
    import torch.distributed as dist
    import hdl_graph_slam_b200 as pkg
    from . import synth
    from ._capi import Pair
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=dev)
    K, W = max(1, args.steps), max(0, args.warmup)
    per_gpu = args.pairs
    n_groups = max(1, per_gpu // GROUP) * world
    distinct = bool(getattr(args, "distinct_shards", False))
    groups, guesses, group_first = loop_workload(n_groups, "vlp16", period=None if distinct else n_groups // world)
    n_pairs = group_first[-1]
    g0, g1 = shard_range(n_groups, world, rank)
    # the keyframe clouds THIS rank needs (its own groups only), pinned on the host and resident copies in HBM
    needed = sorted({f for g in range(g0, g1) for f in [groups[g][0]] + groups[g][1]})
    first = synth.scan("vlp16", frame=needed[0], stride=8)
    n, stride_f = first.shape
    host = torch.empty((len(needed), n, stride_f), dtype=torch.float32, pin_memory=True)
    for i, f in enumerate(needed):
        host[i].copy_(torch.from_numpy(synth.scan("vlp16", frame=f, stride=8)))
    devbuf = host.to(dev)
    torch.cuda.synchronize()
    slot = {f: i for i, f in enumerate(needed)}
    fbytes = n * stride_f * 4

    lb = pkg.RegistrationBatch(params={"registration_method": "FAST_GICP"}, device_id=local_rank)
    if world > 1:
        idt = torch.zeros(128, dtype=torch.uint8, device=dev)
        if rank == 0:
            idt = torch.frombuffer(bytearray(pkg.RegistrationBatch.ncclUniqueId()), dtype=torch.uint8).to(dev)
        dist.broadcast(idt, 0)
        lb.commInit(bytes(idt.cpu().numpy().tobytes()), rank, world)
    stream = torch.cuda.ExternalStream(lb.engine.getStream(), device=dev)
    pairs = (Pair * n_pairs)()
    for p in range(n_pairs):
        gc = np.ascontiguousarray(guesses[p].T.reshape(-1))
        for k in range(16):
            pairs[p].guess[k] = gc[k]
        pairs[p].source = pairs[p].target = -1
    max_range, thresh = args.fitness_max_range, 0.5

    dbg = bool(os.environ.get("B2R_DEBUG_TIMING"))

    def one_pass(device_arm):
        t0 = time.perf_counter()
        base = devbuf.data_ptr() if device_arm else host.data_ptr()
        ids = {f: lb.addCloudRaw(base + slot[f] * fbytes, n, stride_f * 4, device=device_arm) for f in needed}
        for g in range(g0, g1):
            tf, sfs = groups[g]
            for c, sf in enumerate(sfs):
                pairs[group_first[g] + c].source, pairs[group_first[g] + c].target = ids[sf], ids[tf]
        t1 = time.perf_counter()
        best, res = lb.loopDetect(pairs, group_first, max_range, thresh, raw=True)
        t2 = time.perf_counter()
        rounds = lb.lastRounds()
        for cid in ids.values():
            lb.removeCloud(cid)
        if dbg:
            print(f"[rank {rank}] pass: add clouds {1e3 * (t1 - t0):.3f} ms, loopDetect {1e3 * (t2 - t1):.3f} ms, remove {1e3 * (time.perf_counter() - t2):.3f} ms",
                  file=sys.stderr, flush=True)
        return best, res, rounds

    results = {}
    arms = ("value", "e2e") if getattr(args, "no_profile", False) else ("value", "e2e", "profile")
    for arm in arms:
        device_arm = arm != "e2e"
        for _ in range(W):
            one_pass(device_arm)
        lb.synchronize()
        lb.engine.getStats(reset=True)
        lb.engine.setProfiling(arm == "profile")
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        sampler = _clock_sampler(local_rank) if (rank == 0 and arm == "value") else None
        if sampler:
            sampler.start()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        t0 = time.perf_counter()
        rounds_total, pair_rounds_total = 0, 0
        for _ in range(K):
            best, res, (rounds, pair_rounds) = one_pass(device_arm)
            rounds_total += rounds
            pair_rounds_total += pair_rounds
        e1.record(stream)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        ms = e0.elapsed_time(e1)
        t = torch.tensor([ms], dtype=torch.float64, device=dev)
        per_rank = [ms]
        if world > 1:
            dist.barrier()
            allms = torch.zeros(world, dtype=torch.float64, device=dev)
            dist.all_gather_into_tensor(allms, t)
            per_rank = [float(x) for x in allms.cpu()]
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        stats = lb.engine.getStats()
        lb.engine.setProfiling(False)
        clocks = None
        if arm == "value":
            # nvidia-smi needs a few hundred ms under load for its samples: EVERY rank runs the same number of extra untimed passes (a pass
            # holds a collective), derived from the all-reduced time so that all ranks agree on it
            total_ms = float(t.item())
            extra = 0 if total_ms >= 700.0 else min(200, int(math.ceil((700.0 - total_ms) / max(total_ms / K, 1e-3))))
            for _ in range(extra):
                one_pass(device_arm)
            lb.synchronize()
            if sampler:
                sampler.extra_steps += extra
                clocks = sampler.stop()
        results[arm] = dict(ms=float(t.item()), per_rank_ms=per_rank, wall_ms=wall * 1e3, stats=stats, best=best, res=res, clocks=clocks,
                            rounds=rounds_total, pair_rounds=pair_rounds_total)
    lb.close()
    if rank != 0:
        return None
    import bench
    rv, re_ = results["value"], results["e2e"]
    value = n_pairs * K / (rv["ms"] * 1e-3)
    e2e = n_pairs * K / (re_["ms"] * 1e-3)
    res = rv["res"]
    conv = sum(int(res[i].converged) for i in range(n_pairs))
    iters = sum(int(res[i].iterations) for i in range(n_pairs))
    st = results["profile"]["stats"] if "profile" in results else rv["stats"]
    prof = results.get("profile", rv)
    hbm, how = bench.peaks()
    # roofline of the batched LM round (k_pair_search + k_pair_accumulate): SURVEY §8d's fused-iteration formula,
    # 64 (N + M) + 8 N bytes per pair-iteration, times the pair-rounds of this rank, over the CUDA-event time of those launches
    N = M = int(n)
    bytes_per_pair_round = 64 * (N + M) + 8 * N
    round_ms = st["ms"].get("gicp_correspondences", 0.0) + st["ms"].get("gicp_linearize", 0.0)
    roofline = None
    if round_ms > 0 and prof["pair_rounds"] > 0:
        achieved = bytes_per_pair_round * prof["pair_rounds"] / (round_ms * 1e-3) / 1e9
        launches = st["calls"].get("gicp_correspondences", 0) + st["calls"].get("gicp_linearize", 0)
        roofline = {"bound": "hbm", "kernel": "k_pair_search + k_pair_accumulate (one batched LM round = update_correspondences + linearize + compute_error of every pair in flight)",
                    "achieved": achieved, "peak": hbm, "unit": "GB/s", "frac": achieved / hbm,
                    "peak_source": f"of {how} (MEASURED_PEAKS.json hbm_gbs)" if how == "measured" else "of fallback (3.35 TB/s, H100 SXM data sheet)",
                    "algorithmic_bytes_per_pair_round": bytes_per_pair_round, "pair_rounds": prof["pair_rounds"], "rounds": prof["rounds"],
                    "avg_round_us": round_ms * 1e3 / max(prof["rounds"], 1), "launches_timed": launches,
                    "us_per_pair_round": round_ms * 1e3 / prof["pair_rounds"],
                    "share_of_step": round_ms / prof["ms"],
                    "working_set": f"{per_gpu} pairs in flight x {117 * N / 1e6:.1f} MB of per-pair workspace + {len(needed)} clouds x {(16 + 48 + 8) * N / 1e6:.1f} MB >> 50 MB L2"}
    kernel_ms = {k: round(v, 3) for k, v in st["ms"].items() if v > 0}
    if getattr(args, "dump_outputs", None):  # every pair's gathered record of the last timed pass + the per-group best candidate
        bench.dump_outputs(args.dump_outputs, {
            "T": np.array([np.array(res[i].T, np.float32).reshape(4, 4).T for i in range(n_pairs)], np.float32),
            "fitness": [res[i].fitness for i in range(n_pairs)], "converged": [res[i].converged for i in range(n_pairs)],
            "iterations": [res[i].iterations for i in range(n_pairs)], "best": rv["best"]})
    line = {
        "metric": "registrations/sec", "value": value, "unit": "registrations/s", "n_gpus": world, "steps": K, "warmup": W,
        "ms_per_step": rv["ms"] / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32 NN / f64 accumulate", "data": "synthetic",
        "config": {"workload": "BASELINE configs[3]: loop-closure candidate batch (GICP, 64k-pt VLP-16 pairs, 8 candidates per new keyframe), sharded by keyframe group",
                   "pairs_total": n_pairs, "pairs_per_gpu": per_gpu, "points_per_scan": N, "groups": n_groups,
                   "unique_clouds_per_gpu": len(needed),
                   "shards": ("distinct keyframe groups per rank (per-GPU work varies with the shard's iteration counts)" if distinct else
                              "every rank's shard is the same keyframe groups and guesses: per-GPU work exactly fixed (weak scaling); --distinct-shards gives every rank "
                              "different places of the circuit, where the MAX over ranks follows the heaviest shard"), "cloud_cache": "each keyframe cloud is uploaded and preprocessed once per pass and shared by the pairs that name it",
                   "step": "one pass = register the rank's keyframe clouds (upload + search structure + covariances), align + fitness of all its pairs, one ncclAllGather, argmin",
                   "collective": "one ncclAllGather of 80-byte records, issued by libb200reg (in-library NCCL)", "fitness_max_range": max_range,
                   "l2": "inputs larger than L2: a pass streams the rank's keyframe clouds (2 MiB each) and ~7.7 MB of workspace per pair",
                   "mean_iterations": iters / n_pairs, "converged_frac": conv / n_pairs, "loops_found": int(sum(1 for b in rv["best"] if b >= 0)),
                   "lanes_per_query": int(os.environ.get("B2R_BATCH_COPIES", "1"))},
        "e2e": {"value": e2e, "unit": "registrations/s", "h2d_bytes_per_step": re_["stats"]["h2d_bytes"] / K, "d2h_bytes_per_step": re_["stats"]["d2h_bytes"] / K,
                "ms_per_step": re_["ms"] / K},
        "gpu_launches": int(sum(rv["stats"]["launches"].values())),
        "clocks": rv["clocks"],
        "roofline": roofline,
        "kernel_ms_in_timed_region": kernel_ms,
        "kernel_timing": {"pass": "same K passes repeated with per-launch CUDA events on the engine's streams", "ms_per_step": prof["ms"] / K},
        "wall_ms_per_step": rv["wall_ms"] / K,
        "per_rank_ms_per_step": [round(x / K, 3) for x in rv["per_rank_ms"]],
    }
    if world == 1 and getattr(args, "cpu_sample", 0) > 0 and not quiet:
        line["cpu_baseline"] = bench.cpu_baseline_loop(groups, guesses, group_first, max_range)
    return line


def bench_loop_batch(args, rank, world, local_rank):
    import torch
    import torch.distributed as dist
    anchor = None
    if world > 1:
        # the 1-GPU figure of the SAME workload, taken by rank 0 alone on the same box right before the N-GPU passes (the default
        # N = 1 bench line is the odometry chain, BASELINE configs[1]; this makes every N > 1 line carry its own scaling anchor)
        torch.cuda.set_device(local_rank)
        dev = torch.device("cuda", local_rank)
        if not dist.is_initialized():
            dist.init_process_group("nccl", device_id=dev)
        if rank == 0 and not getattr(args, "no_anchor", False):
            import types
            a = types.SimpleNamespace(steps=3, warmup=3, pairs=args.pairs, fitness_max_range=args.fitness_max_range, no_profile=True)
            try:
                one = run_loop_batch(a, 0, 1, local_rank, quiet=True)
                anchor = {"value": one["value"], "unit": one["unit"], "ms_per_step": one["ms_per_step"], "steps": 3, "warmup": 3,
                          "e2e": one["e2e"]["value"], "pairs": one["config"]["pairs_total"],
                          "note": "same workload on ONE GPU of this box (rank 0 alone, before the N-GPU passes): efficiency = value / (n_gpus x this)"}
            except Exception as e:  # noqa: BLE001
                anchor = {"error": repr(e)}
        dist.barrier()
    line = run_loop_batch(args, rank, world, local_rank)
    if rank == 0:
        if anchor is not None:
            line["anchor_n1"] = anchor
        print(json.dumps(line), flush=True)
    if world > 1 and dist.is_initialized():
        dist.destroy_process_group()
