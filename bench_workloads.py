"""bench_workloads.py — part of bench.py: the workloads around the registration path (bench.py --workload voxelgrid | kitti_pipeline).

  voxelgrid       SURVEY §8 row a5 alone: pcl::VoxelGrid::filter of raw 120 000-point scans (apps/prefiltering_nodelet.cpp:138-149),
                  HBM -> HBM through b2r_voxelgrid_device (value) and host -> host through b2r_voxelgrid (e2e)
  kitti_pipeline  BASELINE configs[4], the per-scan part: raw KITTI-shape scan -> PrefilteringNodelet::cloud_callback (distance filter,
                  voxel grid 0.25 m, radius outlier removal: launch/hdl_graph_slam_kitti.launch:22-34) -> ScanMatchingOdometryNodelet::matching
                  (FAST_GICP, :41-59), the filtered cloud never leaving HBM (b2r_prefilter -> b2r_odometry_matching_device).  The loop-closure
                  half of configs[4] is the loop_batch workload.
One step = one scan.  N > 1: independent replicas (a chain does not shard), MAX over ranks of the device time.
"""
import json
import os
import time

import numpy as np

KITTI_PREFILTER = dict(use_distance_filter=1, distance_near_thresh=0.1, distance_far_thresh=100.0, downsample_method=1, downsample_resolution=0.25,
                       outlier_removal_method=2, radius_radius=0.5, radius_min_neighbors=2)
KITTI_ODOMETRY = {"registration_method": "FAST_GICP", "reg_transformation_epsilon": 0.1, "reg_maximum_iterations": 64,
                  "reg_max_correspondence_distance": 2.0, "reg_correspondence_randomness": 20}
KITTI_KEYFRAME = dict(keyframe_delta_trans=5.0, keyframe_delta_angle=2.0, keyframe_delta_time=10000.0)
N_FRAMES = 40  # 40 x 3.84 MB of raw scans = 154 MB > the 50 MB L2: consecutive steps never find their input in cache


def _setup(args, rank, world, local_rank):
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=dev)
    return torch, dist, dev


def _frames(torch, dev, rank, count=N_FRAMES):
    from hdl_graph_slam_b200 import synth
    first = synth.scan("kitti", frame=rank * 1000, stride=8)
    n, stride_f = first.shape
    host = torch.empty((count, n, stride_f), dtype=torch.float32, pin_memory=True)
    for i in range(count):
        host[i].copy_(torch.from_numpy(synth.scan("kitti", frame=rank * 1000 + i, stride=8)))
    devbuf = host.to(dev)
    torch.cuda.synchronize()
    return host, devbuf, int(n), int(stride_f)


def _timed(torch, dist, dev, world, stream, K, body, sampler=None, stats_fn=None, after=None):
    """K timed calls of body; `after` (if given) runs once the timed region has drained, before any untimed hold step"""
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    if sampler:
        sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    t0 = time.perf_counter()
    for k in range(K):
        body(k)
    e1.record(stream)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    clocks = None
    stats = stats_fn() if stats_fn else None  # counters of the timed region only (the hold steps below are not part of it)
    if after:
        after()
    if sampler:  # untimed steps of the same workload until nvidia-smi has sampled the load (bench.ClockSampler)
        sampler.hold(lambda k: body(k % K), torch.cuda.synchronize)
        clocks = sampler.stop()
    ms = e0.elapsed_time(e1)
    t = torch.tensor([ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.barrier()
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item()), wall * 1e3, clocks, stats


def _device_floats(torch, dev, ptr, rows, cols):
    """copy of a float32 (rows, cols) array the engine left in device memory"""
    class _View:
        __cuda_array_interface__ = {"shape": (rows, cols), "typestr": "<f4", "data": (ptr, False), "version": 2, "strides": None}
    return torch.as_tensor(_View(), device=dev).cpu().numpy().copy()


def _cpu_voxelgrid(host, leaf, budget_s=10.0):
    from oracle import oracle as orc  # bench.py's cpu_baseline leg: the checker timed beside the product, never on its path
    t0, done = time.perf_counter(), 0
    while done < host.shape[0] and time.perf_counter() - t0 < budget_s:
        orc.voxelgrid(host[done].numpy(), leaf)
        done += 1
    dt = time.perf_counter() - t0
    return done / dt, done


def bench_voxelgrid(args, rank, world, local_rank, leaf=0.25):
    import bench
    import hdl_graph_slam_b200 as pkg
    torch, dist, dev = _setup(args, rank, world, local_rank)
    host, devbuf, n, stride_f = _frames(torch, dev, rank)
    K, W = max(1, args.steps), max(3, args.warmup)
    reg = pkg.select_registration_method({"registration_method": "FAST_GICP"}, device_id=local_rank)
    stream = torch.cuda.ExternalStream(reg.getStream(), device=dev)
    fbytes = n * stride_f * 4
    counts = []
    last = {}

    def dev_step(k):
        last["ptr"], m, _ = reg.voxelGridFilterDevice(devbuf.data_ptr() + (k % N_FRAMES) * fbytes, n, stride_f * 4, leaf)
        counts.append(m)

    def keep_last_cloud():  # the downsampled cloud of the last timed step, before the hold steps reuse the output buffer
        if args.dump_outputs and rank == 0:
            reg.synchronize()
            last["cloud"] = _device_floats(torch, dev, last["ptr"], counts[-1], stride_f)

    def host_step(k):
        out = reg.voxelGridFilter(host[k % N_FRAMES].numpy(), leaf)
        counts.append(out.shape[0])

    res = {}
    for arm, body in (("value", dev_step), ("e2e", host_step), ("profile", dev_step)):
        for k in range(W):
            body(k)
        reg.synchronize()
        reg.getStats(reset=True)
        reg.setProfiling(arm == "profile")
        counts.clear()
        sampler = bench.ClockSampler(local_rank) if (rank == 0 and arm == "value") else None
        ms, wall, clocks, stats = _timed(torch, dist, dev, world, stream, K, body, sampler, reg.getStats, keep_last_cloud if arm == "value" else None)
        res[arm] = dict(ms=ms, wall=wall, clocks=clocks, stats=stats, n_ds=float(np.mean(counts)))
        reg.setProfiling(False)
    reg.close()
    if rank != 0:
        return
    if args.dump_outputs:
        bench.dump_outputs(args.dump_outputs, {"cloud": last["cloud"]})
    hbm, how = bench.peaks()
    n_ds = res["value"]["n_ds"]
    ab = 2 * 16 * n + 16 * n_ds  # SURVEY §8d: N_raw x 16 x 2 (read for the key + read for the sum) + N_ds x 16
    st = res["profile"]["stats"]
    cls = max(st["ms"], key=lambda c: st["ms"][c])
    per_launch_ms = st["ms"][cls] / max(st["calls"][cls], 1)
    cpu_v, cpu_n = _cpu_voxelgrid(host, leaf)
    line = {
        "metric": "voxel-grid downsamples/sec", "value": world * K / (res["value"]["ms"] * 1e-3), "unit": "scans/s", "n_gpus": world, "steps": K, "warmup": W,
        "ms_per_step": res["value"]["ms"] / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "int32 keys / f32 centroids",
        "data": "synthetic",
        "config": {"workload": "SURVEY §8 row a5: pcl::VoxelGrid of raw KITTI-shape scans (companion kernel of the registration path)", "points_per_scan": n,
                   "leaf": leaf, "mean_output_points": n_ds, "record_bytes": stride_f * 4,
                   "l2": f"inputs larger than L2: {N_FRAMES} distinct scans x {fbytes / 1e6:.2f} MB cycled"},
        "e2e": {"value": world * K / (res["e2e"]["ms"] * 1e-3), "unit": "scans/s", "h2d_bytes_per_step": res["e2e"]["stats"]["h2d_bytes"] / K,
                "d2h_bytes_per_step": res["e2e"]["stats"]["d2h_bytes"] / K, "ms_per_step": res["e2e"]["ms"] / K},
        "gpu_launches": int(sum(res["value"]["stats"]["launches"].values())),
        "clocks": res["value"]["clocks"],
        "roofline": {"bound": "hbm", "kernel": "k_voxelgrid_cluster (keys + cluster radix sort + centroids + compaction in one launch)", "achieved": ab / (per_launch_ms * 1e-3) / 1e9,
                     "peak": hbm, "unit": "GB/s", "frac": ab / (per_launch_ms * 1e-3) / 1e9 / hbm,
                     "peak_source": f"of {how} (MEASURED_PEAKS.json hbm_gbs)" if how == "measured" else "of fallback (3.35 TB/s, H100 SXM data sheet)",
                     "algorithmic_bytes_per_launch": ab, "avg_launch_us": per_launch_ms * 1e3, "launches_timed": st["calls"][cls],
                     "note": "one cluster per scan (16 CTAs where the device accepts that size, else 8): latency bound on a few of 132 SMs; concurrent scans on other streams fill the rest"},
        "cpu_baseline": {"value": cpu_v, "unit": "scans/s", "cores": 1, "kind": "port", "sample": f"{cpu_n} scans of the same workload through the oracle's pcl::VoxelGrid restatement"},
    }
    print(json.dumps(line), flush=True)
    if world > 1 and dist.is_initialized():
        dist.destroy_process_group()


def _cpu_pipeline(host, budget_frames):
    """the oracle through the same per-scan chain: distance filter -> voxel grid -> radius outlier removal -> GICP odometry with the
    KITTI launch file's parameters (kept target kd-tree + covariances while the keyframe stays, as fast_gicp does)"""
    import bench
    from oracle import oracle as orc
    frames = []
    t_pref = time.perf_counter()
    for i in range(budget_frames):
        c = host[i].numpy()
        c = c[orc.distance_filter(c, 0.1, 100.0)]
        v = orc.voxelgrid(c, 0.25)[0]
        full = np.zeros((v.shape[0], 8), np.float32)
        full[:, :3], full[:, 3], full[:, 4] = v[:, :3], 1.0, v[:, 3]
        full = full[orc.radius_outlier(full, 0.5, 2)]
        frames.append(np.ascontiguousarray(full))
    t_pref = time.perf_counter() - t_pref
    threads = bench.best_thread_count(orc, frames[:7], "FAST_GICP", {})[0]
    kf, prev = None, np.eye(4, dtype=np.float32)
    t0 = time.perf_counter()
    for cloud in frames:
        if kf is None:
            kf = orc.GicpTarget(cloud, 20, threads)
            continue
        cov = orc.gicp_covariances(cloud, 20, threads)
        r = kf.align(cloud, prev, threads=threads, src_cov=cov, transformation_epsilon=0.1, max_corr_dist=2.0)
        prev = r["T"]
        if np.linalg.norm(prev[:3, 3]) > 5.0:
            kf, prev = orc.GicpTarget(cloud, 20, threads), np.eye(4, dtype=np.float32)
    t_odo = time.perf_counter() - t0
    return budget_frames / (t_pref + t_odo), threads, t_pref / budget_frames, t_odo / budget_frames


def bench_kitti_pipeline(args, rank, world, local_rank):
    import bench
    import hdl_graph_slam_b200 as pkg
    torch, dist, dev = _setup(args, rank, world, local_rank)
    host, devbuf, n, stride_f = _frames(torch, dev, rank)
    K, W = max(1, args.steps), max(3, args.warmup)
    fbytes = n * stride_f * 4
    res = {}
    for arm in ("value", "e2e", "profile"):
        reg = pkg.select_registration_method(dict(KITTI_ODOMETRY), device_id=local_rank)
        odo = pkg.ScanMatchingOdometry(reg, **KITTI_KEYFRAME)
        stream = torch.cuda.ExternalStream(reg.getStream(), device=dev)
        state = dict(m=[], iters=[], conv=0, kf=0, last=None)

        def step(k, arm=arm, reg=reg, odo=odo, state=state):
            f = k % N_FRAMES
            if arm == "e2e":
                _, dptr, m = reg.prefilter_raw(host.data_ptr() + f * fbytes, n, stride_f * 4, device=False, **KITTI_PREFILTER)
            else:
                _, dptr, m = reg.prefilter_raw(devbuf.data_ptr() + f * fbytes, n, stride_f * 4, device=True, **KITTI_PREFILTER)
            st = odo.matching_raw(0.1 * k, dptr, m, stride_f * 4, device=True)
            state["m"].append(m)
            state["iters"].append(st["iterations"])
            state["conv"] += int(st["converged"])
            state["kf"] += int(st["keyframe_updated"])
            state["last"] = dict(bench.odometry_outputs(st), filtered_points=m)

        for k in range(W):
            step(k)
        reg.synchronize()
        reg.getStats(reset=True)
        reg.setProfiling(arm == "profile")
        for key in ("m", "iters"):
            state[key].clear()
        state["conv"] = state["kf"] = 0
        sampler = bench.ClockSampler(local_rank) if (rank == 0 and arm == "value") else None
        kept = {}
        ms, wall, clocks, stats = _timed(torch, dist, dev, world, stream, K, lambda k: step(k + W), sampler, reg.getStats,
                                         lambda: kept.update(state["last"]))
        res[arm] = dict(ms=ms, wall=wall, clocks=clocks, stats=stats, m=float(np.mean(state["m"])), iters=float(np.mean(state["iters"])),
                        conv=state["conv"], kf=state["kf"], last=kept)
        reg.setProfiling(False)
        odo.close()
        reg.close()
    if rank != 0:
        return
    rv = res["value"]
    if args.dump_outputs:
        bench.dump_outputs(args.dump_outputs, rv["last"])
    hbm, how = bench.peaks()
    st = res["profile"]["stats"]
    m = int(rv["m"])
    cls = max(st["ms"], key=lambda c: st["ms"][c])
    per_launch_ms = st["ms"][cls] / max(st["calls"][cls], 1)
    ab = bench.algorithmic_bytes(cls, m, m, stride_f * 4)
    roofline = None
    if ab:
        roofline = {"bound": "hbm", "kernel": cls, "achieved": ab / (per_launch_ms * 1e-3) / 1e9, "peak": hbm, "unit": "GB/s",
                    "frac": ab / (per_launch_ms * 1e-3) / 1e9 / hbm,
                    "peak_source": f"of {how} (MEASURED_PEAKS.json hbm_gbs)" if how == "measured" else "of fallback (3.35 TB/s, H100 SXM data sheet)",
                    "algorithmic_bytes_per_launch": ab, "avg_launch_us": per_launch_ms * 1e3, "launches_timed": st["calls"][cls],
                    "share_of_step": st["ms"][cls] / res["profile"]["ms"],
                    "note": f"filtered scans are ~{m} points: a pair's working set sits in L2, latency-bound single chain"}
    n_cpu = max(4, min(args.cpu_sample if args.cpu_sample > 0 else 0, N_FRAMES))
    cpu = None
    if args.cpu_sample > 0:
        v, threads, t_pref, t_odo = _cpu_pipeline(host, n_cpu)
        cpu = {"value": v, "unit": "scans/s", "cores": threads, "kind": "port",
               "sample": f"{n_cpu} scans of the same workload through the oracle (prefilters single-threaded {t_pref * 1e3:.0f} ms/scan, GICP odometry on {threads} threads {t_odo * 1e3:.0f} ms/scan)"}
    line = {
        "metric": "registrations/sec", "value": world * K / (rv["ms"] * 1e-3), "unit": "scans/s", "n_gpus": world, "steps": K, "warmup": W,
        "ms_per_step": rv["ms"] / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32 NN / f64 accumulate", "data": "synthetic",
        "config": {"workload": "BASELINE configs[4], per-scan chain: raw 120k-pt scan -> prefilter (distance, voxel grid 0.25, radius outlier) -> GICP odometry; the filtered cloud stays in HBM",
                   "points_per_raw_scan": n, "mean_filtered_points": rv["m"], "mean_iterations": rv["iters"], "converged_frac": rv["conv"] / K, "keyframes": rv["kf"],
                   "prefilter": KITTI_PREFILTER, "odometry": KITTI_ODOMETRY, "keyframe_rule": KITTI_KEYFRAME,
                   "l2": f"inputs larger than L2: {N_FRAMES} distinct raw scans x {fbytes / 1e6:.2f} MB cycled",
                   "parallelism": "replicas only (a chain does not shard)" if world > 1 else "single chain"},
        "e2e": {"value": world * K / (res["e2e"]["ms"] * 1e-3), "unit": "scans/s", "h2d_bytes_per_step": res["e2e"]["stats"]["h2d_bytes"] / K,
                "d2h_bytes_per_step": res["e2e"]["stats"]["d2h_bytes"] / K, "ms_per_step": res["e2e"]["ms"] / K},
        "gpu_launches": int(sum(rv["stats"]["launches"].values())),
        "clocks": rv["clocks"],
        "roofline": roofline,
        "kernel_ms_in_timed_region": {k: round(v, 3) for k, v in st["ms"].items() if v > 0},
        "cpu_baseline": cpu,
    }
    print(json.dumps(line), flush=True)
    if world > 1 and dist.is_initialized():
        dist.destroy_process_group()
