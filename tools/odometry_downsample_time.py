"""Time the odometry mirror's own downsample stage (downsample_method VOXELGRID) on raw VLP-16 frames resident in HBM (development
aid, not part of bench.py):

    python tools/odometry_downsample_time.py [--steps 200] [--warmup 20] [--rounds 5] [--leaf 0.1] [--out record.json]

Arms, on the same seeded 65 536-point frames and bench.py's keyframe parameters (GICP, keyframe_delta_trans 1.0):
  a  the mirror with VOXELGRID and b2r_odometry_prefetch (the next frame filtered on the prefetch stream during this frame's align)
  b  the mirror with VOXELGRID, no prefetch
  c  b2r_voxelgrid_device, then the mirror with NONE on its output
  d  the mirror with NONE on frames filtered beforehand (the floor: no downsample in the timed region)
Every arm starts from a fresh handle, runs `warmup` untimed frames, then `steps` timed frames; the arms alternate in `rounds`
blocks.  A block's time is CUDA-event time on the handle's stream (b2r_get_stream) from before the first timed frame to after the
last; every matching() call returns only once its align has finished, so this is also the host's time per frame.  The per-frame
statuses of a, b and c are compared bitwise.  The card's name and power limit are read in the same run."""
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

KF = dict(keyframe_delta_trans=1.0, keyframe_delta_angle=1.0, keyframe_delta_time=10000.0)  # bench.py


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,driver_version", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable: " + torch.cuda.get_device_name(0)


def status_bits(st):
    return (st["odom"].view(np.uint32).tobytes(), st["trans"].view(np.uint32).tobytes(), st["iterations"], st["converged"], st["keyframe_updated"])


def run_arm(arm, dev, pre, n, sb, leaf, first, count):
    """(ms per timed frame, statuses of the timed frames) of one arm over frames [0, first + count)"""
    reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    method = pkg.B2R_DOWNSAMPLE_VOXELGRID if arm in ("a", "b") else pkg.B2R_DOWNSAMPLE_NONE
    odo = pkg.ScanMatchingOdometry(reg, downsample_method=method, downsample_resolution=leaf, **KF)
    stream = torch.cuda.ExternalStream(reg.getStream())
    fb = n * sb

    def step(i):
        if arm == "a":
            if i + 1 < first + count:
                odo.prefetch_raw(dev.data_ptr() + (i + 1) * fb, n, sb, device=True)
            return odo.matching_raw(0.1 * i, dev.data_ptr() + i * fb, n, sb, device=True)
        if arm == "b":
            return odo.matching_raw(0.1 * i, dev.data_ptr() + i * fb, n, sb, device=True)
        if arm == "c":
            ptr, m, _ = reg.voxelGridFilterDevice(dev.data_ptr() + i * fb, n, sb, leaf)
            return odo.matching_raw(0.1 * i, ptr, m, sb, device=True)
        c = pre[i]
        return odo.matching_raw(0.1 * i, c.data_ptr(), c.shape[0], sb, device=True)

    for i in range(first):
        step(i)
    reg.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    sts = [step(i) for i in range(first, first + count)]
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / count
    odo.close()
    reg.close()
    return ms, sts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to time")
    total = a.warmup + a.steps
    frames = np.stack([synth.scan("vlp16", frame=k, stride=8) for k in range(total)])
    _, n, stride_f = frames.shape
    sb = stride_f * 4
    dev = torch.from_numpy(frames).cuda()
    torch.cuda.synchronize()
    # the floor's inputs: each frame filtered beforehand into a buffer of its own
    reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    pre = []
    for i in range(total):
        filt = reg.voxelGridFilter(frames[i], a.leaf)
        pre.append(torch.from_numpy(np.ascontiguousarray(filt)).cuda())
    reg.close()
    torch.cuda.synchronize()
    arms = ("a", "b", "c", "d")
    t = {k: [] for k in arms}
    ref, identical = None, True
    for _ in range(a.rounds):
        for arm in arms:
            ms, sts = run_arm(arm, dev, pre, n, sb, a.leaf, a.warmup, a.steps)
            t[arm].append(ms)
            if arm != "d":
                bits = [status_bits(s) for s in sts]
                ref = bits if ref is None else ref
                identical = identical and bits == ref
    rec = dict(card=card(), workload="gicp_odometry_vlp16_64k raw frames in HBM, VOXELGRID leaf %g" % a.leaf, points=n,
               filtered_points_mean=float(np.mean([p.shape[0] for p in pre])), steps=a.steps, warmup=a.warmup, rounds=a.rounds,
               arms={"a": "mirror VOXELGRID + prefetch", "b": "mirror VOXELGRID, no prefetch", "c": "b2r_voxelgrid_device + mirror NONE",
                     "d": "mirror NONE on pre-filtered frames (floor)"},
               ms_per_frame={k: dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v)), rounds=v) for k, v in t.items()},
               statuses_a_b_c_bitwise_equal=identical)
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
