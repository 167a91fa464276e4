"""Time MapCloudGenerator::generate from host keyframe arrays against the same map from a b2r_batch's cached keyframes (development
aid, not part of bench.py):

    python tools/map_cloud_time.py [--keyframes 250 1000] [--res 0.05 0] [--steps 5] [--warmup 1] [--rounds 3] [--out record.json]

Keyframes are seeded 16 384-point scans (32-byte pcl::PointXYZI records) at their poses around the synthetic circuit.  Arms:
  pageable  b2r_map_cloud_generate from ordinary (pageable) numpy arrays: every call uploads every keyframe
  pinned    b2r_map_cloud_generate from page-locked arrays
  cached    b2r_batch_map_cloud_generate on the same clouds, added to the batch once beforehand: no point upload
  cached_d  the same, with the result left on the device (d_out) instead of copied to a host array
Every arm writes its result into a host buffer allocated once (cached_d excepted).  The C functions are called directly with
their arguments built beforehand, so the timed region is the library call alone.  A call's time is CUDA-event time on the
engine stream (b2r_get_stream) around it; every call returns only after its results are on the host, so this is also the
caller's time.  The arms alternate in `rounds` blocks of `warmup` untimed and `steps` timed calls; the record keeps each arm's
median over all timed calls, and whether the arms' results are bitwise equal.  The card's name, power limit and clocks are read
in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import hdl_graph_slam_b200 as pkg  # noqa: E402
from hdl_graph_slam_b200 import _capi, synth  # noqa: E402

POINTS = 16384
STRIDE_F = 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem,driver_version", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable: " + torch.cuda.get_device_name(0)


def colmajor(T):
    return np.ascontiguousarray(np.asarray(T, np.float32).T.reshape(-1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, nargs="+", default=[250, 1000])
    ap.add_argument("--res", type=float, nargs="+", default=[0.05, 0.0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to time")
    lib = _capi.load()
    sb = STRIDE_F * 4
    results = []
    for nk in a.keyframes:
        clouds = [synth.scan("vlp16_16k", frame=f, stride=STRIDE_F) for f in range(nk)]
        assert all(c.shape == (POINTS, STRIDE_F) for c in clouds)
        poses = [synth.pose_matrix(f) for f in range(nk)]
        pinned_t = torch.empty((nk, POINTS, STRIDE_F), dtype=torch.float32, pin_memory=True)
        pinned = pinned_t.numpy()
        for k, c in enumerate(clouds):
            pinned[k] = c
        total = nk * POINTS
        lb = pkg.RegistrationBatch(params={"registration_method": "FAST_GICP"})
        ids = [lb.addCloud(c) for c in clouds]
        lb.synchronize()
        stream = torch.cuda.ExternalStream(lb.engine.getStream())
        eng, bh = lb.engine._h, lb._b
        snaps = {}
        for arm, src in (("pageable", clouds), ("pinned", [pinned[k] for k in range(nk)])):
            kf = (_capi.KeyframeSnapshot * nk)()
            for k in range(nk):
                kf[k].points, kf[k].n = src[k].ctypes.data, POINTS
                pc = colmajor(poses[k])
                for j in range(16):
                    kf[k].pose[j] = pc[j]
            snaps[arm] = kf
        idarr = (C.c_int32 * nk)(*ids)
        P = np.concatenate([colmajor(p) for p in poses])
        Pp = P.ctypes.data_as(C.POINTER(C.c_float))
        outs = {arm: np.zeros((total, STRIDE_F), np.float32) for arm in ("pageable", "pinned", "cached")}
        for res in a.res:
            m = C.c_size_t()
            dptr = C.c_void_p()

            def call(arm):
                if arm in ("pageable", "pinned"):
                    o = outs[arm]
                    _capi.check(lib.b2r_map_cloud_generate(eng, snaps[arm], nk, sb, res, o.ctypes.data_as(C.c_void_p), total, C.byref(m)))
                elif arm == "cached":
                    o = outs[arm]
                    _capi.check(lib.b2r_batch_map_cloud_generate(bh, idarr, Pp, nk, res, sb, o.ctypes.data_as(C.c_void_p), total, None, C.byref(m)))
                else:
                    _capi.check(lib.b2r_batch_map_cloud_generate(bh, idarr, Pp, nk, res, sb, None, 0, C.byref(dptr), C.byref(m)))
                return m.value

            arms = ("pageable", "pinned", "cached", "cached_d")
            t = {arm: [] for arm in arms}
            counts = {}
            for _ in range(a.rounds):
                for arm in arms:
                    for _ in range(a.warmup):
                        call(arm)
                    for _ in range(a.steps):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(stream)
                        counts[arm] = call(arm)
                        e1.record(stream)
                        e1.synchronize()
                        t[arm].append(e0.elapsed_time(e1))
            n_out = counts["cached"]
            equal = len(set(counts.values())) == 1 and all(np.array_equal(outs[x][:n_out].view(np.uint32), outs["cached"][:n_out].view(np.uint32))
                                                          for x in ("pageable", "pinned"))
            results.append(dict(keyframes=nk, points=total, resolution=res, map_points=n_out, upload_bytes=total * sb,
                                ms={arm: dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v))) for arm, v in t.items()},
                                results_bitwise_equal=bool(equal)))
            print(json.dumps(results[-1]), flush=True)
        lb.close()
        del pinned, pinned_t
    rec = dict(card=card(), workload="map cloud of N keyframes x 16 384-point vlp16_16k scans (32-byte records) at their circuit poses",
               steps=a.steps, warmup=a.warmup, rounds=a.rounds,
               arms={"pageable": "b2r_map_cloud_generate, pageable keyframe arrays", "pinned": "b2r_map_cloud_generate, pinned keyframe arrays",
                     "cached": "b2r_batch_map_cloud_generate, host output", "cached_d": "b2r_batch_map_cloud_generate, device output (d_out)"},
               results=results)
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
