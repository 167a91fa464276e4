"""One pass over the NDT_OMP KDTREE (`B200_NDT_KDTREE`) code the diagnostic switches select, for test_ndt_kdtree_switches_gpu, which runs it
in a fresh process per switch (the engine reads each switch once per process): both derivative passes and the Hessian-only pass of a
131 072-point pair, an align of it with the line search active, a 6-pair mixed-size batch with fitness, a 24-pair loop batch through
b2r_batch_align and the single-rank b2r_batch_loop_detect (two lanes under B2R_BATCH_LANES=2, several chunks under B2R_BATCH_CHUNK), and a
4-frame odometry mirror with every next frame announced.  Writes every output to the .npz file named on the command line."""
import sys

import numpy as np

import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import batch, synth

P = {"registration_method": "B200_NDT_KDTREE", "reg_resolution": "1.0"}
POSE = np.array([0.1, -0.05, 0.02, 0.01, -0.02, 0.03])


def cfg(flag=0):
    c = pkg.default_config(pkg.B2R_METHOD_NDT_KDTREE)
    c.ndt_resolution = 1.0
    c.ndt_mt_interval_flag = flag
    return c


def records(res):
    return np.array([np.r_[np.asarray(x["T"], np.float64).reshape(-1), x["iterations"], x["converged"], x["fitness"]] for x in res])


def run():
    res = {}
    tgt, src = synth.scan("hdl32e", frame=0, stride=8), synth.scan("hdl32e", frame=1, stride=8)
    r = pkg.Registration(cfg(1))
    r.setInputTarget(tgt)
    r.setInputSource(src)
    s, g, H, n = r.ndtDerivativesAt(POSE)
    res["deriv"] = np.r_[s, g, H.reshape(-1), n]
    res["hess"] = r.ndtHessianAt(POSE).reshape(-1)
    cnt, keys = r.ndtNeighborsAt(POSE, src.shape[0])
    res["neighbours"] = np.r_[cnt.astype(np.int64), keys]
    r.align(np.eye(4, dtype=np.float32))
    res["align"] = np.r_[r.getFinalTransformation().astype(np.float64).reshape(-1), r.nr_iterations, r.hasConverged(), r.getFitnessScore(2.5)]
    r.close()
    clouds = [synth.scan(s, frame=f, stride=8) for s, f in (("vlp16_16k", 0), ("vlp16_16k", 1), ("vlp16", 2), ("hdl32e", 3), ("vlp16_16k", 4),
                                                             ("vlp16", 5), ("hdl32e", 6))]
    for flag in (0, 1):
        b = pkg.RegistrationBatch(cfg=cfg(flag))
        ids = [b.addCloud(c) for c in clouds]
        pairs = [(ids[1], ids[0]), (ids[2], ids[0]), (ids[3], ids[4]), (ids[4], ids[6]), (ids[5], ids[2]), (ids[6], ids[3])]
        res[f"batch_{flag}"] = records(b.align([(s, t, np.eye(4, dtype=np.float32)) for s, t in pairs], True, 2.5))
        b.close()
    groups, guesses, group_first = batch.loop_workload(3, "vlp16_16k")
    lf = sorted({f for tf, sfs in groups for f in [tf] + list(sfs)})
    lb = pkg.RegistrationBatch(params=P)
    ids = {f: lb.addCloud(synth.scan("vlp16_16k", frame=f, stride=8)) for f in lf}
    lpairs = [(ids[sf], ids[tf], guesses[group_first[g] + i]) for g, (tf, sfs) in enumerate(groups) for i, sf in enumerate(sfs)]
    res["loop_align"] = records(lb.align(lpairs, True, 2.5))
    best, det = lb.loopDetect(lpairs, group_first, 2.5, 0.5)
    res["loop_detect"] = records(det)
    res["loop_best"] = np.asarray(best, np.int64)
    lb.close()
    frames = [synth.scan("vlp16_16k", frame=k, stride=8, step=0.1) for k in range(4)]
    reg = pkg.select_registration_method(P)
    odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=0.25, publish_status=True)
    rows = []
    for i, f in enumerate(frames):
        if i + 1 < len(frames):
            nxt = frames[i + 1]
            odo.prefetch_raw(nxt.ctypes.data, nxt.shape[0], nxt.shape[1] * 4)
        st = odo.matching(0.1 * i, f)
        rows.append(np.r_[np.asarray(st["trans"], np.float64).reshape(-1), st["iterations"], st["converged"], st["keyframe_updated"]])
    odo.close()
    reg.close()
    res["odometry"] = np.array(rows)
    return res


if __name__ == "__main__":
    np.savez(sys.argv[1], **run())
