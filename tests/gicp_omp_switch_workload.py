"""One pass over the pclomp GICP (`B200_GICP_OMP`) code the diagnostic switches select, for test_gicp_omp_switches_gpu, which runs it in
a fresh process per switch (the engine reads each switch once per process).  Every align starts from a guess with metres of
translation, so the pose rule of the cost passes is exercised: a pair at 100 000 points (the (16, 8) cluster build) and one at 140 000
(the chained build), the covariances at k = 20 and 49 of a 16 384-point cloud, a 6-pair mixed-size batch with fitness, a 24-pair loop
batch through b2r_batch_align and the single-rank b2r_batch_loop_detect (two lanes under B2R_BATCH_LANES=2, several chunks under
B2R_BATCH_CHUNK), and a 4-frame odometry mirror with every next frame announced.  Writes every output to the .npz file named on the
command line."""
import sys

import numpy as np

import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import batch, synth
from gicp_pcl_ref import pose, scene, transform

P = {"registration_method": "B200_GICP_OMP"}
MOVE = pose((3.3, -2.2, 0.03), (0.0, 0.0, 0.04))
GUESS = (pose((0.03, -0.02, 0.0), (0.0, 0.0, 0.005)) @ np.linalg.inv(MOVE.astype(np.float64))).astype(np.float32)


def pair(n, seed):
    return scene(n, seed=seed), transform(scene(n, seed=seed + 1), MOVE)


def single(tgt, src):
    r = pkg.select_registration_method(P)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    r.align(GUESS)
    out = np.r_[r.getFinalTransformation().astype(np.float64).reshape(-1), r.nr_iterations, r.hasConverged(), r.getFitnessScore(2.5)]
    covs = (r.getCovariances(0, src.shape[0]), r.getCovariances(1, tgt.shape[0]))
    r.close()
    return out, covs


def records(res):
    return np.array([np.r_[np.asarray(x["T"], np.float64).reshape(-1), x["iterations"], x["converged"], x["fitness"]] for x in res])


def run():
    res = {}
    for n, seed in ((100000, 100), (140000, 102)):
        res[f"align_{n}"], _ = single(*pair(n, seed))
    c = scene(16384, seed=120)
    for k in (20, 49):
        r = pkg.select_registration_method(dict(P, reg_correspondence_randomness=str(k)))
        r.setInputSource(c)
        res[f"cov_k{k}"] = r.getCovariances(0, c.shape[0])
        r.close()
    clouds = [transform(scene(n, seed=110 + i), pose((0.1 * i, -0.05 * i, 0.0), (0.0, 0.0, 0.01 * i)))
              for i, n in enumerate((16384, 4096, 33000, 1025, 65536, 9000, 140000))]
    b = pkg.RegistrationBatch(params=P)
    ids = [b.addCloud(c) for c in clouds]
    pairs = [(ids[1], ids[0]), (ids[2], ids[0]), (ids[3], ids[4]), (ids[4], ids[6]), (ids[5], ids[2]), (ids[6], ids[4])]
    res["batch"] = records(b.align([(s, t, pose((1.5, -1.0, 0.0))) for s, t in pairs], True, 2.5))
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
    frames = [transform(scene(20000, seed=130 + i), pose((0.1 * i, 0.0, 0.0), (0.0, 0.0, 0.01 * i))) for i in range(4)]
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
