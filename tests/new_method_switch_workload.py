"""One pass over the four registration methods served last (pcl GICP `GICP`, pcl ICP `B200_ICP`, FastVGICP `FAST_VGICP` and
FastVGICPCuda `B200_VGICP_CUDA`) for test_new_method_switches_gpu, which runs it in a fresh process per diagnostic switch (the engine
reads each switch once per process).  Per method: a pair at 100 000 points (the (16, 8) cluster build, (8, 16) under B2R_NO_CLUSTER16),
a pair at 140 000 points (the chained build above the one-cluster limit), the covariances at k = 20 and 49 of a 16 384-point cloud (the
covariance methods), a 6-pair mixed-size batch with fitness and a 4-frame odometry mirror with every next frame announced.  Writes
every output to the .npz file named on the command line."""
import sys

import numpy as np

import hdl_graph_slam_b200 as pkg
from gicp_pcl_ref import pose, scene, transform

METHODS = {"GICP": {}, "B200_ICP": {}, "FAST_VGICP": {"reg_resolution": "1.0"}, "B200_VGICP_CUDA": {"reg_resolution": "1.0"}}
COV_METHODS = ("GICP", "FAST_VGICP", "B200_VGICP_CUDA")
MOVE = pose((0.3, -0.2, 0.03), (0.0, 0.0, 0.04))


def params(method, **extra):
    p = {"registration_method": method}
    p.update(METHODS[method])
    p.update({k: str(v) for k, v in extra.items()})
    return p


def pair(n, seed):
    return scene(n, seed=seed), transform(scene(n, seed=seed + 1), MOVE)


def cov_cloud():
    return scene(16384, seed=120)


def single(method, tgt, src):
    r = pkg.select_registration_method(params(method))
    r.setInputTarget(tgt)
    r.setInputSource(src)
    r.align(np.eye(4, dtype=np.float32))
    out = np.r_[r.getFinalTransformation().astype(np.float64).reshape(-1), r.nr_iterations, r.hasConverged(), r.getFitnessScore(2.5)]
    covs = (r.getCovariances(0, src.shape[0]), r.getCovariances(1, tgt.shape[0])) if method in COV_METHODS else None
    r.close()
    return out, covs


def run(method):
    res = {}
    for n, seed in ((100000, 100), (140000, 102)):
        tgt, src = pair(n, seed)
        res[f"align_{n}"], _ = single(method, tgt, src)
    if method in COV_METHODS:
        c = cov_cloud()
        for k in (20, 49):
            r = pkg.select_registration_method(params(method, reg_correspondence_randomness=k))
            r.setInputSource(c)
            res[f"cov_k{k}"] = r.getCovariances(0, c.shape[0])
            r.close()
    clouds = [transform(scene(n, seed=110 + i), pose((0.1 * i, -0.05 * i, 0.0), (0.0, 0.0, 0.01 * i)))
              for i, n in enumerate((16384, 4096, 33000, 1025, 65536, 9000, 140000))]
    b = pkg.RegistrationBatch(params=params(method))
    ids = [b.addCloud(c) for c in clouds]
    pairs = [(ids[1], ids[0]), (ids[2], ids[0]), (ids[3], ids[4]), (ids[4], ids[6]), (ids[5], ids[2]), (ids[6], ids[4])]
    out = b.align([(s, t, np.eye(4, dtype=np.float32)) for s, t in pairs], True, 2.5)
    b.close()
    res["batch"] = np.array([np.r_[np.asarray(x["T"], np.float64).reshape(-1), x["iterations"], x["converged"], x["fitness"]] for x in out])
    frames = [transform(scene(20000, seed=130 + i), pose((0.1 * i, 0.0, 0.0), (0.0, 0.0, 0.01 * i))) for i in range(4)]
    reg = pkg.select_registration_method(params(method))
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


def main(out):
    np.savez(out, **{f"{m}_{k}": v for m in METHODS for k, v in run(m).items()})


if __name__ == "__main__":
    main(sys.argv[1])
