"""A pcl ICP workload whose outputs must not depend on the engine's diagnostic switches (run by test_icp_pcl_switches_gpu in a child
process with one switch set): a reciprocal-on and -off odometry chain and a 24-pair loop batch, written to an .npz file."""
import sys

import numpy as np

import hdl_graph_slam_b200 as pkg
from gicp_pcl_ref import pose, scene, transform


def main(out):
    res = {}
    clouds = [transform(scene(16384, seed=50 + i), pose((0.12 * i, 0.03 * i, 0.0), (0.0, 0.0, 0.012 * i))) for i in range(6)]
    for rec in ("false", "true"):
        r = pkg.select_registration_method({"registration_method": "B200_ICP", "reg_use_reciprocal_correspondences": rec})
        o = pkg.ScanMatchingOdometry(r, keyframe_delta_trans=0.0, keyframe_delta_angle=0.0, keyframe_delta_time=0.0)
        odo = []
        for k, c in enumerate(clouds):
            st = o.matching(0.1 * k, c)
            odo.append(np.r_[st["trans"].reshape(-1).astype(np.float64), st["iterations"], st["converged"]])
        res["odometry_" + rec] = np.array(odo)
        o.close()
        lb = pkg.RegistrationBatch(params={"registration_method": "B200_ICP", "reg_use_reciprocal_correspondences": rec})
        ids = [lb.addCloud(c) for c in clouds]
        pairs = [(ids[i % 6], ids[(i + 1 + i // 6) % 6], pose((0.02 * (i % 3), 0.0, 0.0))) for i in range(24)]
        out_b = lb.align(pairs, True, 2.5)
        res["batch_" + rec] = np.array([np.r_[x["T"].reshape(-1).astype(np.float64), x["iterations"], x["converged"], x["fitness"]] for x in out_b])
        lb.close()
    np.savez(out, **res)


if __name__ == "__main__":
    main(sys.argv[1])
