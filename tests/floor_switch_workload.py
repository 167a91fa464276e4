"""Child process of test_floor_switches_gpu.py: runs a fixed set of floor-detection calls under whatever diagnostic switches the
environment sets and writes every output to the .npz named by argv[1]."""
import sys

import numpy as np
import torch  # noqa: F401  (before the engine library)
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import synth

from floor_ref import LAUNCH


def main(path):
    reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    out = {}
    cases = [("vlp16", 0, "hdl"), ("hdl32e", 1, "501"), ("kitti", 2, "hdl"), ((64, 4096), 3, "hdl")]
    rng = np.random.default_rng(9)
    noise = np.zeros((4000, 8), np.float32)
    noise[:, :3] = rng.uniform([-30, -30, -3], [30, 30, -1], (4000, 3))
    for i, (sensor, frame, launch) in enumerate(cases + [(None, 0, "noise")]):
        if sensor is None:
            c, kw = noise, dict(use_normal_filtering=0, floor_pts_thresh=0)
        else:
            c, kw = synth.scan(sensor, frame=frame, stride=8), LAUNCH[launch]
        r = reg.floor_detect(c, **kw)
        for k in ("detected", "n_filtered", "n_inliers", "ransac_iterations", "model_indices", "coeffs", "filtered", "inliers"):
            out[f"{i}_{k}"] = np.asarray(r[k])
        out[f"{i}_reason"] = np.array(r["reason"])
    reg.close()
    np.savez(path, **out)


if __name__ == "__main__":
    main(sys.argv[1])
