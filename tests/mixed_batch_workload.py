"""Mixed-size pcl ICP / pcl GICP loop batches (test_mixed_batches_gpu): sources of 0 to 140 000 points against targets of other sizes,
a pair that converges at iteration 1 (a cloud against itself), pairs that run to the iteration limit (a small limit)
and a pair too far apart to reach the correspondence minimum.  Run as a script it writes every record of the batch (co-scheduled, each
pair alone, and b2r_batch_loop_detect) to an .npz file, so the test can repeat it in a child process under a diagnostic switch."""
import sys

import numpy as np

import hdl_graph_slam_b200 as pkg
from gicp_pcl_ref import pose, scene, transform

# limits below what the 16 384- to 140 000-point pairs need, so they stop at the limit.  ICP takes a tiny epsilon; pcl GICP keeps the
# factory's 0.01, since its test "moved less than epsilon" on a 1e-6 scale would be decided by the last bits of the BFGS line search
MAX_ITERATIONS = {"B200_ICP": 10, "GICP": 2}
EPSILON = {"B200_ICP": 1e-6, "GICP": 0.01}
METHODS = {"B200_ICP": "ICP", "GICP": "GICP"}


def params(method, reciprocal=False):
    p = {"registration_method": method, "reg_maximum_iterations": str(MAX_ITERATIONS[method]), "reg_transformation_epsilon": str(EPSILON[method])}
    if method == "B200_ICP":
        p["reg_use_reciprocal_correspondences"] = "true" if reciprocal else "false"
    return p


def small(n, seed):
    """n points picked from a 4096-point scene (so they have neighbours in it), moved by a few centimetres"""
    base = scene(4096, seed=90)
    rng = np.random.default_rng(seed)
    return transform(base[rng.choice(4096, n, replace=False)], pose((0.03, -0.02, 0.0)))


def clouds_and_pairs():
    """clouds (targets first) and (source index, target index, guess) pairs"""
    sizes_t = [4096, 2048, 16384, 70000, 140000, 1025]
    clouds = [scene(n, seed=80 + i) for i, n in enumerate(sizes_t[:5])]
    clouds.append(scene(4096, seed=90)[:1025])
    tid = {n: i for i, n in enumerate(sizes_t)}
    mv = pose((0.25, -0.15, 0.02), (0.0, 0.0, 0.03))
    src = [
        (np.zeros((0, 4), np.float32), tid[4096], np.eye(4)),
        (small(1, 1), tid[4096], np.eye(4)),
        (small(3, 3), tid[4096], np.eye(4)),
        (small(4, 4), tid[4096], np.eye(4)),
        (small(33, 33), tid[4096], np.eye(4)),
        (transform(scene(4096, seed=90)[:1025], mv), tid[1025], np.eye(4)),
        (transform(scene(16384, seed=91), mv), tid[70000], np.eye(4)),
        (transform(scene(70000, seed=92), mv), tid[140000], np.eye(4)),
        (transform(scene(140000, seed=93), mv), tid[16384], np.eye(4)),
        (None, tid[2048], np.eye(4)),                    # the target itself: converges at iteration 1
        (transform(scene(16384, seed=94), mv), tid[16384], pose((500.0, 0.0, 0.0))),  # too far: below the correspondence minimum
    ]
    pairs = []
    for c, t, g in src:
        if c is None:
            pairs.append((t, t, g.astype(np.float32)))
            continue
        clouds.append(c)
        pairs.append((len(clouds) - 1, t, g.astype(np.float32)))
    return clouds, pairs


def record(x):
    return np.r_[np.asarray(x["T"], np.float64).reshape(-1), x["iterations"], x["converged"], x["fitness"]]


def run_batch(method, reciprocal=False):
    clouds, pairs = clouds_and_pairs()
    b = pkg.RegistrationBatch(params=params(method, reciprocal))
    ids = [b.addCloud(c) for c in clouds]
    bp = [(ids[s], ids[t], g) for s, t, g in pairs]
    together = b.align(bp, True, 2.5)
    alone = [b.align([p], True, 2.5)[0] for p in bp]
    n = len(bp)
    _, loop = b.loopDetect(bp, [0, 4, 8, n], 2.5, 0.5)
    b.close()
    return dict(together=np.array([record(x) for x in together]), alone=np.array([record(x) for x in alone]),
                loop=np.array([np.r_[np.asarray(x["T"], np.float64).reshape(-1), x["converged"], x["fitness"]] for x in loop]))


def main(out):
    res = {}
    for method in METHODS:
        for rec in ((False, True) if method == "B200_ICP" else (False,)):
            for k, v in run_batch(method, rec).items():
                res[f"{METHODS[method]}_{int(rec)}_{k}"] = v
    np.savez(out, **res)


if __name__ == "__main__":
    main(sys.argv[1])
