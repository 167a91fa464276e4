"""One pass over the code every diagnostic switch selects (README, "Environment switches"), run in a fresh process per
configuration because the engine reads each switch once per process.  Prints, as its last line, one JSON object: a SHA-1 per
output (NaN mapped to a fixed value first) and, under "anchor", the few raw values tests/test_diagnostic_switches_gpu.py checks
against the oracle.  Used by that test as `python tests/switch_workload.py`."""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]

import hdl_graph_slam_b200 as pkg  # noqa: E402
from hdl_graph_slam_b200 import synth  # noqa: E402
from common import perturb  # noqa: E402

I4 = np.eye(4, dtype=np.float32)
KF = dict(keyframe_delta_trans=1.5, keyframe_delta_angle=1.0, keyframe_delta_time=10000.0)
NDT_P = [0.9, 0.05, -0.02, 0.01, -0.015, 0.03]


def sha(*arrays):
    h = hashlib.sha1()
    for a in arrays:
        a = np.ascontiguousarray(a)
        if a.dtype.kind == "f":
            a = np.nan_to_num(a.astype(np.float64), nan=-7.0, posinf=7e300, neginf=-7e300)
        h.update(a.tobytes())
    return h.hexdigest()


def status_rows(sts):
    return np.stack([np.concatenate([st["odom"].reshape(-1).view(np.uint32), st["trans"].reshape(-1).view(np.uint32),
                                     [st["iterations"], st["converged"], st["keyframe_updated"], st["frame_rejected"]]]).astype(np.uint64)
                     for st in sts])


def odometry(frames, announce, **kw):
    """ScanMatchingOdometry over `frames`; announce: b2r_odometry_prefetch of the next frame before each matching call"""
    reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    odo = pkg.ScanMatchingOdometry(reg, **dict(KF, **kw))
    sts = []
    for k, c in enumerate(frames):
        if announce and k + 1 < len(frames):
            nxt = frames[k + 1]
            odo.prefetch_raw(nxt.ctypes.data, nxt.shape[0], nxt.shape[1] * 4)
        sts.append(odo.matching(0.1 * k, c))
    odo.close()
    reg.close()
    return sts


def run():
    out, anchor = {}, {}
    # ---- GICP odometry on VLP-16 frames (65 536 points): with the next frame announced (prefetch stream, overlapped
    # covariances), then the strict chain; then the nodelet's own VOXELGRID downsample on the raw frames
    vlp = [synth.scan("vlp16", frame=k, stride=8) for k in range(6)]
    for name, announce, kw in (("odometry_prefetch", True, {}), ("odometry_strict", False, {}),
                               ("odometry_voxelgrid", True, dict(downsample_method=pkg.B2R_DOWNSAMPLE_VOXELGRID, downsample_resolution=0.1))):
        sts = odometry(vlp, announce, **kw)
        out[name] = sha(status_rows(sts))
        if name == "odometry_strict":
            anchor["odometry_trans1"] = sts[1]["trans"].astype(np.float64).tolist()
            anchor["odometry_iterations1"] = int(sts[1]["iterations"])
    # one GICP pair on the single-pair path, with its correspondences
    reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    reg.setInputTarget(vlp[0])
    reg.setInputSource(vlp[1])
    reg.align(I4)
    corr = reg.getCorrespondences(vlp[1].shape[0])
    out["gicp_pair"] = sha(reg.getFinalTransformation(), np.array([reg.nr_iterations, reg.hasConverged()]), corr)
    anchor["gicp_T"] = reg.getFinalTransformation().astype(np.float64).tolist()
    anchor["gicp_iterations"] = reg.nr_iterations
    anchor["gicp_corr"] = sha(corr)
    # ---- k-NN and covariances on a 100 000-point target
    big = synth.scan("hdl32e", frame=3, stride=8)[:100000].copy()
    big[::97, :3] = np.round(big[::97, :3])
    q = synth.scan("vlp16_16k", frame=4, stride=8)
    reg.setInputTarget(big)
    idx, d2 = reg.nearestKSearch(q)
    out["nearest"] = sha(idx, d2.view(np.uint32))
    out["covariances"] = sha(reg.getCovariances(1, big.shape[0]))
    # ---- voxel grid: a 120 000-point KITTI-shape scan and a 100 000-point cloud
    kitti = synth.scan("kitti", frame=2, stride=8)
    for name, c, leaf in (("voxelgrid_kitti", kitti, 0.1), ("voxelgrid_100k", big, 0.25)):
        o, keys, counts, rc = reg.voxelGridFilter(c, leaf, with_keys=True)
        out[name] = sha(o.view(np.uint32), keys, counts, np.array([rc]))
    # ---- prefilter with each outlier method
    for method in (0, 1, 2):
        o, _, m = reg.prefilter(kitti, distance_near_thresh=1.0, distance_far_thresh=60.0, downsample_method=1, downsample_resolution=0.1,
                                outlier_removal_method=method, statistical_mean_k=20, statistical_stddev=1.0, radius_radius=0.5,
                                radius_min_neighbors=2)
        out[f"prefilter_{method}"] = sha(o.view(np.uint32), np.array([m]))
    reg.close()
    # ---- NDT on a 131 072-point source: derivative and Hessian passes at one pose, then aligns with DIRECT7 and DIRECT1
    src = synth.scan("hdl32e", frame=1, stride=8)
    tgt = synth.scan("hdl32e", frame=0, stride=8)
    for search in ("DIRECT7", "DIRECT1"):
        r = pkg.select_registration_method({"registration_method": "NDT_OMP", "reg_resolution": 1.0, "reg_nn_search_method": search})
        r.setInputTarget(tgt)
        r.setInputSource(src)
        score, g, H, npairs = r.ndtDerivativesAt(NDT_P)
        Hh = r.ndtHessianAt(NDT_P)
        out[f"ndt_derivatives_{search}"] = sha(np.array([score]), g, H, np.array([npairs]), Hh)
        if search == "DIRECT7":
            anchor["ndt"] = dict(score=score, g=g.tolist(), H=H.tolist(), npairs=int(npairs))
        r.align(perturb(11, 0.3, 1.5).astype(np.float32))
        out[f"ndt_align_{search}"] = sha(r.getFinalTransformation(), np.array([r.nr_iterations, r.hasConverged()]))
        r.close()
    # ---- GICP batch of 16 pairs (two lanes need 16) with fitness, loop detection and fitness scores
    clouds, pairs, gf = {}, [], [0]
    for gi, tf in enumerate((0, 10)):
        clouds.setdefault(tf, synth.scan("vlp16_16k", frame=tf, stride=8))
        for j, off in enumerate((1, 251, 2, 252, 3, 253, 4, 254)):
            sf = tf + off
            clouds.setdefault(sf, synth.scan("vlp16_16k", frame=sf, stride=8))
            rel = np.linalg.inv(synth.pose_matrix(tf)) @ synth.pose_matrix(sf)
            gg = (rel @ perturb(60 + 7 * gi + j, 0.3, 2.0)).astype(np.float32)
            gg[2, 3] = 0.0
            pairs.append((sf, tf, gg))
        gf.append(len(pairs))
    lb = pkg.RegistrationBatch(params={"registration_method": "FAST_GICP"})
    ids = {f: lb.addCloud(c) for f, c in clouds.items()}
    pl = [(ids[s], ids[t], gg) for s, t, gg in pairs]
    res = lb.align(pl, True, 2.5)
    out["gicp_batch"] = sha(np.stack([r["T"] for r in res]), np.array([[r["iterations"], r["converged"]] for r in res]),
                            np.array([r["fitness"] for r in res]))
    best, lres = lb.loopDetect(pl, gf, 2.5, 0.5)
    out["loop_detect"] = sha(np.array(best), np.stack([r["T"] for r in lres]), np.array([r["fitness"] for r in lres]))
    out["fitness_scores"] = sha(lb.calcFitnessScore([(t, s, gg) for s, t, gg in pl], 2.0))
    lb.close()
    # ---- NDT batch of mixed sizes
    cfg = pkg.default_config(pkg.B2R_METHOD_NDT)
    cfg.ndt_resolution = 1.0
    nclouds = {"a": synth.scan("vlp16_16k", frame=0, stride=8), "b": synth.scan("vlp16", frame=1, stride=8), "c": src,
               "d": synth.scan("vlp16_16k", frame=2, stride=8)[:5000].copy(), "e": tgt}
    npairs_ = [("b", "a", I4), ("a", "b", perturb(3, 0.2, 1.0)), ("c", "e", I4), ("d", "a", perturb(4, 0.2, 1.0)), ("e", "c", perturb(5, 0.2, 1.0))]
    lb = pkg.RegistrationBatch(cfg=cfg)
    nids = {k: lb.addCloud(c) for k, c in nclouds.items()}
    res = lb.align([(nids[s], nids[t], np.asarray(gg, np.float32)) for s, t, gg in npairs_], True, 2.5)
    out["ndt_batch"] = sha(np.stack([r["T"] for r in res]), np.array([[r["iterations"], r["converged"]] for r in res]),
                           np.array([r["fitness"] for r in res]))
    lb.close()
    # ---- pcl NDT (the factory's NDT branch) on the same 131 072-point source: derivative and Hessian passes at one pose, an
    # align with each line-search polarity, then the mixed-size batch
    for flag in (0, 1):
        pcfg = pkg.default_config(pkg.B2R_METHOD_NDT_PCL)
        pcfg.ndt_resolution = 1.0
        pcfg.ndt_mt_interval_flag = flag
        r = pkg.Registration(pcfg)
        r.setInputTarget(tgt)
        r.setInputSource(src)
        if flag == 0:
            score, g, H, npairs = r.ndtDerivativesAt(NDT_P)
            Hh = r.ndtHessianAt(NDT_P)
            out["ndt_pcl_derivatives"] = sha(np.array([score]), g, H, np.array([npairs]), Hh)
            anchor["ndt_pcl"] = dict(score=score, g=g.tolist(), H=H.tolist(), npairs=int(npairs))
        r.align(perturb(11, 0.3, 1.5).astype(np.float32))
        out[f"ndt_pcl_align_flag{flag}"] = sha(r.getFinalTransformation(), np.array([r.nr_iterations, r.hasConverged()]))
        r.close()
    pcfg = pkg.default_config(pkg.B2R_METHOD_NDT_PCL)
    pcfg.ndt_resolution = 1.0
    lb = pkg.RegistrationBatch(cfg=pcfg)
    nids = {k: lb.addCloud(c) for k, c in nclouds.items()}
    res = lb.align([(nids[s], nids[t], np.asarray(gg, np.float32)) for s, t, gg in npairs_], True, 2.5)
    out["ndt_pcl_batch"] = sha(np.stack([r["T"] for r in res]), np.array([[r["iterations"], r["converged"]] for r in res]),
                               np.array([r["fitness"] for r in res]))
    lb.close()
    return out, anchor


if __name__ == "__main__":
    o, a = run()
    print(json.dumps(dict(outputs=o, anchor=a)))
