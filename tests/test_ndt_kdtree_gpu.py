"""GPU: NDT_OMP's KDTREE search (B2R_METHOD_NDT_KDTREE, opted into as B200_NDT_KDTREE) against the sequential CPU reference
tests/ndt_kdtree_ref.cpp: the voxel map bitwise NDT_OMP's, centroids and radius neighbour lists bit for bit, n_pairs the pcl NDT handle's,
both passes to rel 1e-9 at 16k, 64k and 131 072 points and 3.6 km from the origin, aligns with the reference's iterations and flag and
a pose within 1e-4, fitness the oracle's; and every caller (loop matching, the batch co-scheduled and alone, the fitness batch, the
single-rank loop detector, the odometry mirror with and without its own downsample and the announced next frame) bitwise the single
handle."""
import ctypes as C

import numpy as np
import pytest

import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi
from common import rot_err, trans_err, perturb
from ndt_kdtree_ref import Reference
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

KD = "B200_NDT_KDTREE"
MAXR = 2.5
POSES = [np.zeros(6), np.array([0.1, -0.05, 0.02, 0.01, -0.02, 0.03]), np.array([0.4, 0.3, -0.1, 0.2, -0.1, 0.6])]


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("ndt_kdtree_ref"))


def kd_cfg(res=1.0, flag=0, fixed=0, method=pkg.B2R_METHOD_NDT_KDTREE):
    c = pkg.default_config(method)
    c.ndt_resolution = res
    c.ndt_mt_interval_flag = flag
    c.ndt_fixed_iterations = fixed
    return c


def handle(cfg, tgt, src):
    r = pkg.Registration(cfg)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    return r


def rel(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


def shifted(c, off):
    c = c.copy()
    c[:, :3] += np.asarray(off, np.float32)
    return c


def about(p, off):
    """the pose p about the point off (the same relative motion far from the origin)"""
    q = np.array(p, np.float64)
    if any(off):
        from ndt_pcl_ref import pose_matrix
        T = pose_matrix(p).astype(np.float64)
        q[:3] = (T[:3, :3] @ -np.asarray(off, np.float64) + np.asarray(off, np.float64)) + T[:3, 3]
    return q


def test_factory_mapping_defaults_and_refused_names():
    r = pkg.select_registration_method({"registration_method": KD})
    c = r.config
    assert c.method == pkg.B2R_METHOD_NDT_KDTREE == 9
    assert (c.ndt_resolution, c.transformation_epsilon, c.max_iterations, c.ndt_step_size, c.ndt_outlier_ratio, c.ndt_mt_interval_flag,
            c.ndt_fixed_iterations) == (0.5, 0.01, 64, 0.1, 0.55, 0, 0)
    r.close()
    r = pkg.select_registration_method({"registration_method": KD, "reg_resolution": "1.0", "reg_transformation_epsilon": "0.02",
                                        "reg_maximum_iterations": "30", "reg_nn_search_method": "DIRECT1"})  # the search method is not read
    c = r.config
    assert (c.method, c.ndt_resolution, c.transformation_epsilon, c.max_iterations) == (9, 1.0, 0.02, 30)
    r.close()
    for name in ("NDT_OMP", "B200_NDT"):
        with pytest.raises(pkg.B2RError) as e:
            pkg.select_registration_method({"registration_method": name, "reg_nn_search_method": "KDTREE"})
        assert e.value.code == _capi.B2R_EUNSUPPORTED
    with pytest.raises(pkg.B2RError) as e:
        pkg.select_registration_method({"registration_method": "NDT_KDTREE"})
    assert e.value.code == _capi.B2R_EUNSUPPORTED
    lib = pkg.load_library()
    cfg = _capi.Config()
    assert lib.b2r_config_default(C.byref(cfg), 7) == _capi.B2R_EINVAL
    assert lib.b2r_config_default(C.byref(cfg), pkg.B2R_METHOD_NDT_KDTREE) == _capi.B2R_OK and cfg.ndt_resolution == 0.5


@pytest.mark.parametrize("case,res", [("16k", 0.5), ("64k", 0.7), ("131k", 1.0), ("16k_far", 1.0), ("64k_far", 0.5)])
def test_map_neighbours_and_passes_match_the_reference(ref, synth, case, res):
    sensor = {"16k": "vlp16_16k", "64k": "vlp16", "131k": "hdl32e"}[case.split("_")[0]]
    off = (3600.0, -150.0, 20.0) if case.endswith("far") else (0.0, 0.0, 0.0)
    tgt, src = shifted(synth.scan(sensor, frame=0, stride=8), off), shifted(synth.scan(sensor, frame=1, stride=8), off)
    M = ref.map(tgt, res)
    r = handle(kd_cfg(res), tgt, src)
    omp = handle(kd_cfg(res, method=pkg.B2R_METHOD_NDT), tgt, src)
    pcl = handle(kd_cfg(res, method=pkg.B2R_METHOD_NDT_PCL), tgt, src)
    v, vo = r.ndtGetVoxels(), omp.ndtGetVoxels()
    for k in v:
        assert np.asarray(v[k]).tobytes() == np.asarray(vo[k]).tobytes(), k
    rv = M.voxels()
    assert np.array_equal(v["keys"], rv["keys"]) and np.array_equal(v["npts"], rv["npts"])
    k, c = r.ndtGetCentroids()
    rk, rc = M.centroids()
    assert k.size > 100 and np.array_equal(k, rk) and np.array_equal(c.view(np.uint32), rc.view(np.uint32))
    for p0 in POSES:
        p = about(p0, off)
        cnt, keys = r.ndtNeighborsAt(p, src.shape[0])
        rcnt, rkeys = M.neighbors(src, p)
        assert np.array_equal(cnt, rcnt) and np.array_equal(keys, rkeys), f"neighbours at {p0}"
        s, g, H, npairs = r.ndtDerivativesAt(p)
        o = M.derivatives(src, p)
        assert npairs == o["n_pairs"] == keys.size == pcl.ndtDerivativesAt(p)[3] and npairs > 0
        assert abs(s - o["score"]) <= 1e-9 * abs(o["score"]) and rel(g, o["g"]) <= 1e-9 and rel(H, o["H"]) <= 1e-9
        assert rel(r.ndtHessianAt(p), M.hessian_at(src, p)) <= 1e-9
        again = r.ndtDerivativesAt(p)
        assert again[0] == s and np.array_equal(again[1], g) and np.array_equal(again[2], H) and again[3] == npairs
        # not an alias of DIRECT7: the same pose gives other sums
        so, go, Ho, _ = omp.ndtDerivativesAt(p)
        assert so != s and not np.array_equal(go, g)
    for h in (r, omp, pcl):
        h.close()


@pytest.mark.parametrize("sensor,res,fixed", [("vlp16_16k", 1.0, 0), ("vlp16_16k", 0.5, 0), ("vlp16_16k", 1.0, 6), ("vlp16", 0.7, 0)])
@pytest.mark.parametrize("flag", [0, 1])
def test_align_matches_reference(ref, synth, sensor, res, fixed, flag):
    tgt, src = synth.scan(sensor, frame=0, stride=8), synth.scan(sensor, frame=1, stride=8)
    M = ref.map(tgt, res)
    r = handle(kd_cfg(res, flag, fixed), tgt, src)
    for seed in (None, 3):
        G = (np.eye(4) if seed is None else perturb(seed, 0.2, 1.0)).astype(np.float32)
        r.align(G)
        o = M.align(src, G, mt_interval_flag=flag, fixed_iterations=fixed)
        T = r.getFinalTransformation()
        assert r.hasConverged() == o["converged"] and r.nr_iterations == o["iterations"], (r.nr_iterations, o)
        assert trans_err(T, o["T"]) < 1e-4 and rot_err(T, o["T"]) < 1e-4
        if fixed:
            assert r.nr_iterations == fixed
        fit = r.getFitnessScore(MAXR)
        want = orc.fitness(tgt, src, T, MAXR)[0]
        assert abs(fit - want) <= 1e-12 * abs(want)
        al = r.getAligned() if hasattr(r, "getAligned") else None
        if al is not None and al.size:
            x = src[:, :3].astype(np.float64) @ T[:3, :3].T.astype(np.float64) + T[:3, 3]
            assert np.max(np.abs(al[:, :3] - x)) <= 1e-3
    r.close()


def _same(a, b, fitness=True):
    ok = np.array_equal(np.asarray(a["T"]).view(np.uint32), np.asarray(b["T"]).view(np.uint32))
    ok = ok and bool(a["converged"]) == bool(b["converged"]) and a["iterations"] == b["iterations"]
    if fitness:
        ok = ok and np.float64(a["fitness"]).tobytes() == np.float64(b["fitness"]).tobytes()
    return ok


def _pairs(synth):
    clouds, pairs = {}, []
    for gi, tf in enumerate((0, 10)):
        clouds.setdefault(tf, synth.scan("vlp16_16k", frame=tf, stride=8))
        for j, off in enumerate((1, 251, 2, 252)):
            sf = tf + off
            clouds.setdefault(sf, synth.scan("vlp16_16k", frame=sf, stride=8))
            g = (np.linalg.inv(synth.pose_matrix(tf)) @ synth.pose_matrix(sf) @ perturb(60 + 7 * gi + j, 0.3, 2.0)).astype(np.float32)
            g[2, 3] = 0.0
            pairs.append((sf, tf, g))
    return clouds, pairs


def _single(cfg, clouds, pairs):
    r = pkg.Registration(cfg)
    out = []
    for s, t, g in pairs:
        r.setInputTarget(clouds[t])
        r.setInputSource(clouds[s])
        r.align(g)
        out.append({"T": r.getFinalTransformation(), "converged": r.hasConverged(), "iterations": r.nr_iterations, "fitness": r.getFitnessScore(MAXR)})
    r.close()
    return out


@pytest.mark.parametrize("flag", [0, 1])
@pytest.mark.parametrize("alone", [False, True])
def test_batch_loop_matching_and_fitness_equal_single_handle(synth, flag, alone):
    cfg = kd_cfg(1.0, flag)
    clouds, pairs = _pairs(synth)
    want = _single(cfg, clouds, pairs)
    lb = pkg.RegistrationBatch(cfg=cfg)
    ids = {k: lb.addCloud(c) for k, c in clouds.items()}
    pl = [(ids[s], ids[t], g) for s, t, g in pairs]
    got = [lb.align([p], True, MAXR)[0] for p in pl] if alone else lb.align(pl, True, MAXR)
    for i, (a, b) in enumerate(zip(got, want)):
        assert _same(a, b), f"pair {i}"
    best, det = lb.loopDetect(pl, [0, 4, 8], MAXR, 0.5)
    for a, d in zip(got, det):
        assert _same(a, d)
    scores = lb.calcFitnessScore([(ids[t], ids[s], w["T"]) for (s, t, _), w in zip(pairs, want)], MAXR)
    for sc, w in zip(scores, want):
        assert np.float64(sc).tobytes() == np.float64(w["fitness"]).tobytes()
    lb.close()
    reg = pkg.Registration(cfg)
    det = pkg.LoopDetector(reg, fitness_score_max_range=MAXR, fitness_score_thresh=0.5)
    grp = [p for p in pairs if p[1] == 0]
    best, rs = det.matching([clouds[s] for s, _, _ in grp], clouds[0], [g for _, _, g in grp])
    reg.close()
    for a, b in zip(rs, want[:len(grp)]):
        assert _same(a, b)


def test_target_nearest_and_prefetch_promotion_equal_a_fresh_handle(synth):
    frames = [synth.scan("vlp16_16k", frame=k, stride=8, step=0.1) for k in range(4)]
    cfg = kd_cfg(1.0)
    a = pkg.Registration(cfg)
    a.setInputTarget(frames[0])
    a.setInputSource(frames[1])
    a.prefetchSource(frames[2])
    a.align(np.eye(4, dtype=np.float32))
    Ta = a.getFinalTransformation()
    nn_a = a.nearestKSearch(frames[3][:500])
    a.promoteSourceToTarget()
    a.setInputSource(frames[2])
    a.align(np.eye(4, dtype=np.float32))
    Tb = a.getFinalTransformation()
    a.close()
    for t, s, T in ((frames[0], frames[1], Ta), (frames[1], frames[2], Tb)):
        r = handle(cfg, t, s)
        r.align(np.eye(4, dtype=np.float32))
        assert np.array_equal(r.getFinalTransformation().view(np.uint32), T.view(np.uint32))
        if t is frames[0]:
            nn = r.nearestKSearch(frames[3][:500])
            for x, y in zip(nn_a if isinstance(nn_a, tuple) else (nn_a,), nn if isinstance(nn, tuple) else (nn,)):
                assert np.array_equal(np.asarray(x), np.asarray(y))
        r.close()


@pytest.mark.parametrize("prefetch", [False, True])
@pytest.mark.parametrize("ds", ["none", "voxelgrid"])
def test_odometry_mirror_equals_host_loop(synth, prefetch, ds):
    frames = [synth.scan("vlp16_16k", frame=k, stride=8, step=0.1) for k in range(8)]
    cfg = kd_cfg(1.0)
    dsm = pkg.B2R_DOWNSAMPLE_NONE if ds == "none" else pkg.B2R_DOWNSAMPLE_VOXELGRID
    reg = pkg.Registration(cfg)
    odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=0.005, keyframe_delta_angle=1.0, keyframe_delta_time=10000.0, downsample_method=dsm,
                                   downsample_resolution=0.3)
    sts = []
    for k, c in enumerate(frames):
        if prefetch and k + 1 < len(frames):
            odo.prefetch_raw(frames[k + 1].ctypes.data, frames[k + 1].shape[0], frames[k + 1].shape[1] * 4)
        sts.append(odo.matching(0.1 * k, c))
    odo.close()
    reg.close()
    r = pkg.Registration(cfg)
    fr = frames if ds == "none" else [r.voxelGridFilter(c, 0.3) for c in frames]
    keyframe, prev, switches = fr[0], np.eye(4, dtype=np.float32), 0
    for k in range(1, len(frames)):
        r.setInputTarget(keyframe)
        r.setInputSource(fr[k])
        r.align(prev)
        T = r.getFinalTransformation()
        assert np.array_equal(T.view(np.uint32), np.asarray(sts[k]["trans"], np.float32).view(np.uint32)), f"frame {k}"
        assert sts[k]["converged"] == r.hasConverged() and sts[k]["iterations"] == r.nr_iterations
        prev = T
        if sts[k]["keyframe_updated"]:
            keyframe, prev = fr[k], np.eye(4, dtype=np.float32)
            switches += 1
    assert switches >= 1
    r.close()


def test_taps_refuse_other_engines(synth):
    tgt, src = synth.scan("vlp16_16k", frame=0, stride=8), synth.scan("vlp16_16k", frame=1, stride=8)
    for m in (pkg.B2R_METHOD_NDT, pkg.B2R_METHOD_GICP):
        r = handle(kd_cfg(1.0, method=m), tgt, src)
        for tap in (lambda: r.ndtGetCentroids(), lambda: r.ndtNeighborsAt(np.zeros(6), src.shape[0])):
            with pytest.raises(pkg.B2RError) as e:
                tap()
            assert e.value.code == _capi.B2R_ESTATE
        r.close()
