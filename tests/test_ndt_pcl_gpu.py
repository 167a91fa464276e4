"""GPU: the factory's `NDT` branch (pcl::NormalDistributionsTransform, B2R_METHOD_NDT_PCL; registrations.cpp:93-100) against the
sequential CPU reference tests/ndt_pcl_ref.cpp: centroids and radius neighbour lists bit for bit, derivative / Hessian passes to
1e-9, aligns to 1e-4 with the same iteration count and flag; and the single handle, the batch, the loop matcher and the odometry
mirror agree bitwise."""
import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi
from common import rot_err, trans_err, perturb
from ndt_pcl_ref import Reference, room, outside_scene

pytestmark = pytest.mark.gpu

MAXR = 2.5
POSES = [np.zeros(6), np.array([0.1, -0.05, 0.02, 0.01, -0.02, 0.03]), np.array([0.4, 0.3, -0.1, 0.2, -0.1, 0.6]),
         np.array([-0.7, 1.2, 0.05, 0.05, 0.03, 2.8])]  # the last: a large rotation


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("ndt_pcl_ref"))


def pcl_cfg(res=1.0, flag=0, fixed=0, max_iterations=64):
    c = pkg.default_config(pkg.B2R_METHOD_NDT_PCL)
    c.ndt_resolution = res
    c.ndt_mt_interval_flag = flag
    c.ndt_fixed_iterations = fixed
    c.max_iterations = max_iterations
    return c


def handle(cfg, tgt, src):
    r = pkg.Registration(cfg)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    return r


def rel(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


def test_factory_ndt_branch():
    r = pkg.select_registration_method({"registration_method": "NDT"})
    c = r.config
    assert c.method == pkg.B2R_METHOD_NDT_PCL == 2
    assert (c.ndt_resolution, c.transformation_epsilon, c.max_iterations, c.ndt_step_size, c.ndt_outlier_ratio) == (0.5, 0.01, 64, 0.1, 0.55)
    r.close()
    r = pkg.select_registration_method({"registration_method": "NDT", "reg_resolution": 1.0, "reg_transformation_epsilon": 0.02,
                                        "reg_maximum_iterations": 30, "reg_nn_search_method": "KDTREE"})  # the branch does not read it
    c = r.config
    assert (c.method, c.ndt_resolution, c.transformation_epsilon, c.max_iterations) == (2, 1.0, 0.02, 30)
    r.close()
    with pytest.raises(pkg.B2RError) as e:
        pkg.select_registration_method({"registration_method": "NDT_FOO"})
    assert e.value.code == _capi.B2R_EUNSUPPORTED


@pytest.mark.parametrize("scene", ["room", "hdl32e", "outside"])
def test_centroids_neighbours_and_passes(ref, synth, scene):
    if scene == "room":
        tgt, src, res = room(20000, 1), room(16000, 2), 0.5
    elif scene == "outside":  # a voxel whose float32 centroid lies in the next cell, and queries all around it
        tgt, src, _ = outside_scene(0.1)
        res = 0.1
    else:
        tgt, src, res = synth.scan("hdl32e", frame=0, stride=8), synth.scan("hdl32e", frame=1, stride=8), 1.0
    M = ref.map(tgt, res)
    r = handle(pcl_cfg(res), tgt, src)
    k, c = r.ndtGetCentroids()
    rk, rc = M.centroids()
    assert k.size > 100 and np.array_equal(k, rk) and np.array_equal(c.view(np.uint32), rc.view(np.uint32))
    v = r.ndtGetVoxels()
    assert np.array_equal(v["keys"], M.voxels["keys"]) and np.array_equal(v["npts"], M.voxels["npts"])
    for p in POSES:
        cnt, keys = r.ndtNeighborsAt(p, src.shape[0])
        rcnt, rkeys = M.neighbors(src, p)
        assert np.array_equal(cnt, rcnt) and np.array_equal(keys, rkeys), f"neighbours at {p}"
        s, g, H, npairs = r.ndtDerivativesAt(p)
        o = M.derivatives(src, p)
        assert npairs == o["n_pairs"] == keys.size
        if npairs:
            assert abs(s - o["score"]) <= 1e-9 * abs(o["score"])
            assert rel(g, o["g"]) <= 1e-9 and rel(H, o["H"]) <= 1e-9
            assert np.array_equal(r.ndtHessianAt(p), H)  # computeHessian's term is updateDerivatives' Hessian term
        again = r.ndtDerivativesAt(p)
        assert again[0] == s and np.array_equal(again[1], g) and np.array_equal(again[2], H) and again[3] == npairs
    r.close()


@pytest.mark.parametrize("sensor,res,fixed", [("vlp16_16k", 1.0, 0), ("vlp16_16k", 0.5, 0), ("vlp16_16k", 1.0, 6), ("hdl32e", 1.0, 5)])
@pytest.mark.parametrize("flag", [0, 1])
def test_align_matches_reference(ref, synth, sensor, res, fixed, flag):
    tgt, src = synth.scan(sensor, frame=0, stride=8), synth.scan(sensor, frame=1, stride=8)
    M = ref.map(tgt, res)
    r = handle(pcl_cfg(res, flag, fixed), tgt, src)
    for seed in (None, 3):
        G = (np.eye(4) if seed is None else perturb(seed, 0.2, 1.0)).astype(np.float32)
        r.align(G)
        o = M.align(src, G, mt_interval_flag=flag, fixed_iterations=fixed)
        T = r.getFinalTransformation()
        assert r.hasConverged() == o["converged"] and r.nr_iterations == o["iterations"], (r.nr_iterations, o)
        assert trans_err(T, o["T"]) < 1e-4 and rot_err(T, o["T"]) < 1e-4
        if fixed:
            assert r.nr_iterations == fixed
    r.close()


def test_edge_cases(ref, synth):
    tgt, src = synth.scan("vlp16_16k", frame=0, stride=8), synth.scan("vlp16_16k", frame=1, stride=8)
    odd = src.copy()
    odd[::7, :3] = np.nan
    odd[3::11, 0] = 1e12
    odd[5::13, 2] = -1e12
    cases = {"empty": np.zeros((0, 8), np.float32), "all_nan": np.full((64, 8), np.nan, np.float32), "sparse": tgt[:5].copy()}
    for name, t in cases.items():
        r = handle(pcl_cfg(1.0), t, src) if t.shape[0] else pkg.Registration(pcl_cfg(1.0))
        if not t.shape[0]:
            r.setInputSource(src)
            r.setInputTarget(t)
        r.align(np.eye(4, dtype=np.float32))
        assert not r.hasConverged() or name == "sparse", name
        if name != "empty":
            k, _ = r.ndtGetCentroids()
            assert k.size == 0, name
            cnt, keys = r.ndtNeighborsAt(POSES[1], src.shape[0])
            assert cnt.sum() == 0 and keys.size == 0
        r.close()
    M = ref.map(tgt, 1.0)
    r = handle(pcl_cfg(1.0), tgt, odd)
    for p in POSES[:3]:
        cnt, keys = r.ndtNeighborsAt(p, odd.shape[0])
        rcnt, rkeys = M.neighbors(odd, p)
        assert np.array_equal(cnt, rcnt) and np.array_equal(keys, rkeys)
        assert cnt[::7].sum() == 0 and cnt[3::11].sum() == 0
        s, g, H, npairs = r.ndtDerivativesAt(p)
        o = M.derivatives(odd, p)
        assert npairs == o["n_pairs"] and abs(s - o["score"]) <= 1e-9 * abs(o["score"]) and rel(H, o["H"]) <= 1e-9
    r.align(np.eye(4, dtype=np.float32))
    o = M.align(odd)
    assert r.nr_iterations == o["iterations"] and trans_err(r.getFinalTransformation(), o["T"]) < 1e-4
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
def test_batch_and_loop_matching_equal_single_handle(synth, flag):
    cfg = pcl_cfg(1.0, flag)
    clouds, pairs = _pairs(synth)
    want = _single(cfg, clouds, pairs)
    lb = pkg.RegistrationBatch(cfg=cfg)
    ids = {k: lb.addCloud(c) for k, c in clouds.items()}
    got = lb.align([(ids[s], ids[t], g) for s, t, g in pairs], True, MAXR)
    rounds, pair_rounds = lb.lastRounds()
    lb.close()
    assert rounds >= 2
    for i, (a, b) in enumerate(zip(got, want)):
        assert _same(a, b), f"pair {i}"
    reg = pkg.Registration(cfg)
    det = pkg.LoopDetector(reg, fitness_score_max_range=MAXR, fitness_score_thresh=0.5)
    grp = [p for p in pairs if p[1] == 0]
    best, rs = det.matching([clouds[s] for s, _, _ in grp], clouds[0], [g for _, _, g in grp])
    reg.close()
    for a, b in zip(rs, want[:len(grp)]):
        assert _same(a, b)


def test_odometry_mirror_equals_host_loop(synth):
    frames = [synth.scan("vlp16_16k", frame=k, stride=8, step=0.1) for k in range(10)]
    cfg = pcl_cfg(1.0)
    reg = pkg.Registration(cfg)
    odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=0.005, keyframe_delta_angle=1.0, keyframe_delta_time=10000.0)
    sts = []
    for k, c in enumerate(frames):
        if k + 1 < len(frames):
            odo.prefetch_raw(frames[k + 1].ctypes.data, frames[k + 1].shape[0], frames[k + 1].shape[1] * 4)
        sts.append(odo.matching(0.1 * k, c))
    odo.close()
    reg.close()
    r = pkg.Registration(cfg)
    keyframe, prev, switches = frames[0], np.eye(4, dtype=np.float32), 0
    for k in range(1, len(frames)):
        r.setInputTarget(keyframe)
        r.setInputSource(frames[k])
        r.align(prev)
        T = r.getFinalTransformation()
        assert np.array_equal(T.view(np.uint32), np.asarray(sts[k]["trans"], np.float32).view(np.uint32)), f"frame {k}"
        assert sts[k]["converged"] == r.hasConverged() and sts[k]["iterations"] == r.nr_iterations
        prev = T
        if sts[k]["keyframe_updated"]:
            assert np.linalg.norm(T[:3, 3]) > 0.005 or not r.hasConverged()
            keyframe, prev = frames[k], np.eye(4, dtype=np.float32)
            switches += 1
    assert switches >= 1
    r.close()
