"""GPU: the pcl ICP engine (B2R_METHOD_ICP_PCL, pcl::IterativeClosestPoint) against the sequential reference tests/icp_pcl_ref.cpp, and
every entry point against the single handle.  Correspondences and d2 are bit-exact; the estimation's sums within rel 1e-12 and its
transformation within 1e-5; aligns have the reference's iterations and flag and a pose within 1e-5; fitness is the oracle's."""
import numpy as np
import pytest

import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi
import icp_pcl_ref as ir
from gicp_pcl_ref import pose, scene, transform
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return ir.Reference(tmp_path_factory.mktemp("icp_pcl_ref"))


def handle(**extra):
    p = {"registration_method": "B200_ICP"}
    p.update({k: str(v).lower() if isinstance(v, bool) else str(v) for k, v in extra.items()})
    return pkg.select_registration_method(p)


def about(T, offset):
    C = np.eye(4)
    C[:3, 3] = offset
    return (C @ np.asarray(T, np.float64) @ np.linalg.inv(C)).astype(np.float32)


def pair(n, seed=0, offset=(0.0, 0.0, 0.0), T=None):
    tgt = scene(n, seed=seed, offset=offset)
    src = transform(scene(n, seed=seed + 1, offset=offset), about(pose((0.3, -0.2, 0.05), (0.01, -0.01, 0.05)), offset) if T is None else T)
    return tgt, src


def ready(tgt, src, **extra):
    r = handle(**extra)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    return r


def test_factory_mapping_and_parameters():
    r = handle()
    c = r.config
    assert c.method == pkg.B2R_METHOD_ICP_PCL
    assert (c.max_iterations, c.transformation_epsilon, c.max_correspondence_distance, c.use_reciprocal_correspondences) == (64, 0.01, 2.5, 0)
    r.close()
    for v, want in (("true", 1), ("false", 0), ("1", 1), ("0", 0)):
        r = handle(reg_transformation_epsilon=0.05, reg_maximum_iterations=7, reg_max_correspondence_distance=1.5, reg_use_reciprocal_correspondences=v)
        c = r.config
        assert (c.transformation_epsilon, c.max_iterations, c.max_correspondence_distance, c.use_reciprocal_correspondences) == (0.05, 7, 1.5, want)
        r.close()
    with pytest.raises(pkg.B2RError) as e:
        handle(reg_use_reciprocal_correspondences="yes")
    assert e.value.code == _capi.B2R_EINVAL
    with pytest.raises(pkg.B2RError) as e:  # the plain name keeps the reference's own branch
        pkg.select_registration_method({"registration_method": "ICP"})
    assert e.value.code == _capi.B2R_EUNSUPPORTED
    cfg = pkg.registration.default_config(pkg.B2R_METHOD_ICP_PCL)
    cfg.use_reciprocal_correspondences = 2
    with pytest.raises(pkg.B2RError) as e:
        pkg.Registration(cfg)
    assert e.value.code == _capi.B2R_EINVAL


@pytest.mark.parametrize("reciprocal", [False, True])
@pytest.mark.parametrize("n,offset", [(16384, (0, 0, 0)), (65536, (0, 0, 0)), (16384, (3000.0, -2000.0, 50.0))])
def test_correspondences_and_estimate_match_the_reference(ref, n, offset, reciprocal):
    tgt, src = pair(n, seed=1 + n % 7, offset=offset)
    r = ready(tgt, src, reg_use_reciprocal_correspondences=reciprocal)
    for T in (np.eye(4, dtype=np.float32), about(pose((-0.2, 0.1, 0.01), (0.002, -0.003, 0.02)), offset)):
        corr, d2, cnt = r.icpPclCorrespondencesAt(T, src.shape[0])
        wc, wd, wcnt = ref.correspondences(src, tgt, T, 2.5, reciprocal)
        assert cnt == wcnt and np.array_equal(corr, wc) and cnt > 1000
        ok = corr >= 0
        assert np.array_equal(d2[ok].view(np.uint32), wd[ok].view(np.uint32)) and np.isnan(d2[~ok]).all()
        Rt, sums = r.icpPclEstimateAt(T)
        wRt, wsums, _ = ref.estimate(src, tgt, T, 2.5, reciprocal)
        assert np.max(np.abs(sums - wsums) / np.maximum(np.abs(wsums), 1e-12 * np.max(np.abs(wsums)))) <= 1e-12
        assert np.max(np.abs(Rt - wRt)) <= 1e-5
    r.close()


@pytest.mark.parametrize("case", ["16k", "64k", "far", "reciprocal", "reciprocal_far", "tight_epsilon", "tight_epsilon_reciprocal", "guess"])
def test_align_matches_the_reference(ref, case):
    n = 65536 if case == "64k" else 16384
    offset = (3000.0, -2000.0, 50.0) if "far" in case else (0, 0, 0)
    T_true = about(pose((0.4, -0.3, 0.05), (0.01, 0.0, 0.06)), offset)
    tgt, src = pair(n, seed=3, offset=offset, T=T_true)
    reciprocal = "reciprocal" in case
    eps = 1e-6 if "tight" in case else 0.01
    r = ready(tgt, src, reg_use_reciprocal_correspondences=reciprocal, reg_transformation_epsilon=eps)
    guess = (pose((0.05, 0.02, 0.0), (0.0, 0.0, 0.01)) @ np.linalg.inv(T_true)).astype(np.float32) if case == "guess" else np.eye(4, dtype=np.float32)
    r.getStats(reset=True)
    r.align(guess)
    st = r.getStats()
    T, conv, it = r.getFinalTransformation(), r.hasConverged(), r.nr_iterations
    w = ref.align(src, tgt, guess, transformation_epsilon=eps, reciprocal=reciprocal)
    assert (conv, it) == (w["converged"], w["iterations"]) and conv and it >= 1
    assert np.max(np.abs(T - w["T"])) <= 1e-5
    if "tight" in case:
        assert it >= 10
    # rounds on the device: at most 2 launches per iteration, 4 with the reciprocal check, and no covariance work
    per_round = 4 if reciprocal else 2
    assert st["launches"]["icp_pcl_round"] % per_round == 0 and st["launches"]["icp_pcl_round"] >= per_round * it
    assert st["launches"]["knn_covariance"] == 0
    assert np.max(np.abs(r.getAligned()[:, :3] - transform(src, T)[:, :3])) <= 1e-3
    s = r.getFitnessScore()
    want = orc.fitness(tgt, src, T)[0]
    assert abs(s - want) <= 1e-12 * abs(want)
    r.close()


def test_too_few_correspondences_end_unconverged(ref):
    tgt, src = pair(16384, seed=4)
    far = pose((500.0, 0.0, 0.0))
    r = ready(tgt, src)
    r.align(far)
    w = ref.align(src, tgt, far)
    assert (r.hasConverged(), r.nr_iterations) == (False, 0) == (w["converged"], w["iterations"])
    assert np.array_equal(r.getFinalTransformation(), far)
    with pytest.raises(pkg.B2RError) as e:
        r.icpPclEstimateAt(far)
    assert e.value.code == _capi.B2R_ESTATE
    r.close()


def clouds_for(k, n=16384, seed=20):
    return [transform(scene(n, seed=seed + i), pose((0.15 * i, -0.05 * i, 0.0), (0.0, 0.0, 0.015 * i))) for i in range(k)]


@pytest.mark.parametrize("reciprocal", [False, True])
def test_entry_points_agree_bit_for_bit(reciprocal):
    clouds = clouds_for(5)
    guesses = [np.eye(4, dtype=np.float32), pose((0.1, 0.0, 0.0)), pose((0.0, -0.1, 0.0), (0, 0, 0.01)), pose((0.05, 0.05, 0.0))]
    r = handle(reg_use_reciprocal_correspondences=reciprocal)
    single = []
    for i, g in enumerate(guesses):
        r.setInputTarget(clouds[0])
        r.setInputSource(clouds[1 + i])
        r.align(g)
        single.append((r.getFinalTransformation(), r.hasConverged(), r.nr_iterations, r.getFitnessScore(2.5), r.getFitnessScore()))
    best, res = pkg.LoopDetector(r).matching(clouds[1:], clouds[0], guesses)
    for (T, conv, it, _, fit), x in zip(single, res):
        assert np.array_equal(T, x["T"]) and conv == x["converged"] and it == x["iterations"] and fit == x["fitness"]
    r.close()
    params = {"registration_method": "B200_ICP", "reg_use_reciprocal_correspondences": str(reciprocal).lower()}
    lb = pkg.RegistrationBatch(params=params)
    ids = [lb.addCloud(c) for c in clouds]
    pairs = [(ids[1 + i], ids[0], g) for i, g in enumerate(guesses)]
    res = lb.align(pairs, True, 2.5)
    for (T, conv, it, fit, _), x in zip(single, res):
        assert np.array_equal(T, x["T"]) and conv == x["converged"] and it == x["iterations"] and fit == x["fitness"]
    # co-scheduled with other pairs, and alone
    res2 = lb.align(pairs[2:3], True, 2.5)
    assert np.array_equal(res2[0]["T"], res[2]["T"]) and res2[0]["iterations"] == res[2]["iterations"]
    best, det = lb.loopDetect(pairs, [0, 2, 4], 2.5, 0.5)
    for a, d in zip(res, det):
        assert np.array_equal(a["T"], d["T"]) and a["fitness"] == d["fitness"] and a["converged"] == d["converged"]
    for g, (g0, g1) in enumerate(((0, 2), (2, 4))):
        conv = [(res[i]["fitness"], i - g0) for i in range(g0, g1) if res[i]["converged"]]
        want = -1
        if conv:
            bs = min(f for f, _ in conv)
            want = max(i for f, i in conv if f == bs) if bs <= 0.5 else -1
        assert best[g] == want
    scores = lb.calcFitnessScore([(ids[0], ids[1 + i], single[i][0]) for i in range(len(guesses))], 2.5)
    for s, sc in zip(single, scores):
        assert sc == s[3]
    lb.close()


@pytest.mark.parametrize("prefetch", [False, True])
@pytest.mark.parametrize("downsample", [_capi.B2R_DOWNSAMPLE_NONE, _capi.B2R_DOWNSAMPLE_VOXELGRID])
def test_odometry_mirror_equals_a_host_loop(prefetch, downsample):
    """frame k against frame k - 1 (every frame a keyframe at zero thresholds), identity motion guess: the mirror's trans is the single
    handle's align on the same (downsampled) clouds"""
    clouds = clouds_for(5, seed=40)
    o = pkg.ScanMatchingOdometry(handle(), keyframe_delta_trans=0.0, keyframe_delta_angle=0.0, keyframe_delta_time=0.0, downsample_method=downsample,
                                 downsample_resolution=0.2)
    h2 = handle()
    vg = handle()
    filt = (lambda c: vg.voxelGridFilter(c, 0.2)) if downsample == _capi.B2R_DOWNSAMPLE_VOXELGRID else (lambda c: c)
    o.matching(0.0, clouds[0])
    for k in range(1, 5):
        if prefetch and k + 1 < 5:
            o.prefetch_raw(clouds[k + 1].ctypes.data, clouds[k + 1].shape[0], 16)
        st = o.matching(0.1 * k, clouds[k])
        h2.setInputTarget(filt(clouds[k - 1]))
        h2.setInputSource(filt(clouds[k]))
        h2.align(np.eye(4, dtype=np.float32))
        assert np.array_equal(st["trans"], h2.getFinalTransformation()) and st["converged"] == h2.hasConverged() and st["iterations"] == h2.nr_iterations
    o.close()
    h2.close()
    vg.close()


def test_taps_refuse_other_engines_and_method_taps_refuse_this_one():
    tgt, src = pair(4096, seed=6)
    r = ready(tgt, src)
    T = np.eye(4)
    for call in (lambda: r.gicpLinearizeAt(T), lambda: r.gicpErrorAt(T), lambda: r.gicpPclCorrespondencesAt(T, T, src.shape[0]),
                 lambda: r.gicpPclCostAt(T), lambda: r.getCovariances(0, src.shape[0]), lambda: r.getCovariances(1, tgt.shape[0]),
                 lambda: r.getCorrespondences(src.shape[0])):
        with pytest.raises(pkg.B2RError) as e:
            call()
        assert e.value.code == _capi.B2R_ESTATE
    r.align(T)
    with pytest.raises(pkg.B2RError) as e:
        r.getCorrespondences(src.shape[0])
    assert e.value.code == _capi.B2R_ESTATE
    r.close()
    g = pkg.select_registration_method({"registration_method": "GICP"})
    g.setInputTarget(tgt)
    g.setInputSource(src)
    for call in (lambda: g.icpPclCorrespondencesAt(T, src.shape[0]), lambda: g.icpPclEstimateAt(T)):
        with pytest.raises(pkg.B2RError) as e:
            call()
        assert e.value.code == _capi.B2R_ESTATE
    g.close()
