"""GPU: the factory's GICP branch (B2R_METHOD_GICP_PCL, pcl::GeneralizedIterativeClosestPoint) against the sequential reference
tests/gicp_pcl_ref.cpp, and every entry point against the single handle.  Correspondences are bit-exact; covariances within 1e-8 abs;
M within rel 1e-12; cost-pass sums within rel 1e-9; aligns have the reference's outer iterations, correspondence passes and flag, a
pose within 1e-5 and the same number of cost passes up to the line search's order-sensitive comparisons; fitness is the oracle's within rel 1e-12."""
import numpy as np
import pytest

import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi
import gicp_pcl_ref as gr
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return gr.Reference(tmp_path_factory.mktemp("gicp_pcl_ref"))


def handle(**extra):
    p = {"registration_method": "GICP"}
    p.update({k: str(v) for k, v in extra.items()})
    return pkg.select_registration_method(p)


def pair(n, seed=0, offset=(0.0, 0.0, 0.0), T=None):
    tgt = gr.scene(n, seed=seed, offset=offset)
    src = gr.transform(gr.scene(n, seed=seed + 1, offset=offset), gr.pose((0.3, -0.2, 0.05), (0.01, -0.01, 0.05)) if T is None else T)
    return tgt, src


def about(T, offset):
    """T acting about the point `offset` instead of the origin (so a far scene moves as little as one at the origin)"""
    C = np.eye(4)
    C[:3, 3] = offset
    return (C @ np.asarray(T, np.float64) @ np.linalg.inv(C)).astype(np.float32)


def ready(tgt, src, **extra):
    r = handle(**extra)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    return r, r.getCovariances(0, src.shape[0]), r.getCovariances(1, tgt.shape[0])


def rel(a, b):
    return np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300))


def test_factory_mapping_and_refused_names():
    for name in ("GICP", "B200_GICP_PCL", "PCL_GICP"):
        r = pkg.select_registration_method({"registration_method": name})
        c = r.config
        assert c.method == pkg.B2R_METHOD_GICP_PCL
        assert (c.max_iterations, c.k_correspondences, c.max_optimizer_iterations, c.transformation_epsilon, c.rotation_epsilon,
                c.max_correspondence_distance) == (64, 20, 20, 0.01, 2e-3, 2.5)
        r.close()
    r = handle(reg_transformation_epsilon=0.05, reg_maximum_iterations=7, reg_max_correspondence_distance=1.5, reg_correspondence_randomness=12,
               reg_max_optimizer_iterations=3, reg_use_reciprocal_correspondences="true", reg_resolution=4.0)
    c = r.config
    assert (c.transformation_epsilon, c.max_iterations, c.max_correspondence_distance, c.k_correspondences, c.max_optimizer_iterations) == (
        0.05, 7, 1.5, 12, 3)
    r.close()
    assert pkg.select_registration_method({"registration_method": "B200_GICP"}).config.method == pkg.B2R_METHOD_GICP
    assert pkg.select_registration_method({"registration_method": "FAST_VGICP"}).config.method == pkg.B2R_METHOD_VGICP
    for name in ("GICP_OMP", "ICP", "FAST_VGICP_CUDA"):
        with pytest.raises(pkg.B2RError):
            pkg.select_registration_method({"registration_method": name})
    with pytest.raises(pkg.B2RError):
        pkg.select_registration_method({"registration_method": "NDT_OMP", "reg_nn_search_method": "KDTREE"})


@pytest.mark.parametrize("n,offset", [(16384, (0, 0, 0)), (65536, (0, 0, 0)), (16384, (3000.0, -2000.0, 50.0))])
def test_covariances_match_the_reference(ref, n, offset):
    tgt, src = pair(n, seed=n % 5, offset=offset)
    r, scov, tcov = ready(tgt, src)
    assert np.max(np.abs(scov - ref.covariances(src))) <= 1e-8
    assert np.max(np.abs(tcov - ref.covariances(tgt))) <= 1e-8
    r.close()


@pytest.mark.parametrize("n,offset", [(16384, (0, 0, 0)), (65536, (0, 0, 0)), (16384, (3000.0, -2000.0, 50.0))])
def test_correspondences_and_cost_match_the_reference(ref, n, offset):
    tgt, src = pair(n, seed=1 + n % 7, offset=offset, T=about(gr.pose((0.3, -0.2, 0.05), (0.01, -0.01, 0.05)), offset))
    r, scov, tcov = ready(tgt, src)
    guess = about(gr.pose((0.1, 0.05, 0.0), (0.0, 0.0, -0.03)), offset)
    for T_rel in (np.eye(4, dtype=np.float32), about(gr.pose((-0.2, 0.1, 0.01), (0.002, -0.003, 0.02)), offset)):
        corr, M, cnt = r.gicpPclCorrespondencesAt(guess, T_rel, src.shape[0])
        wcorr, wM, wcnt = ref.correspondences(src, tgt, guess, T_rel, scov=scov, tcov=tcov)
        assert cnt == wcnt and np.array_equal(corr, wcorr)
        ok = corr >= 0
        assert ok.sum() > 1000
        assert rel(M[ok], wM[ok]) <= 1e-12 and np.isnan(M[~ok]).all()
        for T in (T_rel, about(gr.pose((-0.15, 0.12, 0.0), (0.001, 0.0, 0.025)), offset)):
            f, g, dR = r.gicpPclCostAt(T)
            want, _ = ref.cost(src, tgt, guess, T_rel, T, scov=scov, tcov=tcov)
            got = np.r_[f, g, dR.reshape(-1)]
            assert np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-12 * np.max(np.abs(want)))) <= 1e-9
    r.close()


def _align(r, guess):
    r.getStats(reset=True)
    r.align(guess)
    st = r.getStats()
    return r.getFinalTransformation(), r.hasConverged(), r.nr_iterations, st["launches"]["gicp_pcl_correspondences"], st["launches"]["gicp_pcl_cost"]


@pytest.mark.parametrize("case", ["16k", "64k", "large_rotation", "far", "one_inner_step"])
def test_align_matches_the_reference(ref, case):
    n = 65536 if case == "64k" else 16384
    offset = (3000.0, -2000.0, 50.0) if case == "far" else (0, 0, 0)
    T_true = gr.pose((0.4, -0.3, 0.05), (0.01, 0.0, 0.6 if case == "large_rotation" else 0.06))
    T_true = about(T_true, offset)
    tgt, src = pair(n, seed=3, offset=offset, T=T_true)
    extra = {"reg_max_optimizer_iterations": 1} if case == "one_inner_step" else {}
    r, scov, tcov = ready(tgt, src, **extra)
    guess = np.linalg.inv(T_true).astype(np.float32) if case == "large_rotation" else np.eye(4, dtype=np.float32)
    if case == "large_rotation":  # a guess near the answer from a rotation of 0.6 rad
        guess = (gr.pose((0.02, 0.01, 0.0), (0.0, 0.0, 0.01)) @ np.linalg.inv(T_true)).astype(np.float32)
    T, conv, it, ncorr, ncost = _align(r, guess)
    w = ref.align(src, tgt, guess, scov=scov, tcov=tcov, max_optimizer_iterations=1 if extra else 20)
    assert (conv, it, ncorr) == (w["converged"], w["iterations"], w["corr_passes"])
    # The cost passes are the reference's up to the line search's order-sensitive comparisons: near the minimum it compares f values
    # that agree to the last bits, and the engine's fixed-tree sums and the reference's index-order sums differ there.  On the
    # large-rotation case the engine takes 43 passes and the reference 41 (the reference alone takes 41 or 43 depending on which
    # covariances it is fed), with the same outer iterations, flag and pose.
    assert abs(ncost - w["cost_passes"]) <= max(2, w["cost_passes"] // 10)
    assert np.max(np.abs(T[:3, 3] - w["T"][:3, 3])) <= 1e-5 and np.max(np.abs(T[:3, :3] - w["T"][:3, :3])) <= 1e-5
    if case != "one_inner_step":
        assert conv and it >= 1
    # the aligned cloud and getFitnessScore at the final pose
    assert np.max(np.abs(r.getAligned()[:, :3] - gr.transform(src, T)[:, :3])) <= 1e-3
    s = r.getFitnessScore()
    want = orc.fitness(tgt, src, T)[0]
    assert abs(s - want) <= 1e-12 * abs(want)
    r.close()


def test_too_few_correspondences_end_unconverged(ref):
    tgt, src = pair(16384, seed=4)
    far = gr.pose((500.0, 0.0, 0.0))
    r, scov, tcov = ready(tgt, src)
    T, conv, it, ncorr, ncost = _align(r, far)
    w = ref.align(src, tgt, far, scov=scov, tcov=tcov)
    assert (conv, it, ncorr, ncost) == (False, 0, 1, 0) == (w["converged"], w["iterations"], w["corr_passes"], w["cost_passes"])
    assert np.array_equal(T, far)
    r.close()


def test_entry_points_agree_bit_for_bit():
    clouds = [gr.transform(gr.scene(16384, seed=10 + i), gr.pose((0.2 * i, 0.05 * i, 0.0), (0.0, 0.0, 0.02 * i))) for i in range(4)]
    guesses = [np.eye(4, dtype=np.float32), gr.pose((-0.1, 0.0, 0.0)), gr.pose((0.0, 0.1, 0.0), (0, 0, 0.01))]
    single = []
    r = handle()
    for i, g in enumerate(guesses):
        r.setInputTarget(clouds[0])
        r.setInputSource(clouds[1 + i])
        r.align(g)
        single.append((r.getFinalTransformation(), r.hasConverged(), r.nr_iterations, r.getFitnessScore()))
    best, res = pkg.LoopDetector(r).matching(clouds[1:], clouds[0], guesses)
    for (T, conv, it, fit), x in zip(single, res):
        assert np.array_equal(T, x["T"]) and conv == x["converged"] and it == x["iterations"] and fit == x["fitness"]
    r.close()
    # the odometry mirror: frame k against the keyframe, identity motion guess, every frame a keyframe at zero thresholds
    o = pkg.ScanMatchingOdometry(handle(), keyframe_delta_trans=0.0, keyframe_delta_angle=0.0, keyframe_delta_time=0.0)
    h2 = handle()
    o.matching(0.0, clouds[0])
    for k in range(1, 4):
        st = o.matching(0.1 * k, clouds[k])
        h2.setInputTarget(clouds[k - 1])
        h2.setInputSource(clouds[k])
        h2.align(np.eye(4, dtype=np.float32))
        assert np.array_equal(st["trans"], h2.getFinalTransformation()) and st["converged"] == h2.hasConverged()
    o.close()
    h2.close()


def test_batch_matches_the_single_handle_bit_for_bit():
    """b2r_batch_align (with fitness), b2r_batch_calc_fitness_score and the single-rank b2r_batch_loop_detect run every pair through the
    single handle's state machine, their passes batched per round: every record equals the single handle's"""
    clouds = [gr.transform(gr.scene(16384, seed=20 + i), gr.pose((0.15 * i, -0.05 * i, 0.0), (0.0, 0.0, 0.015 * i))) for i in range(5)]
    guesses = [np.eye(4, dtype=np.float32), gr.pose((0.1, 0.0, 0.0)), gr.pose((0.0, -0.1, 0.0), (0, 0, 0.01)), gr.pose((0.05, 0.05, 0.0))]
    r = handle()
    single = []
    for i, g in enumerate(guesses):
        r.setInputTarget(clouds[0])
        r.setInputSource(clouds[1 + i])
        r.align(g)
        single.append((r.getFinalTransformation(), r.hasConverged(), r.nr_iterations, r.getFitnessScore(2.5)))
    r.close()
    lb = pkg.RegistrationBatch(params={"registration_method": "GICP"})
    ids = [lb.addCloud(c) for c in clouds]
    pairs = [(ids[1 + i], ids[0], g) for i, g in enumerate(guesses)]
    res = lb.align(pairs, True, 2.5)
    for (T, conv, it, fit), x in zip(single, res):
        assert np.array_equal(T, x["T"]) and conv == x["converged"] and it == x["iterations"] and fit == x["fitness"]
    best, det = lb.loopDetect(pairs, [0, 2, 4], 2.5, 0.5)
    for a, d in zip(res, det):
        assert np.array_equal(a["T"], d["T"]) and a["fitness"] == d["fitness"] and a["converged"] == d["converged"]
    scores = lb.calcFitnessScore([(ids[0], ids[1 + i], single[i][0]) for i in range(len(guesses))], 2.5)  # (cloud1 = target, cloud2, relpose)
    for (T, _, _, fit), sc in zip(single, scores):
        assert sc == fit
    lb.close()


def test_taps_refuse_other_engines_and_linearize_refuses_this_one():
    tgt, src = pair(4096, seed=6)
    r, _, _ = ready(tgt, src)
    T = np.eye(4)
    with pytest.raises(pkg.B2RError) as e:
        r.gicpLinearizeAt(T)
    assert e.value.code == _capi.B2R_ESTATE
    with pytest.raises(pkg.B2RError) as e:
        r.gicpErrorAt(T)
    assert e.value.code == _capi.B2R_ESTATE
    with pytest.raises(pkg.B2RError) as e:
        r.gicpPclCostAt(T)  # no correspondence pass yet
    assert e.value.code == _capi.B2R_ESTATE
    r.close()
    g = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    g.setInputTarget(tgt)
    g.setInputSource(src)
    with pytest.raises(pkg.B2RError) as e:
        g.gicpPclCorrespondencesAt(T, T, src.shape[0])
    assert e.value.code == _capi.B2R_ESTATE
    g.close()
