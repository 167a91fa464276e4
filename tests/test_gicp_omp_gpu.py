"""GPU: the factory's GICP_OMP branch (B2R_METHOD_GICP_OMP, pclomp::GeneralizedIterativeClosestPoint, opted into as B200_GICP_OMP)
against the sequential reference tests/gicp_omp_ref.cpp, against a pcl GICP handle (the same align at an identity guess, a different one
with a translated guess), and every entry point against the single handle.  Correspondences are bit-exact; covariances within 1e-8 abs and M
within rel 1e-12 (as for pcl GICP); cost-pass sums within rel 1e-9; aligns have the reference's outer iterations, correspondence passes and flag and an end point as good
(gicp_pcl_ref.end_point_is_as_good); fitness is the oracle's within rel 1e-12."""
import ctypes as C

import numpy as np
import pytest

import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi
import gicp_omp_ref as gor
import gicp_pcl_ref as gr
from oracle import oracle as orc
from test_gicp_pcl_gpu import about, pair, rel

pytestmark = pytest.mark.gpu
OMP = "B200_GICP_OMP"


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return gor.Reference(tmp_path_factory.mktemp("gicp_omp_ref"))


def handle(method=OMP, **extra):
    p = {"registration_method": method}
    p.update({k: str(v) for k, v in extra.items()})
    return pkg.select_registration_method(p)


def ready(tgt, src, method=OMP, **extra):
    r = handle(method, **extra)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    return r, r.getCovariances(0, src.shape[0]), r.getCovariances(1, tgt.shape[0])


def test_factory_mapping_and_refused_names():
    r = handle()
    c = r.config
    assert c.method == pkg.B2R_METHOD_GICP_OMP == 8
    assert (c.max_iterations, c.k_correspondences, c.max_optimizer_iterations, c.transformation_epsilon, c.rotation_epsilon,
            c.max_correspondence_distance) == (64, 20, 20, 0.01, 2e-3, 2.5)
    r.close()
    r = handle(reg_transformation_epsilon=0.05, reg_maximum_iterations=7, reg_max_correspondence_distance=1.5, reg_correspondence_randomness=12,
               reg_max_optimizer_iterations=3, reg_use_reciprocal_correspondences="true", reg_num_threads=4)
    c = r.config
    assert (c.method, c.transformation_epsilon, c.max_iterations, c.max_correspondence_distance, c.k_correspondences, c.max_optimizer_iterations) == (
        pkg.B2R_METHOD_GICP_OMP, 0.05, 7, 1.5, 12, 3)
    r.close()
    with pytest.raises(pkg.B2RError) as e:
        handle(reg_max_optimizer_iterations=0)
    assert e.value.code == _capi.B2R_EINVAL
    for name in ("GICP_OMP", "FAST_GICP_OMP", "B200_GICP_OMP2"):
        with pytest.raises(pkg.B2RError) as e:
            pkg.select_registration_method({"registration_method": name})
        assert e.value.code == _capi.B2R_EUNSUPPORTED
    lib = pkg.load_library()
    cfg = _capi.Config()
    assert lib.b2r_config_default(C.byref(cfg), 7) == _capi.B2R_EINVAL
    assert lib.b2r_config_default(C.byref(cfg), pkg.B2R_METHOD_GICP_OMP) == _capi.B2R_OK


@pytest.mark.parametrize("n,offset", [(16384, (0, 0, 0)), (65536, (0, 0, 0)), (16384, (3000.0, -2000.0, 50.0))])
def test_covariances_correspondences_and_cost_match_the_reference(ref, n, offset):
    tgt, src = pair(n, seed=1 + n % 7, offset=offset, T=about(gr.pose((0.3, -0.2, 0.05), (0.01, -0.01, 0.05)), offset))
    r, scov, tcov = ready(tgt, src)
    assert np.max(np.abs(scov - ref.covariances(src))) <= 1e-8 and np.max(np.abs(tcov - ref.covariances(tgt))) <= 1e-8
    for guess in (about(gr.pose((0.1, 0.05, 0.0), (0.0, 0.0, -0.03)), offset), about(gr.pose((1.5, -1.0, 0.1), (0.0, 0.0, 0.01)), offset)):
        T_rel = about(gr.pose((-0.2, 0.1, 0.01), (0.002, -0.003, 0.02)), offset)
        corr, M, cnt = r.gicpPclCorrespondencesAt(guess, T_rel, src.shape[0])
        wcorr, wM, wcnt = ref.correspondences(src, tgt, guess, T_rel, scov=scov, tcov=tcov)
        assert cnt == wcnt and np.array_equal(corr, wcorr)
        ok = corr >= 0
        assert ok.sum() > 100
        assert rel(M[ok], wM[ok]) <= 1e-12 and np.isnan(M[~ok]).all()
        for x in ([0, 0, 0, 0, 0, 0], [-0.15, 0.12, 0.0, 0.001, 0.0, 0.025]):
            T = ref.pose(x, guess)  # applyState(guess, x): pclomp's functor pose, applied to the raw source
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


@pytest.mark.parametrize("case", ["16k", "64k", "large_rotation", "translated_guess", "far", "one_inner_step"])
def test_align_matches_the_reference(ref, case):
    n = 65536 if case == "64k" else 16384
    offset = (3000.0, -2000.0, 50.0) if case == "far" else (0, 0, 0)
    T_true = gr.pose((0.4, -0.3, 0.05), (0.01, 0.0, 0.6 if case == "large_rotation" else 0.06))
    if case == "translated_guess":
        T_true = gr.pose((4.0, -3.0, 0.2), (0.0, 0.01, 0.3))
    T_true = about(T_true, offset)
    tgt, src = pair(n, seed=3, offset=offset, T=T_true)
    extra = {"reg_max_optimizer_iterations": 1} if case == "one_inner_step" else {}
    r, scov, tcov = ready(tgt, src, **extra)
    guess = np.eye(4, dtype=np.float32)
    if case in ("large_rotation", "translated_guess"):  # a guess near the answer: a 0.6 rad rotation, or metres of translation
        guess = (gr.pose((0.02, 0.01, 0.0), (0.0, 0.0, 0.01)) @ np.linalg.inv(T_true)).astype(np.float32)
    T, conv, it, ncorr, ncost = _align(r, guess)
    w = ref.align(src, tgt, guess, scov=scov, tcov=tcov, max_optimizer_iterations=1 if extra else 20)
    assert (conv, it, ncorr) == (w["converged"], w["iterations"], w["corr_passes"])
    assert abs(ncost - w["cost_passes"]) <= max(2, w["cost_passes"] // 10)
    gr.end_point_is_as_good(T, w["T"])
    if case != "one_inner_step":
        assert conv and it >= 1
    assert np.max(np.abs(r.getAligned()[:, :3] - gr.transform(src, T)[:, :3])) <= 1e-3
    s = r.getFitnessScore()
    want = orc.fitness(tgt, src, T)[0]
    assert abs(s - want) <= 1e-12 * abs(want)
    r.close()


def test_identity_guess_is_gicp_and_a_translated_guess_is_not(ref):
    tgt, src = pair(16384, seed=5)
    out = {}
    for m in (OMP, "GICP"):
        r, scov, tcov = ready(tgt, src, m)
        T, conv, it, ncorr, ncost = _align(r, np.eye(4, dtype=np.float32))
        out[m] = (T, conv, it, ncorr, ncost, r.getFitnessScore(), scov, tcov)
        r.close()
    a, b = out[OMP], out["GICP"]
    assert np.array_equal(a[0], b[0]) and a[1:6] == b[1:6]
    assert np.array_equal(a[6], b[6]) and np.array_equal(a[7], b[7])
    # several metres of guess translation: pclomp's end pose is its own reference's, not GICP's
    T_true = gr.pose((4.0, -3.0, 0.2), (0.0, 0.01, 0.3))
    tgt, src = pair(16384, seed=6, T=T_true)
    guess = (gr.pose((0.05, -0.05, 0.0), (0.0, 0.0, 0.01)) @ np.linalg.inv(T_true)).astype(np.float32)
    res = {}
    for m in (OMP, "GICP"):
        r, scov, tcov = ready(tgt, src, m)
        res[m] = _align(r, guess)
        r.close()
    w = ref.align(src, tgt, guess, scov=scov, tcov=tcov)
    assert res[OMP][1] and res[OMP][2] == w["iterations"]
    gr.end_point_is_as_good(res[OMP][0], w["T"])
    assert np.max(np.abs(res[OMP][0] - res["GICP"][0])) > 1e-3


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
    guesses = [np.eye(4, dtype=np.float32), gr.pose((-2.0, 0.5, 0.0)), gr.pose((0.0, 3.1, 0.0), (0, 0, 0.01))]
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
    # the odometry mirror (with and without the next frame announced, with and without its own VOXELGRID) against a host loop
    for prefetch in (False, True):
        for ds in (pkg.B2R_DOWNSAMPLE_NONE, pkg.B2R_DOWNSAMPLE_VOXELGRID):
            o = pkg.ScanMatchingOdometry(handle(), keyframe_delta_trans=0.0, keyframe_delta_angle=0.0, keyframe_delta_time=0.0, downsample_method=ds,
                                         downsample_resolution=0.3)
            h2 = handle()
            fr = [c if ds == pkg.B2R_DOWNSAMPLE_NONE else h2.voxelGridFilter(c, 0.3) for c in clouds]
            o.matching(0.0, clouds[0])
            for k in range(1, 4):
                if prefetch and k + 1 < 4:
                    nxt = clouds[k + 1]
                    o.prefetch_raw(nxt.ctypes.data, nxt.shape[0], nxt.shape[1] * 4)
                st = o.matching(0.1 * k, clouds[k])
                h2.setInputTarget(fr[k - 1])
                h2.setInputSource(fr[k])
                h2.align(np.eye(4, dtype=np.float32))
                assert np.array_equal(st["trans"], h2.getFinalTransformation()) and st["converged"] == h2.hasConverged()
            o.close()
            h2.close()


@pytest.mark.parametrize("lanes_alone", [False, True])
def test_batch_matches_the_single_handle_bit_for_bit(lanes_alone):
    """b2r_batch_align (with fitness; all pairs co-scheduled, or each pair alone), b2r_batch_calc_fitness_score and the single-rank
    b2r_batch_loop_detect: every record equals the single handle's"""
    clouds = [gr.transform(gr.scene(16384, seed=20 + i), gr.pose((0.15 * i, -0.05 * i, 0.0), (0.0, 0.0, 0.015 * i))) for i in range(5)]
    guesses = [np.eye(4, dtype=np.float32), gr.pose((2.1, 0.0, 0.0)), gr.pose((0.0, -3.0, 0.0), (0, 0, 0.01)), gr.pose((0.05, 0.05, 0.0))]
    r = handle()
    single = []
    for i, g in enumerate(guesses):
        r.setInputTarget(clouds[0])
        r.setInputSource(clouds[1 + i])
        r.align(g)
        single.append((r.getFinalTransformation(), r.hasConverged(), r.nr_iterations, r.getFitnessScore(2.5)))
    r.close()
    lb = pkg.RegistrationBatch(params={"registration_method": OMP})
    ids = [lb.addCloud(c) for c in clouds]
    pairs = [(ids[1 + i], ids[0], g) for i, g in enumerate(guesses)]
    res = [lb.align([p], True, 2.5)[0] for p in pairs] if lanes_alone else lb.align(pairs, True, 2.5)
    for (T, conv, it, fit), x in zip(single, res):
        assert np.array_equal(T, x["T"]) and conv == x["converged"] and it == x["iterations"] and fit == x["fitness"]
    best, det = lb.loopDetect(pairs, [0, 2, 4], 2.5, 0.5)
    for a, d in zip(res, det):
        assert np.array_equal(a["T"], d["T"]) and a["fitness"] == d["fitness"] and a["converged"] == d["converged"]
    scores = lb.calcFitnessScore([(ids[0], ids[1 + i], single[i][0]) for i in range(len(guesses))], 2.5)
    for (T, _, _, fit), sc in zip(single, scores):
        assert sc == fit
    lb.close()


def test_taps_refuse_other_engines():
    tgt, src = pair(4096, seed=6)
    r, _, _ = ready(tgt, src)
    T = np.eye(4)
    for tap in (r.gicpLinearizeAt, r.gicpErrorAt, r.gicpPclCostAt):  # GICP's taps, and the cost tap before any correspondence pass
        with pytest.raises(pkg.B2RError) as e:
            tap(T)
        assert e.value.code == _capi.B2R_ESTATE
    with pytest.raises(pkg.B2RError) as e:
        r.icpPclCorrespondencesAt(T, src.shape[0])
    assert e.value.code == _capi.B2R_ESTATE
    r.close()
    for m in ("FAST_GICP", "B200_ICP"):
        g = pkg.select_registration_method({"registration_method": m})
        g.setInputTarget(tgt)
        g.setInputSource(src)
        with pytest.raises(pkg.B2RError) as e:
            g.gicpPclCorrespondencesAt(T, T, src.shape[0])
        assert e.value.code == _capi.B2R_ESTATE
        g.close()
