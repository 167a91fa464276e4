"""GPU: the pclomp GICP engine (B2R_METHOD_GICP_OMP) on boundary inputs and through the entry points that move clouds around — an empty
source, clouds with fewer than k points, non-finite points, fewer than 4 correspondences, one optimizer iteration, a 262 144-point
pair, the prefetched source and b2r_promote_source_to_target — each against tests/gicp_omp_ref.cpp (covariances within 1e-8, as for pcl GICP) or against fresh
handles, bit for bit."""
import numpy as np
import pytest

import hdl_graph_slam_b200 as pkg
import gicp_omp_ref as gor
import gicp_pcl_ref as gr

pytestmark = pytest.mark.gpu
OFFSET_GUESS = gr.pose((1.5, -2.0, 0.1), (0.0, 0.0, 0.02))  # a translated guess: the pose rule matters


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return gor.Reference(tmp_path_factory.mktemp("gicp_omp_ref"))


def handle(**extra):
    p = {"registration_method": "B200_GICP_OMP"}
    p.update({k: str(v) for k, v in extra.items()})
    return pkg.select_registration_method(p)


def result(r):
    return r.getFinalTransformation(), r.hasConverged(), r.nr_iterations


def same(a, b):
    return np.array_equal(a[0], b[0]) and a[1:] == b[1:]


def test_empty_source_reports_the_guess_unconverged():
    r = handle()
    r.setInputTarget(gr.scene(4096, seed=32))
    r.setInputSource(np.zeros((0, 4), np.float32))
    r.align(OFFSET_GUESS)
    assert np.array_equal(r.getFinalTransformation(), OFFSET_GUESS) and not r.hasConverged() and r.nr_iterations == 0
    r.close()


@pytest.mark.parametrize("n", [1, 5, 19, 21])
def test_clouds_with_fewer_than_k_points(ref, n):
    rng = np.random.default_rng(n)
    p = np.c_[rng.uniform(-1, 1, (n, 3)), np.ones(n)].astype(np.float32)
    r = handle()
    r.setInputTarget(p)
    r.setInputSource(p)
    assert np.max(np.abs(r.getCovariances(1, n) - ref.covariances(p))) <= 1e-8
    g = gr.pose((0.05, 0.0, 0.0))
    r.align(g)
    w = ref.align(p, p, g, scov=r.getCovariances(0, n), tcov=r.getCovariances(1, n))
    assert (r.hasConverged(), r.nr_iterations) == (w["converged"], w["iterations"])
    assert np.max(np.abs(r.getFinalTransformation() - w["T"])) <= 1e-5
    r.close()


def test_non_finite_points(ref):
    tgt = gr.scene(8192, seed=30)
    src = gr.transform(gr.scene(8192, seed=31), np.linalg.inv(OFFSET_GUESS.astype(np.float64)).astype(np.float32))
    tgt[::97, 0] = np.nan
    src[::89, 1] = np.inf
    src[5::101, 2] = np.nan
    r = handle()
    r.setInputTarget(tgt)
    r.setInputSource(src)
    scov, tcov = r.getCovariances(0, src.shape[0]), r.getCovariances(1, tgt.shape[0])
    bad_s = ~np.isfinite(src[:, :3]).all(axis=1)
    assert np.isnan(scov[bad_s]).all()
    corr, M, cnt = r.gicpPclCorrespondencesAt(OFFSET_GUESS, np.eye(4, dtype=np.float32), src.shape[0])
    wc, _, wcnt = ref.correspondences(src, tgt, OFFSET_GUESS, np.eye(4, dtype=np.float32), scov=scov, tcov=tcov)
    assert cnt == wcnt and np.array_equal(corr, wc) and (corr[bad_s] == -1).all()
    r.align(OFFSET_GUESS)
    w = ref.align(src, tgt, OFFSET_GUESS, scov=scov, tcov=tcov)
    assert (r.hasConverged(), r.nr_iterations) == (w["converged"], w["iterations"])
    gr.end_point_is_as_good(r.getFinalTransformation(), w["T"])
    r.close()


def test_fewer_than_four_correspondences_end_unconverged(ref):
    tgt = gr.scene(4096, seed=33)
    src = tgt[:3].copy()  # three points: three correspondences at most
    r = handle(reg_correspondence_randomness=3)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    r.getStats(reset=True)
    r.align(np.eye(4, dtype=np.float32))
    st = r.getStats()
    assert not r.hasConverged() and r.nr_iterations == 0 and st["launches"]["gicp_pcl_cost"] == 0
    assert np.array_equal(r.getFinalTransformation(), np.eye(4, dtype=np.float32))
    w = ref.align(src, tgt, k=3)
    assert not w["converged"] and w["iterations"] == 0
    r.close()


def test_one_optimizer_iteration(ref):
    tgt = gr.scene(16384, seed=34)
    src = gr.transform(gr.scene(16384, seed=35), np.linalg.inv(OFFSET_GUESS.astype(np.float64)).astype(np.float32) @ gr.pose((0.1, 0.0, 0.0)))
    r = handle(reg_max_optimizer_iterations=1, reg_maximum_iterations=12)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    r.align(OFFSET_GUESS)
    w = ref.align(src, tgt, OFFSET_GUESS, scov=r.getCovariances(0, src.shape[0]), tcov=r.getCovariances(1, tgt.shape[0]), max_optimizer_iterations=1,
                  max_iterations=12)
    assert (r.hasConverged(), r.nr_iterations) == (w["converged"], w["iterations"]) and w["bfgs_steps"] == w["iterations"]
    gr.end_point_is_as_good(r.getFinalTransformation(), w["T"])
    r.close()


def test_262144_points(ref):
    T_true = gr.pose((0.3, -0.2, 0.03), (0.0, 0.0, 0.04))
    tgt = gr.scene(262144, seed=36)
    src = gr.transform(gr.scene(262144, seed=37), T_true)
    guess = (gr.pose((0.02, 0.0, 0.0)) @ np.linalg.inv(T_true)).astype(np.float32)
    r = handle()
    r.setInputTarget(tgt)
    r.setInputSource(src)
    scov, tcov = r.getCovariances(0, src.shape[0]), r.getCovariances(1, tgt.shape[0])
    assert np.max(np.abs(scov - ref.covariances(src))) <= 1e-8
    r.align(guess)
    w = ref.align(src, tgt, guess, scov=scov, tcov=tcov)
    assert (r.hasConverged(), r.nr_iterations) == (w["converged"], w["iterations"]) and r.hasConverged()
    gr.end_point_is_as_good(r.getFinalTransformation(), w["T"])
    r.close()


def test_prefetch_and_promotion_equal_fresh_handles():
    clouds = [gr.transform(gr.scene(16384, seed=40 + i), gr.pose((0.1 * i, 0.0, 0.0), (0.0, 0.0, 0.01 * i))) for i in range(3)]
    a = handle()
    a.setInputTarget(clouds[0])
    a.prefetchSource(clouds[1])
    a.setInputSource(clouds[1])
    a.align(OFFSET_GUESS)
    b = handle()
    b.setInputTarget(clouds[0])
    b.setInputSource(clouds[1])
    b.align(OFFSET_GUESS)
    assert same(result(a), result(b))
    assert np.array_equal(a.getCovariances(0, clouds[1].shape[0]), b.getCovariances(0, clouds[1].shape[0]))
    a.promoteSourceToTarget()
    a.setInputSource(clouds[2])
    a.align(OFFSET_GUESS)
    c = handle()
    c.setInputTarget(clouds[1])
    c.setInputSource(clouds[2])
    c.align(OFFSET_GUESS)
    assert same(result(a), result(c))
    assert np.array_equal(a.getCovariances(1, clouds[1].shape[0]), c.getCovariances(1, clouds[1].shape[0]))
    for h in (a, b, c):
        h.close()
