"""GPU: the pcl GICP engine (B2R_METHOD_GICP_PCL) on boundary inputs and through the entry points that move clouds around — clouds with
fewer than k points (the engine rule: the moments run over the neighbours found), non-finite points (no covariance, no correspondence),
an empty source, the prefetched source, b2r_promote_source_to_target, and the odometry mirror with its own VOXELGRID downsample — each
against tests/gicp_pcl_ref.cpp or against the single handle, bit for bit."""
import numpy as np
import pytest

import hdl_graph_slam_b200 as pkg
import gicp_pcl_ref as gr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return gr.Reference(tmp_path_factory.mktemp("gicp_pcl_ref"))


def handle(**extra):
    p = {"registration_method": "GICP"}
    p.update({k: str(v) for k, v in extra.items()})
    return pkg.select_registration_method(p)


def result(r):
    return r.getFinalTransformation(), r.hasConverged(), r.nr_iterations


def same(a, b):
    return np.array_equal(a[0], b[0]) and a[1:] == b[1:]


@pytest.mark.parametrize("n", [1, 5, 19, 20, 21])
def test_clouds_with_fewer_than_k_points(ref, n):
    rng = np.random.default_rng(n)
    p = np.c_[rng.uniform(-1, 1, (n, 3)), np.ones(n)].astype(np.float32)
    r = handle()
    r.setInputTarget(p)
    r.setInputSource(p)
    assert np.max(np.abs(r.getCovariances(1, n) - ref.covariances(p))) <= 1e-8
    r.align(np.eye(4, dtype=np.float32))
    w = ref.align(p, p, scov=r.getCovariances(0, n), tcov=r.getCovariances(1, n))
    assert (r.hasConverged(), r.nr_iterations) == (w["converged"], w["iterations"])
    assert np.max(np.abs(r.getFinalTransformation() - w["T"])) <= 1e-5
    r.close()


def test_non_finite_points(ref):
    tgt = gr.scene(8192, seed=30)
    src = gr.transform(gr.scene(8192, seed=31), gr.pose((0.2, -0.1, 0.0), (0.0, 0.0, 0.03)))
    tgt[::97, 0] = np.nan
    src[::89, 1] = np.inf
    src[5::101, 2] = np.nan
    r = handle()
    r.setInputTarget(tgt)
    r.setInputSource(src)
    scov, tcov = r.getCovariances(0, src.shape[0]), r.getCovariances(1, tgt.shape[0])
    bad_s = ~np.isfinite(src[:, :3]).all(axis=1)
    bad_t = ~np.isfinite(tgt[:, :3]).all(axis=1)
    assert np.isnan(scov[bad_s]).all() and np.isnan(tcov[bad_t]).all()
    assert np.max(np.abs(scov[~bad_s] - ref.covariances(src)[~bad_s])) <= 1e-8
    assert np.max(np.abs(tcov[~bad_t] - ref.covariances(tgt)[~bad_t])) <= 1e-8
    guess = np.eye(4, dtype=np.float32)
    corr, M, cnt = r.gicpPclCorrespondencesAt(guess, guess, src.shape[0])
    wc, wM, wcnt = ref.correspondences(src, tgt, guess, guess, scov=scov, tcov=tcov)
    assert cnt == wcnt and np.array_equal(corr, wc) and (corr[bad_s] == -1).all() and not np.isin(corr, np.flatnonzero(bad_t)).any()
    r.align(guess)
    w = ref.align(src, tgt, scov=scov, tcov=tcov)
    assert (r.hasConverged(), r.nr_iterations) == (w["converged"], w["iterations"])
    # the BFGS stops at |g| < 1e-2: where the line search's order-sensitive comparisons take another path (see test_gicp_pcl_gpu),
    # the end points differ within that stopping tolerance
    assert np.max(np.abs(r.getFinalTransformation() - w["T"])) <= 1e-4
    r.close()


def test_empty_source_reports_the_guess_unconverged():
    r = handle()
    r.setInputTarget(gr.scene(4096, seed=32))
    r.setInputSource(np.zeros((0, 4), np.float32))
    g = gr.pose((1.0, 2.0, 0.0))
    r.align(g)
    assert np.array_equal(r.getFinalTransformation(), g) and not r.hasConverged() and r.nr_iterations == 0
    r.close()


def test_prefetch_and_promotion_equal_fresh_handles():
    clouds = [gr.transform(gr.scene(16384, seed=40 + i), gr.pose((0.1 * i, 0.0, 0.0), (0.0, 0.0, 0.01 * i))) for i in range(3)]
    # prefetched source == a source set directly
    a = handle()
    a.setInputTarget(clouds[0])
    a.prefetchSource(clouds[1])
    a.setInputSource(clouds[1])
    a.align(np.eye(4, dtype=np.float32))
    b = handle()
    b.setInputTarget(clouds[0])
    b.setInputSource(clouds[1])
    b.align(np.eye(4, dtype=np.float32))
    assert same(result(a), result(b))
    assert np.array_equal(a.getCovariances(0, clouds[1].shape[0]), b.getCovariances(0, clouds[1].shape[0]))
    # the promoted source == the same cloud set as a target
    a.promoteSourceToTarget()
    a.setInputSource(clouds[2])
    a.align(np.eye(4, dtype=np.float32))
    c = handle()
    c.setInputTarget(clouds[1])
    c.setInputSource(clouds[2])
    c.align(np.eye(4, dtype=np.float32))
    assert same(result(a), result(c))
    assert np.array_equal(a.getCovariances(1, clouds[1].shape[0]), c.getCovariances(1, clouds[1].shape[0]))
    for h in (a, b, c):
        h.close()


def test_odometry_with_its_own_downsample_equals_the_single_handle_on_filtered_clouds():
    frames = [gr.transform(gr.scene(32768, seed=50 + k), gr.pose((0.05 * k, 0.0, 0.0), (0.0, 0.0, 0.005 * k))) for k in range(4)]
    leaf = 0.3
    o = pkg.ScanMatchingOdometry(handle(), keyframe_delta_trans=0.0, keyframe_delta_angle=0.0, keyframe_delta_time=0.0,
                                 downsample_method=pkg.B2R_DOWNSAMPLE_VOXELGRID, downsample_resolution=leaf)
    h = handle()
    filt = [h.voxelGridFilter(f, leaf) for f in frames]
    o.matching(0.0, frames[0])
    for k in range(1, len(frames)):
        st = o.matching(0.1 * k, frames[k])
        h.setInputTarget(filt[k - 1])
        h.setInputSource(filt[k])
        h.align(np.eye(4, dtype=np.float32))
        assert np.array_equal(st["trans"], h.getFinalTransformation()) and st["converged"] == h.hasConverged()
    o.close()
    h.close()
