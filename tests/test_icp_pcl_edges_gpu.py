"""GPU: the pcl ICP engine on boundary inputs, against tests/icp_pcl_ref.cpp: empty and tiny clouds, the inclusive threshold to the ulp,
duplicate points under the reciprocal check, non-finite points, one iteration, a 262 144-point cloud, prefetch and promotion."""
import numpy as np
import pytest

import hdl_graph_slam_b200 as pkg
import icp_pcl_ref as ir
from gicp_pcl_ref import pose, scene, transform

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return ir.Reference(tmp_path_factory.mktemp("icp_pcl_ref"))


def handle(**extra):
    p = {"registration_method": "B200_ICP"}
    p.update({k: str(v).lower() if isinstance(v, bool) else str(v) for k, v in extra.items()})
    return pkg.select_registration_method(p)


def check_align(ref, src, tgt, guess=None, **cfg):
    extra = {}
    if "reciprocal" in cfg:
        extra["reg_use_reciprocal_correspondences"] = cfg["reciprocal"]
    if "max_iterations" in cfg:
        extra["reg_maximum_iterations"] = cfg["max_iterations"]
    if "max_dist" in cfg:
        extra["reg_max_correspondence_distance"] = repr(cfg["max_dist"])
    r = handle(**extra)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    g = np.eye(4, dtype=np.float32) if guess is None else guess
    r.align(g)
    w = ref.align(src, tgt, g, **cfg)
    assert (r.hasConverged(), r.nr_iterations) == (w["converged"], w["iterations"])
    assert np.max(np.abs(r.getFinalTransformation() - w["T"])) <= 1e-5
    out = (r.getFinalTransformation(), r.hasConverged(), r.nr_iterations)
    r.close()
    return out


def test_empty_and_tiny_clouds(ref):
    tgt = scene(4096, seed=1)
    empty = np.zeros((0, 4), np.float32)
    r = handle()
    r.setInputTarget(tgt)
    r.setInputSource(empty)
    g = pose((0.1, 0.0, 0.0))
    r.align(g)
    assert not r.hasConverged() and r.nr_iterations == 0 and np.array_equal(r.getFinalTransformation(), g)
    r.setInputTarget(empty)
    r.setInputSource(tgt)
    r.align(g)
    assert not r.hasConverged() and r.nr_iterations == 0
    r.close()
    for n in (1, 2, 3, 4, 31, 33, 1025):
        t = scene(max(n, 4), seed=2)[:n]
        s = transform(t, pose((0.05, 0.0, 0.0)))
        check_align(ref, s, t)


@pytest.mark.parametrize("reciprocal", [False, True])
def test_threshold_is_inclusive_to_the_ulp(ref, reciprocal):
    """d2 == (float) max_dist^2 is accepted, one ulp above is refused, forward and reverse"""
    t = np.zeros((64, 4), np.float32)
    t[:, 0] = np.arange(64) * 10.0
    t[:, 3] = 1
    s = t.copy()
    s[:, 1] = 0.75  # d2 = 0.5625 exactly
    s[1::2, 1] = np.nextafter(np.float32(0.75), np.float32(1))
    r = handle(reg_max_correspondence_distance=0.75, reg_use_reciprocal_correspondences=reciprocal)
    r.setInputTarget(t)
    r.setInputSource(s)
    corr, d2, cnt = r.icpPclCorrespondencesAt(np.eye(4), 64)
    wc, wd, wcnt = ref.correspondences(s, t, np.eye(4), 0.75, reciprocal)
    assert np.array_equal(corr, wc) and cnt == wcnt == 32
    assert (corr[0::2] == np.arange(0, 64, 2)).all() and (corr[1::2] == -1).all()
    r.close()


@pytest.mark.parametrize("reciprocal", [False, True])
def test_duplicate_points(ref, reciprocal):
    tgt = scene(8192, seed=3)
    src = transform(scene(8192, seed=4), pose((0.2, 0.1, 0.0), (0, 0, 0.02)))
    src = np.vstack([src, src[:500]])          # duplicate source points: the reverse search keeps the lower index only
    tgt = np.vstack([tgt, tgt[100:600]])       # duplicate target points: the forward search keeps the lower index
    r = handle(reg_use_reciprocal_correspondences=reciprocal)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    corr, d2, cnt = r.icpPclCorrespondencesAt(np.eye(4), src.shape[0])
    wc, wd, wcnt = ref.correspondences(src, tgt, np.eye(4), 2.5, reciprocal)
    assert np.array_equal(corr, wc) and cnt == wcnt
    assert not np.isin(corr, np.arange(8192, 8192 + 500)).any()
    if reciprocal:
        assert (corr[8192:] == -1).all()
    r.close()
    check_align(ref, src, tgt, reciprocal=reciprocal)


@pytest.mark.parametrize("reciprocal", [False, True])
def test_non_finite_points(ref, reciprocal):
    tgt = scene(8192, seed=5)
    src = transform(scene(8192, seed=6), pose((0.2, 0.0, 0.0)))
    src[::50, 1] = np.nan
    src[7::91, 2] = np.inf
    tgt[3::77, 0] = -np.inf
    r = handle(reg_use_reciprocal_correspondences=reciprocal)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    corr, d2, cnt = r.icpPclCorrespondencesAt(pose((0.01, 0, 0)), src.shape[0])
    wc, wd, wcnt = ref.correspondences(src, tgt, pose((0.01, 0, 0)), 2.5, reciprocal)
    assert np.array_equal(corr, wc) and cnt == wcnt
    assert (corr[::50] == -1).all() and not np.isin(corr, np.arange(3, 8192, 77)).any()
    r.close()
    check_align(ref, src, tgt, reciprocal=reciprocal)


def test_one_iteration_and_a_large_cloud(ref):
    tgt = scene(16384, seed=7)
    src = transform(scene(16384, seed=8), pose((0.3, 0.0, 0.0), (0, 0, 0.03)))
    T, conv, it = check_align(ref, src, tgt, max_iterations=1)
    assert conv and it == 1
    tgt = scene(262144, seed=9)
    src = transform(scene(262144, seed=10), pose((0.2, -0.1, 0.0), (0, 0, 0.02)))
    for reciprocal in (False, True):
        check_align(ref, src, tgt, reciprocal=reciprocal)


def test_prefetch_and_promotion(ref):
    clouds = [transform(scene(16384, seed=30 + i), pose((0.1 * i, 0.0, 0.0), (0, 0, 0.01 * i))) for i in range(3)]
    a = handle()
    a.setInputTarget(clouds[0])
    a.setInputSource(clouds[1])
    a.prefetchSource(clouds[2])
    a.align(np.eye(4))
    T1 = a.getFinalTransformation()
    a.promoteSourceToTarget()
    a.setInputSource(clouds[2])  # adopts the prefetched cloud
    a.align(np.eye(4))
    T2 = a.getFinalTransformation()
    a.getStats(reset=True)
    a.close()
    b = handle()
    for (t, s), T in (((0, 1), T1), ((1, 2), T2)):
        b.setInputTarget(clouds[t])
        b.setInputSource(clouds[s])
        b.align(np.eye(4))
        assert np.array_equal(b.getFinalTransformation(), T)
    st = b.getStats()
    assert st["launches"]["knn_covariance"] == 0
    b.close()
