"""GPU: B200_VGICP_CUDA on degenerate and boundary inputs against tests/vgicp_cuda_ref.cpp: empty and tiny clouds (fewer than k points),
no source point inside any voxel, every point in one voxel, coordinates on the half-cell boundaries and at -0.0, non-finite points and the
21-bit extent limit.  Covariances, cells, counts, means, voxel covariances and correspondences bit-exact, cost within rel 1e-9."""
import numpy as np
import pytest

import hdl_graph_slam_b200 as pkg
import vgicp_cuda_ref as vc
import vgicp_ref as vr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return vc.Reference(tmp_path_factory.mktemp("vgicp_cuda_ref"))


def handle(res):
    return pkg.select_registration_method({"registration_method": "B200_VGICP_CUDA", "reg_resolution": str(res)})


def same_nan(a, b):
    return np.array_equal(a, b, equal_nan=True)


def check_against_ref(ref, tgt, src, res, T=np.eye(4)):
    r = handle(res)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    tcov, scov = r.getCovariances(1, tgt.shape[0]), r.getCovariances(0, src.shape[0])
    fin_t, fin_s = np.isfinite(tgt[:, :3]).all(axis=1), np.isfinite(src[:, :3]).all(axis=1)
    assert np.array_equal(tcov[fin_t], ref.covariances(tgt)[fin_t]) and np.array_equal(scov[fin_s], ref.covariances(src)[fin_s])
    m = ref.map(tgt, res, tcov)
    want, got = m.voxels(), r.vgicpGetVoxels()
    for key in ("cells", "counts", "mean", "cov"):
        assert np.array_equal(got[key], want[key]), key
    H, b, cost, nc, vox = r.vgicpLinearizeAt(T, src.shape[0])
    _, _, cr, vr_ = m.linearize(src, T, scov)
    assert np.array_equal(vox, vr_) and abs(cost - cr) <= 1e-9 * max(abs(cr), 1e-300)
    r.close()
    return want, vox


def test_empty_and_tiny_clouds(ref):
    r = handle(1.0)
    r.setInputTarget(np.zeros((0, 4), np.float32))
    r.setInputSource(vr.room(100))
    g = vr.rigid(0.1, [1, 2, 0]).astype(np.float32)
    r.align(g)
    assert not r.hasConverged() and r.nr_iterations == 0 and np.array_equal(r.getFinalTransformation(), g)
    assert r.vgicpGetVoxels()["counts"].size == 0
    r.close()
    # fewer than k points: the moments run over the neighbours found; the flag and pose are the reference's
    tgt = vr.records([[0.9, 0.9, 0.9], [1.2, 0.8, 0.7], [0.8, 1.3, 0.9], [1.1, 1.1, 1.4], [0.7, 0.6, 1.2]])
    src = vr.records([[0.85, 0.95, 0.9], [1.15, 0.85, 0.75], [0.8, 1.2, 1.0]])
    check_against_ref(ref, tgt, src, 1.0)
    r = handle(1.0)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    o = ref.map(tgt, 1.0, r.getCovariances(1, 5)).align(src, scov=r.getCovariances(0, 3))
    r.align(np.eye(4, dtype=np.float32))
    assert r.hasConverged() == o["converged"] and r.nr_iterations == o["iterations"]
    assert np.max(np.abs(r.getFinalTransformation().astype(np.float64) - o["T"])) <= 1e-6
    r.close()


def test_no_source_point_inside_any_voxel(ref):
    tgt = vr.room(3000, seed=1)
    src = vr.records(vr.room(2000, seed=2)[:, :3] + np.float32(100.0))
    _, vox = check_against_ref(ref, tgt, src, 1.0)
    assert (vox < 0).all()
    r = handle(1.0)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    r.align(np.eye(4, dtype=np.float32))
    o = ref.map(tgt, 1.0, r.getCovariances(1, tgt.shape[0])).align(src, scov=r.getCovariances(0, src.shape[0]))
    assert o["lm_failed"] and not o["converged"]  # "lm not converged": H = 0 has no step, the guess is kept
    assert not r.hasConverged() and r.nr_iterations == o["iterations"]
    assert np.array_equal(r.getFinalTransformation(), np.eye(4, dtype=np.float32))
    r.close()


def test_every_point_in_one_voxel(ref):
    rng = np.random.default_rng(3)
    tgt = vr.records(rng.uniform(0.51, 1.49, (500, 3)))  # cell 0 of floor(x - 0.5)
    src = vr.records(rng.uniform(0.51, 1.49, (400, 3)))
    want, vox = check_against_ref(ref, tgt, src, 1.0)
    assert want["counts"].tolist() == [500] and want["cells"].tolist() == [[0, 0, 0]] and (vox == 0).all()


@pytest.mark.parametrize("res", [0.25, 0.5, 1.0, 2.0])
def test_half_cell_boundaries_and_negative_zero(ref, res):
    k = np.arange(-6, 7, dtype=np.float64)
    g = (np.stack(np.meshgrid(k, k, k[5:8], indexing="ij"), -1).reshape(-1, 3) + 0.5) * res  # x / res - 0.5 whole: on a boundary
    g32 = g.astype(np.float32)
    pts = np.r_[g, g + res / 2, [[-0.0, -0.0, -0.0], [-0.0, 0.0, -0.0]], np.nextafter(g32, np.float32(-np.inf))]
    tgt = vr.records(pts)
    src = vr.records(pts[::3] + np.float32(res / 4))
    want, _ = check_against_ref(ref, tgt, src, res)
    # the float32 rule itself: x / res and - 0.5 rounded separately (a point one ulp below a boundary can round back onto it)
    rule = np.floor(tgt[:, :3] / np.float32(res) - np.float32(0.5)).astype(np.int64)
    assert np.array_equal(want["cells"], np.unique(rule, axis=0))
    assert [0, 0, 0] in want["cells"].tolist() and [-1, -1, -1] in want["cells"].tolist()


def test_non_finite_points(ref):
    tgt = vr.room(4000, seed=4)
    src = vr.room(3000, seed=5)
    tgt[::97, 1] = np.nan
    tgt[5::131, 2] = np.inf
    src[::89, 0] = -np.inf
    src[7::113, 2] = np.nan
    want, vox = check_against_ref(ref, tgt, src, 0.5)
    assert want["counts"].sum() == np.isfinite(tgt[:, :3]).all(axis=1).sum()
    assert (vox[~np.isfinite(src[:, :3]).all(axis=1)] == -1).all()


def test_extent_limit():
    res = 0.25
    r = handle(res)
    ok = vr.room(2000, seed=6)
    ok[0, :3] = [np.float32(2 ** 20 * res), 0, 0]  # floor(2^20 - 0.5) = 2^20 - 1
    r.setInputTarget(ok)
    assert r.vgicpGetVoxels()["cells"][:, 0].max() == 2 ** 20 - 1
    bad = ok.copy()
    bad[1, :3] = [0, -2 ** 20 * res - 1.0, 0]
    with pytest.raises(pkg.B2RError) as e:
        r.setInputTarget(bad)
    assert e.value.args and "21-bit" in str(e.value)
    r.close()
