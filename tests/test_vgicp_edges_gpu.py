"""GPU: FAST_VGICP on degenerate and boundary inputs against tests/vgicp_ref.cpp: empty and tiny clouds, no source point inside any
voxel, every point in one voxel, coordinates on cell boundaries and at -0.0, non-finite points and the 21-bit extent limit."""
import numpy as np
import pytest

import hdl_graph_slam_b200 as pkg
import vgicp_ref as vr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return vr.Reference(tmp_path_factory.mktemp("vgicp_ref"))


def handle(res):
    return pkg.select_registration_method({"registration_method": "FAST_VGICP", "reg_resolution": str(res)})


def check_against_ref(ref, tgt, src, res, T=np.eye(4)):
    r = handle(res)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    m = ref.map(tgt, res, r.getCovariances(1, tgt.shape[0]))
    want, got = m.voxels(), r.vgicpGetVoxels()
    assert np.array_equal(got["cells"], want["cells"]) and np.array_equal(got["counts"], want["counts"]) and np.array_equal(got["mean"], want["mean"])
    H, b, cost, nc, vox = r.vgicpLinearizeAt(T, src.shape[0])
    _, _, cr, vr_ = m.linearize(src, T, r.getCovariances(0, src.shape[0]))
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
    r.setInputTarget(vr.records([[0.5, 0.5, 0.5]]))
    r.setInputSource(vr.records([[0.4, 0.4, 0.4]]))
    v = r.vgicpGetVoxels()
    assert v["counts"].tolist() == [1] and v["cells"].tolist() == [[0, 0, 0]]
    # one correspondence: H has rank 3, the LM's damping makes every step solvable; the flag and pose are the reference's
    src = vr.records([[0.4, 0.4, 0.4]])
    o = ref.map(vr.records([[0.5, 0.5, 0.5]]), 1.0, r.getCovariances(1, 1)).align(src, scov=r.getCovariances(0, 1))
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
    assert not r.hasConverged() and np.array_equal(r.getFinalTransformation(), np.eye(4, dtype=np.float32))
    r.close()


def test_every_point_in_one_voxel(ref):
    rng = np.random.default_rng(3)
    tgt = vr.records(rng.uniform(0.01, 0.99, (500, 3)))
    src = vr.records(rng.uniform(0.01, 0.99, (400, 3)))
    want, vox = check_against_ref(ref, tgt, src, 1.0)
    assert want["counts"].tolist() == [500] and (vox == 0).all()


@pytest.mark.parametrize("res", [0.25, 0.5, 1.0, 2.0])
def test_cell_boundaries_and_negative_zero(ref, res):
    k = np.arange(-6, 7, dtype=np.float64)
    g = np.stack(np.meshgrid(k, k, k[5:8], indexing="ij"), -1).reshape(-1, 3) * res  # z = -1, 0, 1 cells
    pts = np.r_[g, g + res / 2, [[-0.0, -0.0, -0.0], [-0.0, 0.0, -0.0]], np.nextafter(g.astype(np.float32), np.float32(-np.inf))]
    tgt = vr.records(pts)
    src = vr.records(pts[::3] + np.float32(res / 4))
    want, _ = check_against_ref(ref, tgt, src, res)
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
    ok[0, :3] = [np.float32((2 ** 20 - 1) * res), 0, 0]
    r.setInputTarget(ok)
    assert r.vgicpGetVoxels()["cells"][:, 0].max() == 2 ** 20 - 1
    bad = ok.copy()
    bad[1, :3] = [0, -2 ** 20 * res - 1.0, 0]
    with pytest.raises(pkg.B2RError) as e:
        r.setInputTarget(bad)
    assert e.value.args and "21-bit" in str(e.value)
    r.close()


def test_gicp_error_tap_refuses_a_vgicp_handle():
    """b2r_gicp_error_at reads GICP correspondences (target point positions): on a VGICP handle, even after an align, it is B2R_ESTATE"""
    from hdl_graph_slam_b200 import _capi
    r = handle(1.0)
    r.setInputTarget(vr.room(3000, seed=8))
    r.setInputSource(vr.room(2000, seed=9))
    r.align(np.eye(4, dtype=np.float32))
    r.vgicpLinearizeAt(np.eye(4), 2000)
    with pytest.raises(pkg.B2RError) as e:
        r.gicpErrorAt(np.eye(4))
    assert e.value.code == _capi.B2R_ESTATE
    r.close()
