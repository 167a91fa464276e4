"""CPU-only: the sequential VGICP reference (tests/vgicp_ref.cpp) against an independent numpy / scipy restatement of
fast_gicp::FastVGICP (np.floor(p / res) cells, np.unique grouping, cKDTree k-NN PLANE covariances, H / b / cost by plain sums), and
known-answer tests: a hand-computed voxel, a one-point voxel, w = sqrt(num_points), the cost's derivative against b, recovery of a
known transform and the extent limit."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

import vgicp_ref as vr
from common import axis_lines, jacobisvd_diagonal_normal


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return vr.Reference(tmp_path_factory.mktemp("vgicp_ref"))


def np_covariances(pts, k=20):
    """FastGICP::calculate_covariances, PLANE: k-NN (self included) covariance / k, singular values replaced by (1, 1, 1e-3)"""
    p = pts[:, :3].astype(np.float64)
    _, idx = cKDTree(pts[:, :3]).query(pts[:, :3], k=k)
    out = np.empty((p.shape[0], 3, 3))
    for i in range(p.shape[0]):
        nb = p[idx[i]]
        d = nb - nb.mean(axis=0)
        C = d.T @ d / k
        n = jacobisvd_diagonal_normal(C)  # tied singular values of an exactly diagonal C: JacobiSVD's column, not LAPACK's
        if n is not None:
            out[i] = np.eye(3) - (1.0 - 1e-3) * np.outer(n, n)
            continue
        U, _, Vt = np.linalg.svd(C)
        out[i] = U @ np.diag([1.0, 1.0, 1e-3]) @ Vt
    return out


def np_voxels(tgt, cov, res):
    p = tgt[:, :3].astype(np.float64)
    fin = np.isfinite(p).all(axis=1)
    cells = np.floor(p[fin] / res).astype(np.int64)
    u, inv, cnt = np.unique(cells, axis=0, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    mean = np.zeros((u.shape[0], 3))
    C = np.zeros((u.shape[0], 3, 3))
    np.add.at(mean, inv, p[fin])
    np.add.at(C, inv, cov[fin])
    return dict(cells=u.astype(np.int32), counts=cnt.astype(np.int32), mean=mean / cnt[:, None], cov=C / cnt[:, None, None])


def np_linearize(vox, res, src, scov, T):
    lut = {tuple(c): v for v, c in enumerate(vox["cells"])}
    R, t0 = T[:3, :3], T[:3, 3]
    H = np.zeros((6, 6))
    b = np.zeros(6)
    cost = 0.0
    vox_of = np.full(src.shape[0], -1, np.int32)
    for i, a in enumerate(src[:, :3].astype(np.float64)):
        if not np.isfinite(a).all():
            continue
        ta = R @ a + t0
        v = lut.get(tuple(np.floor(ta / res).astype(np.int64)))
        if v is None:
            continue
        vox_of[i] = v
        M = np.linalg.inv(vox["cov"][v] + R @ scov[i] @ R.T)
        w = np.sqrt(vox["counts"][v])
        e = vox["mean"][v] - ta
        J = np.c_[np.array([[0, -ta[2], ta[1]], [ta[2], 0, -ta[0]], [-ta[1], ta[0], 0]]), -np.eye(3)]
        cost += w * e @ M @ e
        H += w * J.T @ M @ J
        b += w * J.T @ M @ e
    return H, b, cost, vox_of


def test_covariances_match_the_independent_restatement():
    tgt = vr.room(3000, seed=1)
    got = vr.covariances(tgt)
    want = np_covariances(tgt)
    assert np.max(np.abs(got - want)) < 1e-8


def test_axis_line_covariances_match_the_independent_restatement():
    """exactly diagonal covariances (common.axis_lines): the restatement's diagonal branch against the oracle; the regularised matrix
    depends on the normal alone, so the tie order of the k-NN lists does not matter"""
    p = axis_lines(n_per_axis=4, seed=1)
    assert np.max(np.abs(vr.covariances(p, 20) - np_covariances(p, 20))) <= 1e-12


@pytest.mark.parametrize("res", [0.25, 0.5, 1.0, 2.0])
def test_voxel_map_matches_the_independent_restatement(ref, res):
    tgt = vr.room(4000, seed=2)
    cov = vr.covariances(tgt)
    m = ref.map(tgt, res, cov)
    assert m.status == 0
    got = m.voxels()
    want = np_voxels(tgt, cov, res)
    assert np.array_equal(got["cells"], want["cells"]) and np.array_equal(got["counts"], want["counts"])
    assert np.allclose(got["mean"], want["mean"], rtol=0, atol=1e-12)
    assert np.max(np.abs(got["cov"] - want["cov"])) < 1e-12


@pytest.mark.parametrize("res", [0.5, 1.0])
def test_linearize_matches_the_independent_restatement(ref, res):
    tgt = vr.room(4000, seed=3)
    T = vr.rigid(0.03, [0.2, -0.1, 0.05])
    src = vr.moved(vr.room(3000, seed=4), T)
    tcov, scov = vr.covariances(tgt), vr.covariances(src)
    m = ref.map(tgt, res, tcov)
    at = vr.rigid(0.02, [0.15, -0.05, 0.0])
    H, b, cost, vox = m.linearize(src, at, scov)
    Hn, bn, cn, vn = np_linearize(np_voxels(tgt, tcov, res), res, src, scov, at)
    assert np.array_equal(vox, vn) and (vox >= 0).sum() > 1000
    assert abs(cost - cn) <= 1e-9 * abs(cn)
    assert np.max(np.abs(H - Hn)) <= 1e-9 * np.max(np.abs(Hn))
    assert np.max(np.abs(b - bn)) <= 1e-9 * np.max(np.abs(bn))


def test_hand_computed_voxel(ref):
    """three points of cell (1, 0, -1) at resolution 0.5 and one of cell (0, 0, 0): counts, means and covariances by hand"""
    pts = vr.records([[0.5, 0.0, -0.5], [0.75, 0.25, -0.25], [0.9, 0.4, -0.1], [0.1, 0.1, 0.1]])
    cov = np.stack([np.eye(3) * s for s in (1.0, 2.0, 6.0, 5.0)])
    v = ref.map(pts, 0.5, cov).voxels()
    assert v["cells"].tolist() == [[0, 0, 0], [1, 0, -1]]
    assert v["counts"].tolist() == [1, 3]
    want = (np.float64(np.float32(0.5)) + np.float64(np.float32(0.75)) + np.float64(np.float32(0.9))) / 3
    assert v["mean"][1][0] == want
    assert np.array_equal(v["cov"][1], np.eye(3) * 3.0)


def test_one_point_voxel_and_non_finite_points(ref):
    pts = vr.records([[3.3, -2.2, 1.1], [np.nan, 0, 0], [0, np.inf, 0]])
    cov = np.stack([np.diag([1.0, 2.0, 3.0]), np.eye(3), np.eye(3)])
    v = ref.map(pts, 1.0, cov).voxels()
    assert v["cells"].tolist() == [[3, -3, 1]] and v["counts"].tolist() == [1]
    assert np.array_equal(v["mean"][0], pts[0, :3].astype(np.float64)) and np.array_equal(v["cov"][0], cov[0])


def test_cost_weight_is_sqrt_num_points(ref):
    """four target points in one voxel, unit covariances, one source point: M = I / 2, w = sqrt(4) = 2, cost = |e|^2"""
    tgt = vr.records([[0.1, 0.1, 0.1], [0.3, 0.2, 0.1], [0.2, 0.4, 0.3], [0.2, 0.1, 0.7]])
    src = vr.records([[0.5, 0.5, 0.5]])
    m = ref.map(tgt, 1.0, np.stack([np.eye(3)] * 4))
    _, _, cost, vox = m.linearize(src, np.eye(4), np.stack([np.eye(3)]))
    e = m.voxels()["mean"][0] - src[0, :3].astype(np.float64)
    assert vox.tolist() == [0] and abs(cost - e @ e) <= 1e-15


def test_cost_derivative_is_twice_b(ref):
    """compute_error with the correspondences of T: central differences of the cost along exp(eps e_k) T equal 2 b_k"""
    tgt = vr.room(3000, seed=5)
    src = vr.moved(vr.room(2000, seed=6), vr.rigid(0.02, [0.1, 0.05, 0.0]))
    m = ref.map(tgt, 1.0)
    T = np.eye(4)
    _, b, _, _ = m.linearize(src, T)
    h = 1e-6
    for k in range(6):
        xi = np.zeros(6)
        xi[k] = h
        d = []
        for sgn in (1, -1):
            D = np.eye(4)
            w = sgn * xi[:3]
            th = np.linalg.norm(w)
            K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
            D[:3, :3] = np.eye(3) + (np.sin(th) / th if th else 1) * K + ((1 - np.cos(th)) / th ** 2 if th else 0.5) * K @ K
            D[:3, 3] = sgn * xi[3:]
            d.append(m.error(src, T, D @ T))
        assert abs((d[0] - d[1]) / (2 * h) - 2 * b[k]) <= 1e-5 * max(1.0, np.max(np.abs(b)))


def test_recovers_a_known_transform(ref):
    tgt = vr.room(20000, seed=7)
    T_true = vr.rigid(0.05, [0.3, -0.2, 0.05])
    src = vr.moved(tgt, T_true)
    o = ref.map(tgt, 0.5).align(src)
    assert o["converged"]
    assert np.max(np.abs(o["T64"][:3, 3] - T_true[:3, 3])) < 0.02
    assert np.max(np.abs(o["T64"][:3, :3] - T_true[:3, :3])) < 5e-3


def test_extent_limit(ref):
    res = 0.25
    edge = np.float32((2 ** 20 - 1) * res)
    ok = ref.map(vr.records([[edge, 0, 0], [-2 ** 20 * res, 0, 0]]), res, np.stack([np.eye(3)] * 2))
    assert ok.status == 0 and ok.voxels()["cells"][:, 0].tolist() == [-2 ** 20, 2 ** 20 - 1]
    assert ref.map(vr.records([[2 ** 20 * res, 0, 0]]), res, np.stack([np.eye(3)])).status == 1
