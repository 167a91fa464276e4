"""CPU-only: the sequential FastVGICPCuda reference (tests/vgicp_cuda_ref.cpp) against an independent numpy / scipy restatement of
fast_gicp::FastVGICPCuda (float32 moments on cKDTree lists, np.floor(np.float32(x) / np.float32(res) - np.float32(0.5)) cells, np.unique
grouping, float32 terms by plain loops), and known answers: a hand-computed voxel, a one-point voxel, w = sqrt(num_points), the cost's
central differences against 2 b, recovery of a known transform, cells on the half-cell boundary and a cloud far from the origin."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

import vgicp_cuda_ref as vc
import vgicp_ref as vr

f32 = np.float32


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return vc.Reference(tmp_path_factory.mktemp("vgicp_cuda_ref"))


def np_lists(pts, k):
    """k-NN lists (self included) in ascending (float32 d2, index), from cKDTree candidates"""
    p = pts[:, :3]
    kk = min(k + 4, p.shape[0])
    _, cand = cKDTree(p.astype(np.float64)).query(p.astype(np.float64), k=kk)
    cand = cand.reshape(p.shape[0], kk)
    d = p[cand] - p[:, None, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    order = np.array([np.lexsort((c, e)) for c, e in zip(cand, d2)])
    return np.take_along_axis(cand, order, axis=1)[:, :min(k, p.shape[0])]


def np_moments(pts, k=20):
    """float32 raw moments: mean += p, S += p p^T over the list in order; cov = S / k - mean mean^T (n, 3, 3) float32"""
    p = np.ascontiguousarray(pts[:, :3], f32)
    idx = np_lists(pts, k)
    kk = idx.shape[1]
    m = np.zeros((p.shape[0], 3), f32)
    S = np.zeros((p.shape[0], 3, 3), f32)
    for j in range(kk):
        q = p[idx[:, j]]
        m = m + q
        S = S + q[:, :, None] * q[:, None, :]
    kf = f32(kk)
    m = m / kf
    return S / kf - m[:, :, None] * m[:, None, :]


def np_plane(C):
    """U diag(1, 1, 1e-3) U^T of the eigenvectors in float64"""
    _, U = np.linalg.eigh(C.astype(np.float64))
    return U @ np.diag([1e-3, 1.0, 1.0]) @ np.swapaxes(U, -1, -2)


def np_cells(p, res):
    return np.floor(np.asarray(p, f32) / f32(res) - f32(0.5)).astype(np.int64)


def np_voxels(tgt, cov, res):
    p = np.asarray(tgt[:, :3], f32)
    fin = np.isfinite(p).all(axis=1)
    u, inv = np.unique(np_cells(p[fin], res), axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    pf, cf = p[fin], np.asarray(cov[fin], f32)
    V = u.shape[0]
    mean = np.zeros((V, 3), f32)
    C = np.zeros((V, 3, 3), f32)
    cnt = np.zeros(V, np.int32)
    for i in range(pf.shape[0]):  # ascending point index
        v = inv[i]
        cnt[v] += 1
        mean[v] = mean[v] + pf[i]
        C[v] = C[v] + cf[i]
    return dict(cells=u.astype(np.int32), counts=cnt, mean=mean / cnt.astype(f32)[:, None], cov=C / cnt.astype(f32)[:, None, None])


def np_terms(vox, res, src, scov, T):
    """float32 terms per correspondence (plain loops), summed in float64 in source index order"""
    lut = {tuple(c): v for v, c in enumerate(vox["cells"])}
    Tf = np.asarray(T, np.float64)[:3].astype(f32)
    R = Tf[:, :3]
    H = np.zeros((6, 6))
    b = np.zeros(6)
    cost = 0.0
    vox_of = np.full(src.shape[0], -1, np.int32)
    for i in range(src.shape[0]):
        a = src[i, :3].astype(f32)
        if not np.isfinite(a).all():
            continue
        x = np.array([((Tf[r, 0] * a[0] + Tf[r, 1] * a[1]) + Tf[r, 2] * a[2]) + Tf[r, 3] for r in range(3)], f32)
        v = lut.get(tuple(np_cells(x, res)))
        if v is None:
            continue
        vox_of[i] = v
        CA = scov[i].astype(f32)
        CB = vox["cov"][v].astype(f32)
        RC = np.array([[(R[r, 0] * CA[0, j] + R[r, 1] * CA[1, j]) + R[r, 2] * CA[2, j] for j in range(3)] for r in range(3)], f32)
        m = np.zeros((3, 3), f32)
        for r in range(3):
            for j in range(r, 3):
                m[r, j] = m[j, r] = CB[r, j] + ((RC[r, 0] * R[j, 0] + RC[r, 1] * R[j, 1]) + RC[r, 2] * R[j, 2])
        cof = np.zeros((3, 3), f32)
        for r in range(3):
            for j in range(3):
                r1, r2, j1, j2 = (r + 1) % 3, (r + 2) % 3, (j + 1) % 3, (j + 2) % 3
                cof[r, j] = m[r1, j1] * m[r2, j2] - m[r1, j2] * m[r2, j1]
        inv = f32(1) / ((cof[0, 0] * m[0, 0] + cof[1, 0] * m[1, 0]) + cof[2, 0] * m[2, 0])
        M = (cof.T * inv).astype(f32)
        w = np.sqrt(f32(vox["counts"][v]))
        e = (vox["mean"][v].astype(f32) - x).astype(f32)
        Me = np.array([(M[r, 0] * e[0] + M[r, 1] * e[1]) + M[r, 2] * e[2] for r in range(3)], f32)

        def st(k, X):  # (skew(x)^T X)_k
            return [x[2] * X[1] - x[1] * X[2], x[0] * X[2] - x[2] * X[0], x[1] * X[0] - x[0] * X[1]][k]
        MS = np.array([[st(c, M[r]) for c in range(3)] for r in range(3)], f32)
        for p_ in range(6):
            for q_ in range(p_, 6):
                if q_ < 3:
                    h = w * st(p_, MS[:, q_])
                elif p_ < 3:
                    h = -(w * st(p_, M[:, q_ - 3]))
                else:
                    h = w * M[p_ - 3, q_ - 3]
                H[p_, q_] += float(h)
        for k in range(3):
            b[k] += float(w * st(k, Me))
            b[3 + k] += float(-(w * Me[k]))
        cost += float(w * ((e[0] * Me[0] + e[1] * Me[1]) + e[2] * Me[2]))
    H = np.triu(H) + np.triu(H, 1).T
    return H, b, cost, vox_of


def test_covariances_match_the_independent_restatement(ref):
    pts = vr.room(3000, seed=1)
    got = ref.covariances(pts)
    want = np_plane(np_moments(pts))
    assert np.max(np.abs(got - want)) < 2e-4
    assert np.array_equal(got, np.swapaxes(got, 1, 2))  # stored from the upper triangle
    assert np.array_equal(got.astype(f32).astype(np.float64), got)  # float32 values


def test_far_from_origin_moments_are_float32(ref):
    """at (3000, -2000, 50) the float32 raw moments cancel: the covariances differ visibly from FastGICP's (float64, demeaned) while
    matching the float32 restatement"""
    off = np.array([3000.0, -2000.0, 50.0])
    pts = vr.records(vr.room(2000, seed=9)[:, :3].astype(np.float64) + off)
    got = ref.covariances(pts)
    want32 = np_plane(np_moments(pts))
    fast = vr.covariances(pts)
    near = np.max(np.abs(got - want32), axis=(1, 2)) < 2e-3
    assert near.mean() > 0.95
    assert np.max(np.abs(got - fast)) > 0.1


@pytest.mark.parametrize("res", [0.25, 0.5, 1.0, 2.0])
def test_voxel_map_matches_the_independent_restatement(ref, res):
    tgt = vr.room(4000, seed=2)
    cov = ref.covariances(tgt)
    m = ref.map(tgt, res, cov)
    assert m.status == 0
    got = m.voxels()
    want = np_voxels(tgt, cov, res)
    assert np.array_equal(got["cells"], want["cells"]) and np.array_equal(got["counts"], want["counts"])
    assert np.array_equal(got["mean"], want["mean"].astype(np.float64))
    assert np.array_equal(got["cov"], want["cov"].astype(np.float64))


@pytest.mark.parametrize("res", [0.5, 1.0])
def test_linearize_matches_the_independent_restatement(ref, res):
    tgt = vr.room(3000, seed=3)
    T = vr.rigid(0.03, [0.2, -0.1, 0.05])
    src = vr.moved(vr.room(1500, seed=4), T)
    tcov, scov = ref.covariances(tgt), ref.covariances(src)
    m = ref.map(tgt, res, tcov)
    at = vr.rigid(0.02, [0.15, -0.05, 0.0])
    H, b, cost, vox = m.linearize(src, at, scov)
    Hn, bn, cn, vn = np_terms(np_voxels(tgt, tcov, res), res, src, scov, at)
    assert np.array_equal(vox, vn) and (vox >= 0).sum() > 500
    assert abs(cost - cn) <= 1e-12 * abs(cn)
    assert np.max(np.abs(H - Hn)) <= 1e-12 * np.max(np.abs(Hn))
    assert np.max(np.abs(b - bn)) <= 1e-12 * np.max(np.abs(bn))


def test_hand_computed_voxel(ref):
    """cell = floor(x / 0.5 - 0.5): three points of cell (1, -1, -2) and one of cell (-1, -1, -1); means in float32 by hand"""
    pts = vr.records([[0.8, 0.0, -0.5], [0.75, 0.1, -0.55], [0.9, 0.2, -0.6], [0.1, 0.1, 0.1]])
    cov = np.stack([np.eye(3) * s for s in (1.0, 2.0, 6.0, 5.0)])
    v = ref.map(pts, 0.5, cov).voxels()
    assert v["cells"].tolist() == [[-1, -1, -1], [1, -1, -2]]
    assert v["counts"].tolist() == [1, 3]
    want = ((f32(0.8) + f32(0.75)) + f32(0.9)) / f32(3)
    assert v["mean"][1][0] == np.float64(want)
    assert np.array_equal(v["cov"][1], np.eye(3) * 3.0)


def test_one_point_voxel_and_non_finite_points(ref):
    pts = vr.records([[3.3, -2.2, 1.1], [np.nan, 0, 0], [0, np.inf, 0]])
    cov = np.stack([np.diag([1.0, 2.0, 3.0]), np.eye(3), np.eye(3)])
    v = ref.map(pts, 1.0, cov).voxels()
    assert v["cells"].tolist() == [[2, -3, 0]] and v["counts"].tolist() == [1]
    assert np.array_equal(v["mean"][0], pts[0, :3].astype(np.float64)) and np.array_equal(v["cov"][0], cov[0])


def test_half_cell_boundary(ref):
    """x / res - 0.5 exactly whole: the point opens the upper cell; one ulp below it stays in the lower one"""
    res = 0.5
    on = f32(0.75)  # 0.75 / 0.5 - 0.5 = 1
    below = np.nextafter(on, f32(0))
    v = ref.map(vr.records([[on, -0.25, 0.25], [below, -0.25, 0.25]]), res, np.stack([np.eye(3)] * 2)).voxels()
    assert v["cells"].tolist() == [[0, -1, 0], [1, -1, 0]]
    assert np.array_equal(v["cells"], np.unique(np_cells(np.array([[on, -0.25, 0.25], [below, -0.25, 0.25]], f32), res), axis=0))


def test_cost_weight_is_sqrt_num_points(ref):
    """four target points in one voxel, unit covariances, one source point: M = I / 2, w = 2, cost = |e|^2 (float32)"""
    tgt = vr.records([[0.6, 0.6, 0.6], [0.8, 0.7, 0.6], [0.7, 0.9, 0.8], [0.7, 0.6, 1.2]])
    src = vr.records([[1.0, 1.0, 1.0]])
    m = ref.map(tgt, 1.0, np.stack([np.eye(3)] * 4))
    _, _, cost, vox = m.linearize(src, np.eye(4), np.stack([np.eye(3)]))
    e = m.voxels()["mean"][0] - src[0, :3].astype(np.float64)
    assert vox.tolist() == [0] and abs(cost - e @ e) <= 1e-6 * (e @ e)


def test_cost_derivative_is_twice_b(ref):
    """compute_error with the correspondences of T: central differences of the cost along exp(eps e_k) T approach 2 b_k (float32 terms:
    a step of 1e-3 keeps the rounding noise of the cost below the tolerance)"""
    tgt = vr.room(3000, seed=5)
    src = vr.moved(vr.room(2000, seed=6), vr.rigid(0.02, [0.1, 0.05, 0.0]))
    m = ref.map(tgt, 1.0)
    T = np.eye(4)
    _, b, _, _ = m.linearize(src, T)
    h = 1e-3
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
        assert abs((d[0] - d[1]) / (2 * h) - 2 * b[k]) <= 2e-2 * max(1.0, np.max(np.abs(b)))


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
    ok = ref.map(vr.records([[f32(2 ** 20 * res), 0, 0], [-2 ** 20 * res + 0.125, 0, 0]]), res, np.stack([np.eye(3)] * 2))
    assert ok.status == 0 and ok.voxels()["cells"][:, 0].tolist() == [-2 ** 20, 2 ** 20 - 1]
    assert ref.map(vr.records([[2 ** 20 * res + 0.25, 0, 0]]), res, np.stack([np.eye(3)])).status == 1
