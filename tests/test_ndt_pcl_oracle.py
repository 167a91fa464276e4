"""CPU: the reference of pcl::NormalDistributionsTransform (tests/ndt_pcl_ref.cpp) against an independent numpy / scipy derivation
that shares no code with it, the oracle or the engine: centroids as sequential float32 sums, radius neighbours from cKDTree with an
enlarged radius filtered by the exact float32 test, score / gradient / Hessian summed in plain float64 (gradient also by central
differences); and known answers for an invalid leaf, the strict radius and a centroid that rounds out of its own voxel."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

from ndt_pcl_ref import Reference, room, records, outside_scene

F = np.float32


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("ndt_pcl_ref"))


# ---------------------------------------------------------------------------------------------- independent derivation
def np_leaf_keys(pts, leaf):
    xyz = pts[:, :3].astype(F)
    ok = np.isfinite(xyz).all(axis=1)
    inv = F(1) / F(leaf)
    cell = np.floor(xyz[ok] * inv)
    mn = cell.min(axis=0).astype(np.int64)
    mx = cell.max(axis=0).astype(np.int64)
    div = mx - mn + 1
    ijk = (cell - mn.astype(F)).astype(np.int64)
    keys = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1]
    return np.flatnonzero(ok), keys


def np_centroids(pts, leaf):
    """leaf keys ascending and float32 centroids of the leaves of >= 6 points: sequential float32 sums in index order"""
    idx, keys = np_leaf_keys(pts, leaf)
    order = np.lexsort((idx, keys))
    ks, first, cnt = np.unique(keys[order], return_index=True, return_counts=True)
    out_k, out_c = [], []
    for k, f, c in zip(ks, first, cnt):
        if c < 6:
            continue
        members = pts[idx[order[f:f + c]], :3].astype(F)
        s = np.add.accumulate(members, axis=0, dtype=F)[-1]  # accumulate is sequential
        out_k.append(k)
        out_c.append(s / F(c))
    return np.array(out_k, np.int64), np.array(out_c, F).reshape(-1, 3)


def np_pose(p):
    """Translation * AngleAxis(x) * AngleAxis(y) * AngleAxis(z) in float32, each product rounded (no FMA)"""
    R = []
    for a in range(3):
        ang = F(p[3 + a])
        s, c = F(np.sin(np.float64(ang))), F(np.cos(np.float64(ang)))
        m = np.array([[c, 0, 0], [0, c, 0], [0, 0, c]], F)
        m[a, a] = (F(1) - c) + c
        o1, o2 = [(1, 2), (0, 2), (0, 1)][a]
        m[o1, o2], m[o2, o1] = (F(0) - s, F(0) + s) if a != 1 else (F(0) + s, F(0) - s)
        R.append(m)

    def mm(A, B):
        O = np.zeros((3, 3), F)
        for r in range(3):
            for c in range(3):
                O[r, c] = F(F(A[r, 0] * B[0, c]) + F(A[r, 1] * B[1, c])) + F(A[r, 2] * B[2, c])
        return O
    T = np.eye(4, dtype=F)
    T[:3, :3] = mm(mm(R[0], R[1]), R[2])
    T[:3, 3] = np.asarray(p[:3], np.float64).astype(F)
    return T


def np_transform(T, pts):
    x = pts[:, :3].astype(F)
    out = np.empty_like(x)
    for r in range(3):
        out[:, r] = ((T[r, 0] * x[:, 0] + T[r, 1] * x[:, 1]) + T[r, 2] * x[:, 2]) + T[r, 3]
    return out


def np_neighbours(cent, q, r):
    """per query: centroid indices with float32 ((dx*dx + dy*dy) + dz*dz) < (float)(r*r), ascending by (d2, index)"""
    r2 = F(r * r)
    tree = cKDTree(cent.astype(np.float64)) if len(cent) else None
    out = []
    for i in range(q.shape[0]):
        if tree is None or not np.isfinite(q[i]).all():
            out.append([])
            continue
        cand = np.array(tree.query_ball_point(q[i].astype(np.float64), r * 1.001), np.int64)
        if cand.size == 0:
            out.append([])
            continue
        d = q[i][None, :] - cent[cand]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        keep = d2 < r2
        cand, d2 = cand[keep], d2[keep]
        out.append(cand[np.lexsort((cand, d2))].tolist())
    return out


def np_gauss(res, outlier=0.55):
    c1 = 10 * (1 - outlier)
    c2 = outlier / res ** 3
    d3 = -np.log(c2)
    d1 = -np.log(c1 + c2) - d3
    d2 = -2 * np.log((-np.log(c1 * np.exp(-0.5) + c2) - d3) / d1)
    return d1, d2


def np_point_derivatives(x, p):
    """J (n, 3, 6) and the second derivative vectors Hv (n, 6, 6, 3) of T(p) x with respect to p (Magnusson 2009, eq. 6.19 / 6.21)"""
    cx, cy, cz = [1.0 if abs(a) < 10e-5 else np.cos(a) for a in p[3:]]
    sx, sy, sz = [0.0 if abs(a) < 10e-5 else np.sin(a) for a in p[3:]]
    X = x.astype(np.float64)
    n = X.shape[0]
    J = np.zeros((n, 3, 6))
    J[:, 0, 0] = J[:, 1, 1] = J[:, 2, 2] = 1.0
    d = lambda a, b, c: X @ np.array([a, b, c])  # noqa: E731
    J[:, 1, 3] = d(-sx * sz + cx * sy * cz, -sx * cz - cx * sy * sz, -cx * cy)
    J[:, 2, 3] = d(cx * sz + sx * sy * cz, cx * cz - sx * sy * sz, -sx * cy)
    J[:, 0, 4] = d(-sy * cz, sy * sz, cy)
    J[:, 1, 4] = d(sx * cy * cz, -sx * cy * sz, sx * sy)
    J[:, 2, 4] = d(-cx * cy * cz, cx * cy * sz, -cx * sy)
    J[:, 0, 5] = d(-cy * sz, -cy * cz, 0)
    J[:, 1, 5] = d(cx * cz - sx * sy * sz, -cx * sz - sx * sy * cz, 0)
    J[:, 2, 5] = d(sx * cz + cx * sy * sz, cx * sy * cz - sx * sz, 0)
    Z = np.zeros(n)
    a = np.c_[Z, d(-cx * sz - sx * sy * cz, -cx * cz + sx * sy * sz, sx * cy), d(-sx * sz + cx * sy * cz, -cx * sy * sz - sx * cz, -cx * cy)]
    b = np.c_[Z, d(cx * cy * cz, -cx * cy * sz, cx * sy), d(sx * cy * cz, -sx * cy * sz, sx * sy)]
    c = np.c_[Z, d(-sx * cz - cx * sy * sz, sx * sz - cx * sy * cz, 0), d(cx * cz - sx * sy * sz, -sx * sy * cz - cx * sz, 0)]
    dd = np.c_[d(-cy * cz, cy * sz, sy), d(-sx * sy * cz, sx * sy * sz, sx * cy), d(cx * sy * cz, -cx * sy * sz, -cx * cy)]
    e = np.c_[d(sy * sz, sy * cz, 0), d(-sx * cy * sz, -sx * cy * cz, 0), d(cx * cy * sz, cx * cy * cz, 0)]
    f = np.c_[d(-cy * cz, cy * sz, 0), d(-cx * sz - sx * sy * cz, -cx * cz + sx * sy * sz, 0), d(-sx * sz + cx * sy * cz, -cx * sy * sz - sx * cz, 0)]
    Hv = np.zeros((n, 6, 6, 3))
    for (i, j), v in {(3, 3): a, (3, 4): b, (4, 3): b, (3, 5): c, (5, 3): c, (4, 4): dd, (4, 5): e, (5, 4): e, (5, 5): f}.items():
        Hv[:, i, j] = v
    return J, Hv


class NpMap:
    """the independent pcl NDT target: the oracle's voxel Gaussians (by key) plus the numpy centroids"""

    def __init__(self, tgt, res, voxels):
        self.res = res
        self.keys, self.cent = np_centroids(tgt, res)
        slot = {int(k): i for i, k in enumerate(voxels["keys"])}
        s = np.array([slot[int(k)] for k in self.keys], np.int64)
        self.mean, self.icov = voxels["mean"][s], voxels["icov"][s]

    def terms(self, src, p, xt=None):
        """score, g, H summed over every (point, neighbour) pair (neighbours found at the float32 transform)"""
        q = np_transform(np_pose(p), src) if xt is None else xt
        nb = np_neighbours(self.cent, q, self.res)
        pi = np.repeat(np.arange(src.shape[0]), [len(v) for v in nb])
        ci = np.array([c for v in nb for c in v], np.int64)
        d1, d2 = np_gauss(self.res)
        J, Hv = np_point_derivatives(src[pi, :3], p)
        xq = q[pi].astype(np.float64) - self.mean[ci]
        C = self.icov[ci]
        e = np.exp(-d2 * np.einsum("ni,nij,nj->n", xq, C, xq) / 2)
        ok = (d2 * e <= 1) & (d2 * e >= 0)
        w = d1 * d2 * e
        xC = np.einsum("ni,nij->nj", xq, C)
        gq = np.einsum("nj,njk->nk", xC, J)
        score = np.sum(np.where(ok, -d1 * e, 0.0))
        g = np.sum(np.where(ok[:, None], gq * w[:, None], 0.0), axis=0)
        H = (-d2 * gq[:, :, None] * gq[:, None, :] + np.einsum("nj,nabj->nab", xC, Hv) + np.einsum("nja,njk,nkb->nba", J, C, J))
        H = np.sum(np.where(ok[:, None, None], H * w[:, None, None], 0.0), axis=0)
        return score, g, H, nb

    def score64(self, src, p, pairs):
        """the score with a float64 transform over fixed (point, centroid) pairs: what central differences differentiate"""
        T = np.eye(4)
        cx, cy, cz = np.cos(p[3:]); sx, sy, sz = np.sin(p[3:])
        T[:3, :3] = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) @ np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
        T[:3, 3] = p[:3]
        pi, ci = pairs
        x = src[pi, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3] - self.mean[ci]
        d1, d2 = np_gauss(self.res)
        return np.sum(-d1 * np.exp(-d2 * np.einsum("ni,nij,nj->n", x, self.icov[ci], x) / 2))


def rel(a, b):
    return np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(np.asarray(b))), 1e-300)


POSES = [np.zeros(6), np.array([0.1, -0.05, 0.02, 0.01, -0.02, 0.03]), np.array([0.3, 0.2, -0.1, 0.15, -0.1, 0.5])]


@pytest.mark.parametrize("res", [0.5, 1.0])
def test_reference_equals_independent_derivation(ref, res):
    tgt, src = room(12000, 1), room(6000, 2)
    M = ref.map(tgt, res)
    N = NpMap(tgt, res, M.voxels)
    k, c = M.centroids()
    assert k.size > 50 and np.array_equal(k, N.keys) and np.array_equal(c.view(np.uint32), N.cent.view(np.uint32))
    for p in POSES:
        score, g, H, nb = N.terms(src, p)
        cnt, keys = M.neighbors(src, p)
        assert np.array_equal(cnt, [len(v) for v in nb])
        assert np.array_equal(keys, np.concatenate([np.sort(N.keys[v]) for v in nb if v] or [np.zeros(0, np.int64)]))
        o = M.derivatives(src, p)
        assert o["n_pairs"] == cnt.sum() > 0
        assert abs(o["score"] - score) <= 1e-9 * abs(score) and rel(o["g"], g) <= 1e-9 and rel(o["H"], H) <= 1e-9


def test_gradient_is_the_derivative_of_the_score(ref):
    tgt, src = room(12000, 3), room(3000, 4)
    res = 1.0
    M = ref.map(tgt, res)
    N = NpMap(tgt, res, M.voxels)
    p = POSES[1]
    _, g, _, nb = N.terms(src, p)
    pairs = (np.repeat(np.arange(src.shape[0]), [len(v) for v in nb]), np.array([c for v in nb for c in v], np.int64))
    h = 1e-6
    fd = np.array([(N.score64(src, p + h * np.eye(6)[i], pairs) - N.score64(src, p - h * np.eye(6)[i], pairs)) / (2 * h) for i in range(6)])
    assert rel(g, fd) < 1e-3


def test_invalid_leaf_adds_minus_d1_per_point(ref):
    """a voxel of identical points has a zero covariance: invalidated (nr_points = -1), inverse still zero, but its centroid was emitted
    and stays searchable: every source point within r adds exactly -d1 and nothing to g or H"""
    tgt = records(np.tile([[0.25, 0.25, 0.25]], (8, 1)))
    src = records(np.array([[0.3, 0.2, 0.25], [0.6, 0.6, 0.6], [1.5, 0.25, 0.25], [0.25, 0.25, 1.2], [5.0, 5.0, 5.0]]))
    M = ref.map(tgt, 1.0)
    assert M.voxels["npts"].tolist() == [-1] and not M.voxels["icov"].any()
    k, c = M.centroids()
    assert k.tolist() == [0] and c.tolist() == [[0.25, 0.25, 0.25]]
    cnt, _ = M.neighbors(src, np.zeros(6))
    assert cnt.tolist() == [1, 1, 0, 1, 0]
    d1, _ = np_gauss(1.0)
    o = M.derivatives(src, np.zeros(6))
    assert o["score"] == -d1 + -d1 + -d1 and not o["g"].any() and not o["H"].any()


def test_radius_is_strict_to_the_ulp(ref):
    """a centroid at (0.5, 0.5, 0.5): a query at exactly distance r = 1 is not a neighbour, one float32 ulp closer is"""
    tgt = records(np.tile([[0.5, 0.5, 0.5]], (6, 1)))
    inside = np.nextafter(F(1.5), F(0))
    src = records(np.array([[1.5, 0.5, 0.5], [inside, 0.5, 0.5], [0.5, -0.5, 0.5], [0.5, 0.5, inside]], F))
    M = ref.map(tgt, 1.0)
    assert M.centroids()[1].tolist() == [[0.5, 0.5, 0.5]]
    cnt, _ = M.neighbors(src, np.zeros(6))
    assert cnt.tolist() == [0, 1, 0, 1]
    N = NpMap(tgt, 1.0, M.voxels)
    assert [len(v) for v in np_neighbours(N.cent, src[:, :3], 1.0)] == [0, 1, 0, 1]


def test_centroid_outside_its_voxel_is_found(ref):
    tgt, q, (x, n, k) = outside_scene(0.1)
    M = ref.map(tgt, 0.1)
    N = NpMap(tgt, 0.1, M.voxels)
    inv = F(1) / F(0.1)
    assert np.floor(x * inv) == k - 1
    i = np.flatnonzero(np.abs(N.cent[:, 0] - F(k * 0.1)) < 1e-6)
    assert i.size >= 1 and (np.floor(N.cent[i, 0] * inv) == k).any()  # the centroid lies in the next cell
    cnt, keys = M.neighbors(q, np.zeros(6))
    nb = np_neighbours(N.cent, q[:, :3], 0.1)
    assert np.array_equal(cnt, [len(v) for v in nb]) and cnt.sum() > 0
    assert np.array_equal(keys, np.concatenate([np.sort(N.keys[v]) for v in nb if v]))
