"""CPU: the reference of NDT_OMP's KDTREE search (tests/ndt_kdtree_ref.cpp) against an independent numpy / scipy restatement that shares
no code with it, the oracle or the engine: centroids as sequential float32 sums, radius neighbours from cKDTree with an enlarged radius
filtered by the exact float32 test, ndt_omp's term written in numpy float32 (every operation rounded, no FMA), the float64 Hessian of
the Hessian-only pass, g against central differences, a known transform recovered; and known answers for an invalidated leaf.  The
neighbour lists are also those of the pcl NDT reference, and the oracle's own entry points compiled into the same library are
unchanged."""
import numpy as np
import pytest

from oracle import oracle as orc
import ndt_pcl_ref
from ndt_kdtree_ref import Reference
from ndt_pcl_ref import room, records
from test_ndt_pcl_oracle import NpMap, np_gauss, np_neighbours, np_point_derivatives, np_pose, np_transform, rel

F = np.float32
POSES = [np.zeros(6), np.array([0.1, -0.05, 0.02, 0.01, -0.02, 0.03]), np.array([0.3, 0.2, -0.1, 0.15, -0.1, 0.5])]


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("ndt_kdtree_ref"))


@pytest.fixture(scope="module")
def pcl(tmp_path_factory):
    return ndt_pcl_ref.Reference(tmp_path_factory.mktemp("ndt_pcl_ref"))


def f32_dot(a, x):
    """((a0 x + a1 y) + a2 z) in float32, each product and sum rounded"""
    return (F(a[0]) * x[:, 0] + F(a[1]) * x[:, 1]) + F(a[2]) * x[:, 2]


def omp_terms(N, src, p):
    """ndt_omp's float32 updateDerivatives over every (point, radius neighbour) pair: score, g, H, summed per point in neighbour order
    and over the points in index order (float64)"""
    q32 = np_transform(np_pose(p), src)
    nb = np_neighbours(N.cent, q32, N.res)
    d1, d2 = np_gauss(N.res)
    d2f = F(d2)
    Je, He = np_point_derivatives(np.eye(3), p)  # row k: the coefficients of x_k, i.e. the j_ang / h_ang rows
    x = src[:, :3].astype(F)
    J = np.zeros((src.shape[0], 3, 6), F)
    J[:, 0, 0] = J[:, 1, 1] = J[:, 2, 2] = F(1)
    for r in range(3):
        for c in range(3, 6):
            J[:, r, c] = f32_dot(Je[:, r, c], x)
    PH = np.zeros((src.shape[0], 6, 6, 3), F)
    for i in range(3, 6):
        for j in range(3, 6):
            for r in range(3):
                PH[:, i, j, r] = f32_dot(He[:, i, j, r], x)
    score, g, H = 0.0, np.zeros(6), np.zeros((6, 6))
    for i, v in enumerate(nb):
        if not v:
            continue
        ci = np.array(v, np.int64)
        qv = (q32[i].astype(np.float64)[None, :] - N.mean[ci]).astype(F)
        C = N.icov[ci].astype(F)
        qC = np.stack([(qv[:, 0] * C[:, 0, j] + qv[:, 1] * C[:, 1, j]) + qv[:, 2] * C[:, 2, j] for j in range(3)], 1)
        qCq = (qv[:, 0] * qC[:, 0] + qv[:, 1] * qC[:, 1]) + qv[:, 2] * qC[:, 2]
        e = np.exp(((-d2f) * qCq * F(0.5)).astype(np.float64)).astype(F)
        s_inc = (-d1 * e.astype(np.float64)).astype(F)
        e = d2f * e
        ok = ~((e > 1) | (e < 0) | (e != e))
        e = (e.astype(np.float64) * d1).astype(F)
        Ji = J[i]
        CJ = np.stack([np.stack([(C[:, r, 0] * Ji[0, c] + C[:, r, 1] * Ji[1, c]) + C[:, r, 2] * Ji[2, c] for c in range(6)], 1) for r in range(3)], 1)
        gq = np.stack([(qv[:, 0] * CJ[:, 0, c] + qv[:, 1] * CJ[:, 1, c]) + qv[:, 2] * CJ[:, 2, c] for c in range(6)], 1)
        sp, gp, Hp = 0.0, np.zeros(6), np.zeros((6, 6))
        for t in range(len(v)):  # neighbour order, as the per-point accumulation
            if not ok[t]:
                continue
            sp += float(s_inc[t])
            gp += (e[t] * gq[t]).astype(np.float64)
            for a in range(6):
                for b in range(6):
                    xh = F(0)
                    if a >= 3 and b >= 3:
                        xh = (qC[t, 0] * PH[i, a, b, 0] + qC[t, 1] * PH[i, a, b, 1]) + qC[t, 2] * PH[i, a, b, 2]
                    P = (Ji[0, b] * CJ[t, 0, a] + Ji[1, b] * CJ[t, 1, a]) + Ji[2, b] * CJ[t, 2, a]
                    u = (((-d2f) * gq[t, a]) * gq[t, b] + xh) + P
                    Hp[a, b] += float(e[t] * u)
        score += sp
        g += gp
        H += Hp
    return score, g, H, nb


def test_reference_equals_independent_derivation(ref):
    res = 1.0
    tgt, src = room(12000, 1), room(1500, 2)
    M = ref.map(tgt, res)
    N = NpMap(tgt, res, M.voxels())
    k, c = M.centroids()
    assert k.size > 50 and np.array_equal(k, N.keys) and np.array_equal(c.view(np.uint32), N.cent.view(np.uint32))
    for p in POSES:
        score, g, H, nb = omp_terms(N, src, p)
        cnt, keys = M.neighbors(src, p)
        assert np.array_equal(cnt, [len(v) for v in nb])
        assert np.array_equal(keys, np.concatenate([np.sort(N.keys[v]) for v in nb if v] or [np.zeros(0, np.int64)]))
        o = M.derivatives(src, p)
        assert o["n_pairs"] == cnt.sum() > 0
        assert abs(o["score"] - score) <= 1e-9 * abs(score) and rel(o["g"], g) <= 1e-9 and rel(o["H"], H) <= 1e-9
        # the Hessian-only pass: the float64 updateHessian over the same neighbours
        _, _, H64, _ = N.terms(src, p)
        assert rel(M.hessian_at(src, p), H64) <= 1e-9


def test_neighbours_and_centroids_are_pcl_ndts(ref, pcl):
    tgt, src = room(16000, 5), room(4000, 6)
    for res in (0.5, 0.7, 1.0):
        M, P = ref.map(tgt, res), pcl.map(tgt, res)
        ka, ca = M.centroids()
        kb, cb = P.centroids()
        assert np.array_equal(ka, kb) and np.array_equal(ca.view(np.uint32), cb.view(np.uint32))
        for p in POSES:
            a, b = M.neighbors(src, p), P.neighbors(src, p)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
            assert M.derivatives(src, p)["n_pairs"] == P.derivatives(src, p)["n_pairs"] == a[0].sum()


def test_gradient_is_the_derivative_of_the_score(ref):
    tgt, src = room(12000, 3), room(3000, 4)
    res = 1.0
    M = ref.map(tgt, res)
    N = NpMap(tgt, res, M.voxels())
    p = POSES[1]
    nb = np_neighbours(N.cent, np_transform(np_pose(p), src), res)
    pairs = (np.repeat(np.arange(src.shape[0]), [len(v) for v in nb]), np.array([c for v in nb for c in v], np.int64))
    h = 1e-6
    fd = np.array([(N.score64(src, p + h * np.eye(6)[i], pairs) - N.score64(src, p - h * np.eye(6)[i], pairs)) / (2 * h) for i in range(6)])
    assert rel(M.derivatives(src, p)["g"], fd) < 1e-3


def test_known_transform_is_recovered(ref):
    tgt = room(20000, 7)
    truth = np.array([0.15, -0.1, 0.05, 0.01, -0.015, 0.04])
    T = np_pose(truth).astype(np.float64)
    Ti = np.linalg.inv(T)
    src = records((tgt[::3, :3].astype(np.float64) @ Ti[:3, :3].T + Ti[:3, 3]).astype(F))
    M = ref.map(tgt, 1.0)
    out = M.align(src)
    assert out["converged"]
    assert np.max(np.abs(out["p"][:3] - truth[:3])) < 0.02 and np.max(np.abs(out["p"][3:] - truth[3:])) < 0.01
    # with the active line search as well
    out1 = M.align(src, mt_interval_flag=1)
    assert np.max(np.abs(out1["p"][:3] - truth[:3])) < 0.02 and np.max(np.abs(out1["p"][3:] - truth[3:])) < 0.01
    assert out1["hessian_passes"] >= 0


def test_invalidated_leaf_adds_minus_d1_only(ref):
    """a voxel of identical points is invalidated (nr_points = -1) with a zero inverse, but its centroid was emitted: every source point
    within r adds the float32 -d1 and nothing to g or H, where DIRECT7 skips the leaf"""
    tgt = records(np.tile([[0.25, 0.25, 0.25]], (8, 1)))
    src = records(np.array([[0.3, 0.2, 0.25], [0.6, 0.6, 0.6], [1.5, 0.25, 0.25], [0.25, 0.25, 1.2], [5.0, 5.0, 5.0]]))
    M = ref.map(tgt, 1.0)
    v = M.voxels()
    assert v["npts"].tolist() == [-1] and not v["icov"].any()
    cnt, _ = M.neighbors(src, np.zeros(6))
    assert cnt.tolist() == [1, 1, 0, 1, 0]
    d1, _ = np_gauss(1.0)
    s1 = float(F(-d1))
    o = M.derivatives(src, np.zeros(6))
    assert o["score"] == (s1 + s1) + s1 and not o["g"].any() and not o["H"].any() and o["n_pairs"] == 3
    assert not M.hessian_at(src, np.zeros(6)).any()
    d7 = orc.NdtMap(tgt, 1.0).derivatives(src, np.zeros(6))
    assert d7["score"] == 0.0 and d7["n_pairs"] == 0


def test_oracle_entry_points_in_the_library_are_unchanged(ref):
    """with no KDTREE entry point running, the oracle's own passes compiled into the reference library are liboracle's, bit for bit"""
    import ctypes as C
    tgt, src = room(12000, 8), room(3000, 9)
    om = orc.NdtMap(tgt, 1.0)
    M = ref.map(tgt, 1.0)
    L = ref.lib
    L.orc_ndt_derivatives.restype = C.c_double
    for p in POSES:
        a = om.derivatives(src, p)
        s = np.ascontiguousarray(src, F)
        cfg = om._cfg()
        g, H, npairs = np.empty(6), np.empty((6, 6)), C.c_uint64()
        score = L.orc_ndt_derivatives(C.c_void_p(L.ref_kd_voxels(M._m)), C.c_void_p(s.ctypes.data), C.c_size_t(s.shape[0]), C.c_size_t(s.shape[1]),
                                      C.byref(cfg), C.c_void_p(np.ascontiguousarray(p).ctypes.data), C.c_void_p(g.ctypes.data),
                                      C.c_void_p(H.ctypes.data), C.byref(npairs), None)
        assert score == a["score"] and np.array_equal(g, a["g"]) and np.array_equal(H, a["H"]) and npairs.value == a["n_pairs"]
