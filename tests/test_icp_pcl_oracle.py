"""CPU: the sequential reference of pcl::IterativeClosestPoint (tests/icp_pcl_ref.cpp) against an independent numpy / scipy restatement,
known answers of the SVD step and the convergence criteria, and the device's step source (csrc/linalg.cuh, built for the host) against the
reference bit for bit."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

import icp_pcl_ref as ir
from gicp_pcl_ref import pose, scene, transform


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return ir.Reference(tmp_path_factory.mktemp("icp_pcl_ref"))


@pytest.fixture(scope="module")
def dev(tmp_path_factory):
    return ir.DeviceStep(tmp_path_factory.mktemp("icp_pcl_harness"))


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def sigmas():
    rng = np.random.default_rng(7)
    out = [np.zeros((3, 3)), np.eye(3), np.diag([2.0, 2.0, 1.0]), np.diag([1.0, 1.0, 1.0]) * 3, np.diag([3.0, 2.0, -1.0])]
    for k in range(400):
        A = rng.normal(size=(3, 3))
        kind = k % 6
        if kind == 1:  # rank 2
            A[:, 2] = A[:, 0] * 0.5 - A[:, 1]
        elif kind == 2:  # rank 1
            A = np.outer(rng.normal(size=3), rng.normal(size=3))
        elif kind == 3:  # det < 0
            A = A if np.linalg.det(A) < 0 else A[:, ::-1]
        elif kind == 4:  # repeated singular values
            Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
            A = Q @ np.diag([2.0, 2.0, rng.uniform(0, 2)])
        A = A * [1.0, 1e-20, 1e20, 1e-3, 1e3, 1.0][k % 6 if kind != 5 else (k // 6) % 6]
        out.append(A)
    return [np.asarray(a, np.float32) for a in out]


def test_device_step_source_equals_the_reference_bitwise(ref, dev):
    """icp_jacobi_svd3 / icp_umeyama / icp_has_converged (what k_icp_step's last block runs) == the reference's restatement of Eigen's
    JacobiSVD, pcl::umeyama and DefaultConvergenceCriteria, bit for bit, on random and degenerate sigmas"""
    rng = np.random.default_rng(3)
    for A in sigmas():
        for a, b in zip(ref.svd(A), dev.svd(A)):
            assert np.array_equal(bits(a), bits(b)), A
        sm, dm = rng.normal(size=3), rng.normal(size=3) * 100
        assert np.array_equal(bits(ref.umeyama(A, sm, dm)), bits(dev.umeyama(A, sm, dm))), A
    for T in (np.eye(4), pose((0.05, 0.0, 0.0), (0, 0, 0.01)), pose((1.0, 0.0, 0.0))):
        for it, mse, prev in ((1, 0.5, 1e300), (64, 0.5, 0.6), (3, 0.5, 0.5 + 1e-13)):
            assert ref.has_converged(T, it, 64, 0.01, mse, prev) == dev.has_converged(T, it, 64, 0.01, mse, prev)


def test_svd_is_a_decomposition(ref):
    for A in sigmas()[:200]:
        U, d, V = ref.svd(A)
        A64 = A.astype(np.float64)
        scale = max(np.abs(A64).max(), 1e-300)
        assert np.all(d[:-1] >= d[1:]) and np.all(d >= 0)
        assert np.abs(U.astype(np.float64) @ np.diag(d) @ V.T.astype(np.float64) - A64).max() <= 1e-5 * scale
        assert np.abs(U.T.astype(np.float64) @ U - np.eye(3)).max() <= 1e-5 and np.abs(V.T.astype(np.float64) @ V - np.eye(3)).max() <= 1e-5
        assert np.allclose(np.sort(d.astype(np.float64))[::-1], np.linalg.svd(A64, compute_uv=False), rtol=1e-4, atol=1e-5 * scale)


def umeyama64(src, dst):
    """pcl::umeyama in float64 with the rank-2 branch"""
    sm, dm = src.mean(0), dst.mean(0)
    sigma = (dst - dm).T @ (src - sm) / len(src)
    U, d, Vt = np.linalg.svd(sigma)
    S = np.ones(3)
    if np.linalg.det(sigma) < 0:
        S[2] = -1
    rank = int(np.sum(~(np.abs(d) <= np.abs(d[0]) * 1e-5)))
    if rank == 2:
        S[2] = 1.0 if np.linalg.det(U) * np.linalg.det(Vt) > 0 else -1.0
    R = U @ np.diag(S) @ Vt
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = dm - R @ sm
    return T


def sigma_of(src, dst):
    sm, dm = src.mean(0).astype(np.float32), dst.mean(0).astype(np.float32)
    C = (dst.astype(np.float32) - dm).astype(np.float64).T @ (src.astype(np.float32) - sm).astype(np.float64)
    return (C / len(src)).astype(np.float32), sm, dm


@pytest.mark.parametrize("case", ["general", "reflection", "planar"])
def test_umeyama_known_answers(ref, case):
    rng = np.random.default_rng(11)
    T_true = pose((0.3, -0.2, 0.1), (0.02, -0.01, 0.2)).astype(np.float64)
    src = rng.uniform(-5, 5, (200, 3))
    if case == "planar":  # every correspondence on one plane, as on ground-only scans: sigma has rank 2
        src[:, 2] = 0.0
    dst = src @ T_true[:3, :3].T + T_true[:3, 3]
    if case == "reflection":  # a mirrored target: det(sigma) < 0, the answer is still a rotation
        dst[:, 0] = -dst[:, 0]
    sigma, sm, dm = sigma_of(src, dst)
    Rt = ref.umeyama(sigma, sm, dm).astype(np.float64)
    assert abs(np.linalg.det(Rt[:3, :3]) - 1.0) <= 1e-5
    want = umeyama64(src, dst)
    assert np.abs(Rt - want).max() <= 1e-4
    if case != "reflection":
        assert np.abs(Rt - T_true).max() <= 1e-4
    if case == "planar":
        U, d, V = ref.svd(sigma)
        assert d[2] <= d[0] * 1e-5 < d[1]


def f32(x):
    return float(np.float32(x))


def test_criteria_boundaries(ref):
    """tsq == eps and cos == 1 - eps exactly in float converge, one ulp beyond does not; |d mse| < 1e-12 converges; the iteration cap
    converges (failure_after_max_iter_ is false)"""
    eps = 0.0625  # a float whose square root is exact: tsq == eps exactly
    T = np.eye(4, dtype=np.float32)
    T[0, 3] = 0.25
    assert ref.has_converged(T, 1, 64, eps, 1.0, 1e300) == (True, 1e300)
    T[0, 3] = np.nextafter(np.float32(0.25), np.float32(1))
    assert ref.has_converged(T, 1, 64, eps, 1.0, 1e300) == (False, 1.0)
    # cos == 1 - eps: t00 + t11 + t22 - 1 == 2 (1 - eps) with t11 = t22 = 1
    T = np.eye(4, dtype=np.float32)
    T[0, 0] = np.float32(1 - 2 * eps)
    assert 0.5 * float(np.float32(np.float32(T[0, 0] + T[1, 1]) + T[2, 2]) - np.float32(1)) == 1 - eps
    assert ref.has_converged(T, 1, 64, eps, 1.0, 1e300)[0]
    # one ulp of the float sum beyond: the smallest decrease of t00 that the sum ((t00 + t11) + t22) - 1 does not absorb
    cos = lambda: 0.5 * float(np.float32(np.float32(T[0, 0] + T[1, 1]) + T[2, 2]) - np.float32(1))  # noqa: E731
    while cos() == 1 - eps:
        T[0, 0] = np.nextafter(T[0, 0], np.float32(0))
    assert cos() == 1 - eps - 0.5 * 2.0 ** -22
    assert not ref.has_converged(T, 1, 64, eps, 1.0, 1e300)[0]
    far = pose((1.0, 0.0, 0.0))
    assert ref.has_converged(far, 3, 64, 0.01, 0.5, 0.5 + 0.9e-12)[0]
    assert ref.has_converged(far, 3, 64, 0.01, 0.5, 0.5 + 1.1e-12) == (False, 0.5)
    assert ref.has_converged(far, 64, 64, 0.01, 0.5, 10.0)[0] and ref.has_converged(far, 65, 64, 0.01, 0.5, 10.0)[0]


def np_correspondences(src, tgt, T, max_dist, reciprocal):
    """independent restatement: float32 transform and d2, cKDTree candidates, the (d2, index) tie rule, inclusive float64 threshold"""
    s, t = src[:, :3].astype(np.float32), tgt[:, :3].astype(np.float32)
    T = np.asarray(T, np.float32)
    q = np.empty_like(s)
    for r in range(3):
        q[:, r] = ((T[r, 0] * s[:, 0] + T[r, 1] * s[:, 1]) + T[r, 2] * s[:, 2]) + T[r, 3]

    def nn(queries, pts):
        tree = cKDTree(pts.astype(np.float64))
        lists = tree.query_ball_point(queries.astype(np.float64), max_dist * 1.001 + 1e-6)
        idx = np.full(len(queries), -1)
        dd = np.full(len(queries), np.inf, np.float32)
        for i, L in enumerate(lists):
            if not L:
                continue
            L = np.asarray(sorted(L))
            d = pts[L] - queries[i]
            d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
            k = np.lexsort((L, d2))[0]
            idx[i], dd[i] = L[k], d2[k]
        return idx, dd

    j, d2 = nn(q, t)
    ok = (j >= 0) & (d2.astype(np.float64) <= max_dist * max_dist)
    if reciprocal:
        back, bd = nn(t[np.where(ok, j, 0)], q)
        ok &= (back == np.arange(len(q))) & (bd.astype(np.float64) <= max_dist * max_dist)
    return np.where(ok, j, -1), np.where(ok, d2, np.nan).astype(np.float32), q


@pytest.mark.parametrize("reciprocal", [False, True])
def test_reference_agrees_with_an_independent_restatement(ref, reciprocal):
    tgt = scene(4096, seed=1)
    src = transform(scene(4096, seed=2), pose((0.3, -0.2, 0.05), (0.01, -0.01, 0.05)))
    src[::97] = src[::97]  # keep the layout
    src = np.vstack([src, src[:8]])  # duplicate source points: the reciprocal check keeps only the lower index
    T = pose((0.1, 0.05, 0.0), (0.0, 0.0, -0.03))
    corr, d2, cnt = ref.correspondences(src, tgt, T, 2.5, reciprocal)
    wc, wd, q = np_correspondences(src, tgt, T, 2.5, reciprocal)
    assert np.array_equal(corr, wc) and cnt == (wc >= 0).sum()
    assert np.array_equal(np.isnan(d2), np.isnan(wd)) and np.array_equal(d2[corr >= 0], wd[corr >= 0])
    if reciprocal:
        assert (corr[-8:] == -1).all() or (corr[:8] == -1).all()
    Rt, sums, _ = ref.estimate(src, tgt, T, 2.5, reciprocal)
    ok = corr >= 0
    assert sums[0] == ok.sum() and abs(sums[1] - d2[ok].astype(np.float64).sum()) <= 1e-9 * sums[1]
    assert np.abs(Rt - umeyama64(q[ok].astype(np.float64), tgt[corr[ok], :3].astype(np.float64))).max() <= 1e-5
    # the loop: per-iteration counts and the criteria restated in Python
    out = ref.align(src, tgt, T, reciprocal=reciprocal)
    cur = T.astype(np.float32)
    prev, it, counts = 1e300, 0, []
    while True:
        c, d, _ = np_correspondences(src, tgt, cur, 2.5, reciprocal)
        counts.append(int((c >= 0).sum()))
        if counts[-1] < 3:
            conv = False
            break
        _, Tinc = None, ref.estimate(src, tgt, cur, 2.5, reciprocal)[0]
        cur = (Tinc.astype(np.float64) @ cur.astype(np.float64)).astype(np.float32)
        it += 1
        mse = float(np.sum(d[c >= 0].astype(np.float64)) / counts[-1])
        if it >= 64 or (0.5 * (np.trace(Tinc[:3, :3]) - 1) >= 0.99 and float(np.sum(Tinc[:3, 3] ** 2)) <= 0.01) or abs(mse - prev) < 1e-12:
            conv = True
            break
        prev = mse
    assert out["converged"] == conv and out["iterations"] == it and list(out["counts"]) == counts
    assert np.abs(out["T"] - cur).max() <= 1e-4


def test_too_few_correspondences_and_the_identity_guess(ref):
    tgt = scene(2048, seed=5)
    src = transform(scene(2048, seed=6), pose((0.2, 0.0, 0.0)))
    out = ref.align(src, tgt, pose((500.0, 0.0, 0.0)))
    assert (out["converged"], out["iterations"], list(out["counts"])) == (False, 0, [0])
    assert np.array_equal(out["T"], pose((500.0, 0.0, 0.0)))
    # a later iteration: 3 points of which only the first iteration keeps three within 0.2 m of a lone target point set
    tiny_t = np.array([[0, 0, 0, 1], [1, 0, 0, 1], [0, 1, 0, 1]], np.float32)
    tiny_s = np.array([[0.05, 0, 0, 1], [1.05, 0, 0, 1], [0.05, 1, 0, 1]], np.float32)
    out = ref.align(tiny_s, tiny_t, max_dist=0.2)
    assert out["converged"] and out["iterations"] >= 1 and out["counts"][0] == 3
    out = ref.align(tiny_s, tiny_t[:2], max_dist=0.2)
    assert (out["converged"], out["iterations"]) == (False, 0)
    # the identity guess is a copy, a non-identity guess a float32 transform: both give the reference's own answer
    a = ref.align(src, tgt, np.eye(4, dtype=np.float32))
    b = ref.align(transform(src, np.eye(4)), tgt)
    assert np.array_equal(a["T"], b["T"]) and a["iterations"] == b["iterations"]
    # max_iterations = 1 converges after one step
    one = ref.align(src, tgt, max_iterations=1)
    assert one["converged"] and one["iterations"] == 1
