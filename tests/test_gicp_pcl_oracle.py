"""CPU: the sequential pcl GICP reference (tests/gicp_pcl_ref.cpp) against an independent numpy / scipy restatement that shares no code
with it — covariances from a brute-force k-NN, correspondences and M with np.linalg.inv, f and its gradient (the gradient also against
central differences) — and known answers: a planar patch, a far patch where PCL's raw moments part from FastGICP's, recovery of a
known transform, the line-search conditions, the too-few-correspondences path and a single BFGS step per outer iteration."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import gicp_pcl_ref as gr
from common import axis_lines, jacobisvd_diagonal_normal
from oracle import oracle as orc

EPS = 1e-3


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return gr.Reference(tmp_path_factory.mktemp("gicp_pcl_ref"))


def d2_f32(q, pts):
    d = (q[None, :3] - pts[:, :3]).astype(np.float32)
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def knn(pts, q, k):
    d2 = d2_f32(q, pts)
    order = np.lexsort((np.arange(len(pts)), d2))
    return order[:k], d2[order[:k]]


def np_covariances(pts, k=20):
    out = np.empty((len(pts), 3, 3))
    for i, q in enumerate(pts):
        idx, _ = knn(pts, q, k)
        p = pts[idx, :3].astype(np.float32)
        mean = np.zeros(3)
        raw = np.zeros((3, 3))
        for v in p:
            mean += v.astype(np.float64)
            raw += np.outer(v, v).astype(np.float32).astype(np.float64)  # each product rounded to float32
        mean /= len(p)
        C = raw / len(p) - np.outer(mean, mean)
        n = jacobisvd_diagonal_normal(C)  # tied eigenvalues of an exactly diagonal C: JacobiSVD's column, not eigh's
        if n is None:
            n = np.linalg.eigh(C)[1][:, 0]
        out[i] = np.eye(3) - (1 - EPS) * np.outer(n, n)
    return out


def xf32(T, pts):
    T = np.asarray(T, np.float32)
    p = pts[:, :3].astype(np.float32)
    return np.stack([((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3] for r in range(3)], axis=1)


def np_correspondences(src, tgt, scov, tcov, guess, T_rel, corr_dist=2.5):
    out = xf32(guess, src)
    q = xf32(T_rel, out)
    R = (np.asarray(T_rel, np.float64) @ np.asarray(guess, np.float64))[:3, :3]
    corr = np.full(len(src), -1, np.int32)
    M = np.full((len(src), 3, 3), np.nan)
    for i in range(len(src)):
        d2 = d2_f32(q[i], tgt)
        j = int(np.lexsort((np.arange(len(tgt)), d2))[0])
        if float(d2[j]) < corr_dist * corr_dist:
            corr[i] = j
            M[i] = np.linalg.inv(R @ scov[i] @ R.T + tcov[j])
    return corr, M, out


def np_cost(x, out, tgt, corr, M, f64_pose=False):
    """f(x) and the 6-gradient of OptimizationFunctorWithIndices; f64_pose: the pose in float64 (smooth, for finite differences)"""
    R = Rotation.from_euler("ZYX", [x[5], x[4], x[3]]).as_matrix()
    ok = corr >= 0
    p = out[ok].astype(np.float64)
    q = tgt[corr[ok], :3].astype(np.float64)
    if f64_pose:
        res = p @ R.T + np.asarray(x[:3]) - q
    else:
        T = np.eye(4, dtype=np.float32)
        T[:3, :3] = R.astype(np.float32)
        T[:3, 3] = np.asarray(x[:3], np.float32)
        res = (xf32(T, out[ok]) - tgt[corr[ok], :3]).astype(np.float64)
    t = np.einsum("nij,nj->ni", M[ok], res)
    m = ok.sum()
    f = np.einsum("ni,ni->", res, t) / m
    g = np.zeros(6)
    g[:3] = 2.0 / m * t.sum(0)
    dRsum = 2.0 / m * p.T @ t
    for a in range(3):  # d R / d angle by central differences of the rotation (exact to ~1e-10)
        h = 1e-6
        xp, xm = np.array(x, float), np.array(x, float)
        xp[3 + a] += h
        xm[3 + a] -= h
        dR = (Rotation.from_euler("ZYX", [xp[5], xp[4], xp[3]]).as_matrix() - Rotation.from_euler("ZYX", [xm[5], xm[4], xm[3]]).as_matrix()) / (2 * h)
        g[3 + a] = np.sum(dR * dRsum.T)
    return f, g


def small_pair(n=1500, seed=0, offset=(0, 0, 0)):
    tgt = gr.scene(n, seed=seed, offset=offset)
    src = gr.transform(gr.scene(n, seed=seed + 1, offset=offset), gr.pose((0.2, -0.1, 0.02), (0.005, -0.004, 0.03)))
    return tgt, src


def test_covariances_match_numpy(ref):
    tgt, _ = small_pair(1200, seed=2)
    for k in (20, 7):
        got = ref.covariances(tgt, k)
        assert np.max(np.abs(got - np_covariances(tgt, k))) <= 1e-8


@pytest.mark.parametrize("k", [2, 20])
def test_axis_lines_take_the_jacobisvd_normal(ref, k):
    """exactly diagonal raw-moment covariances (common.axis_lines): the restatement's diagonal branch against the reference"""
    p = axis_lines(n_per_axis=4, seed=k)
    want = np_covariances(p, k)
    assert np.max(np.abs(ref.covariances(p, k) - want)) <= 1e-12
    assert (np.abs(np.diagonal(want, axis1=1, axis2=2) - 1e-3) < 1e-12).any(axis=1).all()


def test_planar_patch_gives_the_plane_covariance(ref):
    rng = np.random.default_rng(3)
    p = np.c_[rng.uniform(-1, 1, (400, 2)), np.zeros(400), np.ones(400)].astype(np.float32)
    want = np.eye(3) - (1 - EPS) * np.outer([0, 0, 1], [0, 0, 1])
    assert np.max(np.abs(ref.covariances(p) - want)) <= 1e-12


def test_far_patch_differs_from_fastgicp(ref):
    """raw moments far from the origin cancel catastrophically: PCL's answer, not FastGICP's centred one"""
    rng = np.random.default_rng(4)
    xy = rng.uniform(-0.3, 0.3, (300, 2))
    local = np.c_[xy, 0.02 * xy[:, 0] + rng.normal(0, 0.002, 300)]
    p = np.c_[local + [3000.0, -2500.0, 40.0], np.ones(300)].astype(np.float32)
    got = ref.covariances(p)
    assert np.max(np.abs(got - np_covariances(p))) <= 1e-8
    assert np.max(np.abs(got - orc.gicp_covariances(p, 20))) > 1e-4


def test_correspondences_and_mahalanobis_match_numpy(ref):
    tgt, src = small_pair(1500, seed=5)
    scov, tcov = ref.covariances(src), ref.covariances(tgt)
    guess = gr.pose((0.05, 0.0, 0.0), (0, 0, -0.01))
    for T_rel in (np.eye(4, dtype=np.float32), gr.pose((-0.1, 0.05, 0.0), (0.0, 0.002, 0.02))):
        corr, M, cnt = ref.correspondences(src, tgt, guess, T_rel, scov=scov, tcov=tcov)
        wc, wM, _ = np_correspondences(src, tgt, scov, tcov, guess, T_rel)
        assert np.array_equal(corr, wc) and cnt == (wc >= 0).sum() > 500
        ok = wc >= 0
        assert np.max(np.abs(M[ok] - wM[ok]) / np.abs(wM[ok]).max(axis=(1, 2))[:, None, None]) <= 1e-10
        assert np.isnan(M[~ok]).all()


def test_cost_and_gradient_match_numpy_and_finite_differences(ref):
    tgt, src = small_pair(1500, seed=6)
    scov, tcov = ref.covariances(src), ref.covariances(tgt)
    guess = np.eye(4, dtype=np.float32)
    T_rel = gr.pose((-0.15, 0.08, 0.0), (0.0, 0.0, 0.02))
    corr, M, _ = ref.correspondences(src, tgt, guess, T_rel, scov=scov, tcov=tcov)
    out = xf32(guess, src)
    for x in ([-0.15, 0.08, 0.0, 0.0, 0.0, 0.02], [-0.2, 0.1, 0.01, 0.003, -0.002, 0.035]):
        f, g, m = ref.fdf(src, tgt, guess, T_rel, x, scov=scov, tcov=tcov)
        wf, wg = np_cost(x, out, tgt, corr, M)
        assert m == (corr >= 0).sum()
        assert abs(f - wf) <= 1e-9 * abs(wf)
        assert np.max(np.abs(g - wg)) <= 1e-6 * np.max(np.abs(wg))
        fd = np.zeros(6)
        for a in range(6):
            h = 1e-5
            xp, xm = np.array(x, float), np.array(x, float)
            xp[a] += h
            xm[a] -= h
            fd[a] = (np_cost(xp, out, tgt, corr, M, True)[0] - np_cost(xm, out, tgt, corr, M, True)[0]) / (2 * h)
        assert np.max(np.abs(g - fd)) <= 1e-3 * np.max(np.abs(fd))
        # the 13 cost-pass sums are the same numbers before scaling
        sums, _ = ref.cost(src, tgt, guess, T_rel, ref.apply_state(x), scov=scov, tcov=tcov)
        assert abs(sums[0] / m - f) <= 1e-12 * abs(f) and np.allclose(sums[1:4] * 2.0 / m, g[:3], rtol=1e-12, atol=0)


def test_apply_state_is_euler_zyx(ref):
    x = [0.3, -0.2, 0.1, 0.05, -0.4, 1.2]
    T = ref.apply_state(x)
    assert np.max(np.abs(T[:3, :3] - Rotation.from_euler("ZYX", [x[5], x[4], x[3]]).as_matrix())) <= 1e-6
    assert np.array_equal(T[:3, 3], np.asarray(x[:3], np.float32)) and np.array_equal(T[3], [0, 0, 0, 1])


def test_recovers_a_known_transform_and_line_search_conditions_hold(ref):
    T_true = gr.pose((0.4, -0.3, 0.05), (0.01, 0.0, 0.06))
    tgt = gr.scene(8000, seed=7)
    src = gr.transform(tgt, T_true)
    w = ref.align(src, tgt, trace=True)
    assert w["converged"] and w["iterations"] >= 1
    want = np.linalg.inv(T_true.astype(np.float64))
    assert np.max(np.abs(w["T"][:3, 3] - want[:3, 3])) <= 1e-3 and np.max(np.abs(w["T"][:3, :3] - want[:3, :3])) <= 1e-4
    tr = w["trace"]
    assert len(tr) >= w["iterations"]
    f0, fp0, alpha, fa, fpa = tr.T
    assert (fp0 < 0).all() and (alpha > 0).all()
    assert (fa <= f0 + 0.01 * alpha * fp0).all()          # sufficient decrease (rho)
    assert (np.abs(fpa) <= -0.01 * fp0).all()             # curvature (sigma)


def test_too_few_correspondences_end_the_align_unconverged(ref):
    tgt, src = small_pair(800, seed=8)
    far = gr.pose((400.0, 0.0, 0.0))
    w = ref.align(src, tgt, far)
    assert not w["converged"] and w["iterations"] == 0 and w["corr_passes"] == 1 and w["cost_passes"] == 0
    assert np.array_equal(w["T"], far)
    # three correspondences (fewer than 4) take the same exit
    few = src[:3]
    w = ref.align(few, tgt, k=3)
    assert not w["converged"] and w["iterations"] == 0


def test_one_optimizer_iteration_takes_one_bfgs_step_per_outer_iteration(ref):
    tgt, src = small_pair(1500, seed=9)
    w = ref.align(src, tgt, max_optimizer_iterations=1, max_iterations=10)
    assert w["bfgs_steps"] == w["iterations"] >= 1
    w20 = ref.align(src, tgt)
    assert w20["bfgs_steps"] > w20["iterations"]


def test_fewer_than_k_points_use_the_neighbours_found(ref):
    """engine rule for a cloud smaller than k (upstream reads past its neighbour list): the moments run over every point, divided by
    their count"""
    rng = np.random.default_rng(10)
    for n in (4, 7, 19):  # at least 4 points in general position: a unique normal
        p = np.c_[rng.uniform(-1, 1, (n, 3)), np.ones(n)].astype(np.float32)
        assert np.max(np.abs(ref.covariances(p, 20) - np_covariances(p, 20))) <= 1e-8
