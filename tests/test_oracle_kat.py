"""Known-answer tests that pin the CPU oracle (CPU only).  The reference ships no tests or golden vectors for this path
("parity unpinned", SURVEY.md §0.2/§8c), so the oracle is pinned against analytic ground truth, brute force and numpy
re-derivations of the published formulas, plus the frozen fixtures of tests/golden/ (see gen_golden.py)."""
import numpy as np
import pytest
from common import rot_err, trans_err, perturb


def brute_knn(pts, q, k):
    d = (q[:, None, 0] - pts[None, :, 0]) ** 2
    d = (d + (q[:, None, 1] - pts[None, :, 1]) ** 2).astype(np.float32)
    d = (d + (q[:, None, 2] - pts[None, :, 2]) ** 2).astype(np.float32)
    idx = np.lexsort((np.broadcast_to(np.arange(pts.shape[0]), d.shape), d), axis=1)[:, :k]
    return idx.astype(np.int32), np.take_along_axis(d, idx, 1)


def test_knn_exact_vs_bruteforce(oracle):
    rng = np.random.default_rng(0)
    pts = rng.normal(size=(700, 4)).astype(np.float32)
    q = rng.normal(size=(200, 4)).astype(np.float32)
    for k in (1, 5, 20):
        idx, d2 = oracle.knn(pts, q, k)
        bi, bd = brute_knn(pts, q, k)
        assert np.array_equal(idx, bi) and np.array_equal(d2, bd)


def test_knn_ties_go_to_lowest_index(oracle):
    g = np.array([[x, y, z, 1] for x in range(6) for y in range(6) for z in range(3)], np.float32)
    pts = np.concatenate([g, g])  # every point duplicated: ties everywhere
    q = g[::5] + np.array([0.5, 0.5, 0.0, 0], np.float32)  # equidistant from 4 lattice points
    idx, d2 = oracle.knn(pts, q, 8)
    bi, bd = brute_knn(pts, q, 8)
    assert np.array_equal(idx, bi) and np.array_equal(d2, bd)
    assert np.all(idx[:, 0] < g.shape[0])


def test_gicp_covariance_plane_regularisation(oracle):
    rng = np.random.default_rng(1)
    pts = np.zeros((400, 4), np.float32)
    pts[:, :2] = rng.uniform(-1, 1, (400, 2))
    pts[:, 2] = 0.3 * pts[:, 0] + rng.normal(0, 1e-3, 400)  # tilted plane z = 0.3 x
    cov = oracle.gicp_covariances(pts, 20)
    n = np.array([-0.3, 0, 1]) / np.linalg.norm([-0.3, 0, 1])
    w, V = np.linalg.eigh(cov)
    assert np.allclose(w, [1e-3, 1, 1], atol=1e-12)          # PLANE: singular values replaced by (1, 1, 1e-3)
    assert np.min(np.abs(V[:, :, 0] @ n)) > 0.99              # smallest axis = plane normal
    assert np.max(np.abs(cov - np.transpose(cov, (0, 2, 1)))) < 1e-15


def test_gicp_linearize_against_numpy(oracle, synth):
    tgt = synth.scan("vlp16_16k", frame=0)[::8].copy()
    src = synth.scan("vlp16_16k", frame=1)[::8].copy()
    sc, tc = oracle.gicp_covariances(src, 20), oracle.gicp_covariances(tgt, 20)
    T = perturb(3, 0.2, 1.0)
    o = oracle.gicp_linearize(src, sc, tgt, tc, T, 2.5)
    Tf = T.astype(np.float32)
    q = (Tf[:3, 0] * src[:, 0:1] + Tf[:3, 1] * src[:, 1:2]).astype(np.float32)
    q = ((q + Tf[:3, 2] * src[:, 2:3]).astype(np.float32) + Tf[:3, 3]).astype(np.float32)
    bi, bd = brute_knn(tgt, q, 1)
    corr = np.where(bd[:, 0].astype(np.float64) < 6.25, bi[:, 0], -1)
    assert np.array_equal(o["corr"], corr)
    H = np.zeros((6, 6)); b = np.zeros(6); e = 0.0
    R = T[:3, :3]
    for i in np.nonzero(corr >= 0)[0]:
        M = np.linalg.inv(tc[corr[i]] + R @ sc[i] @ R.T)
        ta = R @ src[i, :3].astype(np.float64) + T[:3, 3]
        err = tgt[corr[i], :3].astype(np.float64) - ta
        S = np.array([[0, -ta[2], ta[1]], [ta[2], 0, -ta[0]], [-ta[1], ta[0], 0]])
        J = np.hstack([S, -np.eye(3)])
        H += J.T @ M @ J; b += J.T @ M @ err; e += err @ M @ err
    assert np.allclose(o["H"], H, rtol=1e-10, atol=1e-8) and np.allclose(o["b"], b, rtol=1e-10, atol=1e-8) and abs(o["err"] - e) < 1e-9 * e
    assert abs(oracle.gicp_error(src, tgt, o["corr"], o["mahal"], T) - e) < 1e-9 * e


def test_gicp_align_recovers_known_transform(oracle):
    rng = np.random.default_rng(2)
    # three noisy orthogonal planes (a room corner): fully constrained
    a = rng.uniform(0, 4, (1500, 2))
    planes = [np.c_[a[:500], np.zeros(500)], np.c_[a[500:1000, 0], np.zeros(500), a[500:1000, 1]], np.c_[np.zeros(500), a[1000:]]]
    tgt = np.concatenate(planes) + rng.normal(0, 0.002, (1500, 3))
    Ttrue = perturb(5, 0.15, 3.0)
    src = (np.linalg.inv(Ttrue)[:3, :3] @ tgt.T).T + np.linalg.inv(Ttrue)[:3, 3]
    pad = lambda x: np.c_[x, np.ones(len(x))].astype(np.float32)
    r = oracle.gicp_align(pad(src), pad(tgt), np.eye(4))
    assert r["converged"] and 1 <= r["iterations"] <= 64 and not r["lm_failed"]
    assert trans_err(r["T"], Ttrue) < 2e-3 and rot_err(r["T"], Ttrue) < 2e-3
    # identical clouds + identity guess => identity, converged after the first step
    r0 = oracle.gicp_align(pad(tgt), pad(tgt), np.eye(4))
    assert r0["converged"] and trans_err(r0["T"], np.eye(4)) < 1e-6 and rot_err(r0["T"], np.eye(4)) < 1e-6
    # empty input: initCompute fails silently, converged stays false
    assert not oracle.gicp_align(np.zeros((0, 4), np.float32), pad(tgt))["converged"]


def test_fitness_semantics(oracle):
    tgt = np.array([[0, 0, 0, 1], [1, 0, 0, 1], [5, 0, 0, 1]], np.float32)
    src = np.array([[0.1, 0, 0, 1], [1.0, 0.3, 0, 1], [3.0, 0, 0, 1]], np.float32)
    score, nr, inl = oracle.fitness(tgt, src, np.eye(4))
    d2 = np.array([np.float32(0.1) ** 2, np.float32(0.3) ** 2, 4.0], np.float64)
    assert nr == 3 and inl == 2 and abs(score - d2.astype(np.float32).astype(np.float64).mean()) < 1e-12
    # max_range is compared against the SQUARED distance (information_matrix_calculator.cpp:69)
    score, nr, inl = oracle.fitness(tgt, src, np.eye(4), max_range=0.05)
    assert nr == 1 and abs(score - np.float64(np.float32(0.1) * np.float32(0.1))) < 1e-12
    score, nr, _ = oracle.fitness(tgt, src, np.eye(4), max_range=1e-9)
    assert nr == 0 and score == np.finfo(np.float64).max


def test_voxelgrid_hand_computed(oracle):
    pts = np.array([[0.01, 0.02, 0.03, 1, 10, 0, 0, 0], [0.04, 0.05, 0.06, 1, 20, 0, 0, 0], [0.51, 0.0, 0.0, 1, 7, 0, 0, 0],
                    [-0.2, 0.0, 0.0, 1, 1, 0, 0, 0]], np.float32)
    out, keys, counts, rc = oracle.voxelgrid(pts, 0.5)
    # min_b.x = floor(-0.2/0.5) = -1  => keys: (-0.2)->0, (0.01,0.04)->1, (0.51)->2
    assert rc == 0 and list(keys) == [0, 1, 2] and list(counts) == [1, 2, 1]
    assert np.allclose(out[1], [0.025, 0.035, 0.045, 15.0]) and np.allclose(out[0], [-0.2, 0, 0, 1]) and np.allclose(out[2], [0.51, 0, 0, 7])


def test_ndt_voxel_gaussian_formula(oracle):
    rng = np.random.default_rng(3)
    pts = np.zeros((60, 4), np.float32)
    pts[:40, :3] = rng.uniform(0.05, 0.95, (40, 3))                      # voxel (0,0,0): 40 pts, full rank
    pts[40:45, :3] = rng.uniform(1.05, 1.95, (5, 3))                     # voxel (1,1,1): 5 pts -> below min_points (6)
    pts[45:, :3] = np.c_[rng.uniform(2.05, 2.95, (15, 2)), np.full(15, 0.5) + rng.normal(0, 1e-4, 15)]  # flat voxel -> eigen clamp
    m = oracle.NdtMap(pts, 1.0).dump()
    # keys ascending: (0,0,0)->0, (2,2,0)->8, (1,1,1)->13
    assert list(m["keys"]) == [0, 8, 13] and list(m["npts"]) == [40, 15, 5] and list(m["div_b"]) == [3, 3, 2]
    p = pts[:40, :3].astype(np.float64)
    mean = p.mean(0)
    cov = (p.T @ p - 2 * np.outer(p.sum(0), mean)) / 40 + np.outer(mean, mean)
    cov *= 39.0 / 40.0                                                     # PCL's (n-1)/n factor
    assert np.allclose(m["mean"][0], mean, atol=1e-15) and np.allclose(m["cov"][0], cov, atol=1e-14)
    assert np.allclose(m["icov"][0] @ m["cov"][0], np.eye(3), atol=1e-9)
    w = np.linalg.eigvalsh(m["cov"][1])
    assert abs(w[0] / w[2] - 0.01) < 1e-9                                  # smallest eigenvalue clamped to 0.01 * largest


def test_ndt_gradient_is_consistent_with_score(oracle, synth):
    tgt = synth.scan("vlp16_16k", frame=0)
    src = synth.scan("vlp16_16k", frame=1)[::4].copy()
    m = oracle.NdtMap(tgt, 1.0)
    p0 = np.array([0.9, 0.02, -0.01, 0.004, -0.003, 0.02])
    o = m.derivatives(src, p0)
    assert o["score"] > 0 and o["n_pairs"] > src.shape[0]  # gauss_d1 < 0: the score is a likelihood, maximised
    # the float32 per-point math limits finite differences to ~1e-3 relative; direction and magnitude must agree
    for k, h in ((0, 2e-3), (1, 2e-3), (5, 1e-3)):
        d = np.zeros(6); d[k] = h
        num = (m.derivatives(src, p0 + d)["score"] - m.derivatives(src, p0 - d)["score"]) / (2 * h)
        assert abs(num - o["g"][k]) < 0.10 * abs(o["g"][k]) + 2e-2 * np.linalg.norm(o["g"])
    assert np.allclose(o["H"], o["H"].T, rtol=1e-4, atol=1e-3 * np.abs(o["H"]).max())


def test_ndt_align_on_synthetic_pair(oracle, synth):
    tgt = synth.scan("vlp16_16k", frame=0)
    src = synth.scan("vlp16_16k", frame=1)
    gt = np.linalg.inv(synth.pose_matrix(0)) @ synth.pose_matrix(1)
    m = oracle.NdtMap(tgt, 1.0)
    # NDT is a local method (and the sensor-centred ground rings reward "no translation"): like the reference's odometry,
    # which seeds align() with the previous motion (scan_matching_odometry_nodelet.cpp:210), start near the truth.
    r = m.align(src, gt.astype(np.float32), search_method=7)
    assert r["converged"] and r["iterations"] >= 1
    assert trans_err(r["T"], gt) < 0.1 and rot_err(r["T"], gt) < 0.02
    # ndt_omp polarity: exactly one derivative pass per iteration (+ the initial one)
    assert r["derivative_passes"] == r["iterations"] + 1
    r30 = m.align(src, gt.astype(np.float32), fixed_iterations=30)
    assert r30["iterations"] == 30 and trans_err(r30["T"], gt) < 0.1
    rmt = m.align(src, (gt @ perturb(2, 0.2, 1.0)).astype(np.float32), mt_interval_flag=1)
    assert rmt["converged"] and trans_err(rmt["T"], gt) < 0.1 and rmt["derivative_passes"] > rmt["iterations"] + 1
    # identical clouds, identity guess: stays at identity
    rid = m.align(tgt, np.eye(4, dtype=np.float32))
    assert rid["converged"] and trans_err(rid["T"], np.eye(4)) < 1e-3


def test_voxelgrid_leaf_too_small_when_the_grid_volume_overflows_int64(oracle):
    """pcl::VoxelGrid's "leaf size is too small" guard on a grid of ~3e6 leaves per axis: the volume (~2.8e19) does not fit in
    int64, so a product formed in one go would wrap and let the grid through; the guard must still fire and pass the input on"""
    c = np.array([[-60.0, -20.0, -2.0, 1.0, 5.0, 0, 0, 0], [3000.0, 3000.0, 3000.0, 1.0, 7.0, 0, 0, 0]], np.float32)
    out, keys, counts, rc = oracle.voxelgrid(c, 0.001)
    assert rc == 1 and np.array_equal(out[:, :3], c[:, :3]) and np.array_equal(out[:, 3], c[:, 4])
    assert np.all(keys == -1) and np.all(counts == 1)
