"""CPU: the sequential pclomp GICP reference (tests/gicp_omp_ref.cpp) against an independent numpy / scipy restatement of pclomp's
functor and its pose composition applyState(guess, x), against the pcl GICP reference it is built from (the identity that maps one
functor onto the other, and the whole align at an identity guess), and the known consequence of the pose rule: with a translated
guess the two methods end at different poses."""
import numpy as np
import pytest

import gicp_omp_ref as gor
import gicp_pcl_ref as gr
from test_gicp_pcl_oracle import np_correspondences, xf32


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return gor.Reference(tmp_path_factory.mktemp("gicp_omp_ref"))


@pytest.fixture(scope="module")
def gicp(tmp_path_factory):
    return gr.Reference(tmp_path_factory.mktemp("gicp_pcl_ref_for_omp"))


GUESSES = [np.eye(4, dtype=np.float32), gr.pose((0, 0, 0), (0.01, -0.02, 0.05)), gr.pose((3.0, -2.0, 0.4), (0.0, 0.01, 0.04))]
XS = [[0.0, 0.0, 0.0, 0.0, 0.0, 0.0], [-0.1, 0.05, 0.01, 0.002, -0.003, 0.02], [0.2, -0.15, 0.0, -0.004, 0.001, -0.03]]


def np_pose(A, guess):
    """applyState(guess, x) in numpy float32, from A = applyState(I, x): [R(x) R_g | t_g + t(x)], ((a0 b0 + a1 b1) + a2 b2) unfused"""
    A, G = np.asarray(A, np.float32), np.asarray(guess, np.float32)
    T = G.copy()
    for i in range(3):
        for j in range(3):
            T[i, j] = (A[i, 0] * G[0, j] + A[i, 1] * G[1, j]) + A[i, 2] * G[2, j]
        T[i, 3] = G[i, 3] + A[i, 3]
    return T


def np_cost_omp(T, src, out, tgt, corr, M):
    """pclomp's OptimizationFunctorWithIndices at the float32 pose T: res = T p - q on the raw source, dR over output_i = guess p.
    Returns f, the translation gradient and the unscaled sum (guess p) (M res)^T."""
    ok = corr >= 0
    res = (xf32(T, src[ok]) - tgt[corr[ok], :3]).astype(np.float64)
    t = np.einsum("nij,nj->ni", M[ok], res)
    m = ok.sum()
    return np.einsum("ni,ni->", res, t) / m, 2.0 / m * t.sum(0), out[ok].astype(np.float64).T @ t, t.sum(0)


def rot_grad(x, dRsum):
    """<dR/dangle, dRsum> (matricesInnerProd) with dR/dangle from central differences of the ZYX rotation"""
    from scipy.spatial.transform import Rotation
    g = np.zeros(3)
    for a in range(3):
        h = 1e-6
        xp, xm = np.array(x, float), np.array(x, float)
        xp[3 + a] += h
        xm[3 + a] -= h
        dR = (Rotation.from_euler("ZYX", [xp[5], xp[4], xp[3]]).as_matrix() - Rotation.from_euler("ZYX", [xm[5], xm[4], xm[3]]).as_matrix()) / (2 * h)
        g[a] = np.sum(dR * dRsum.T)
    return g


def f_smooth(x, guess, src, tgt, corr, M):
    """pclomp's f with the pose in float64 (smooth, for finite differences)"""
    from scipy.spatial.transform import Rotation
    R = Rotation.from_euler("ZYX", [x[5], x[4], x[3]]).as_matrix()
    G = np.asarray(guess, np.float64)
    ok = corr >= 0
    p = src[ok, :3].astype(np.float64)
    res = p @ (R @ G[:3, :3]).T + G[:3, 3] + np.asarray(x[:3]) - tgt[corr[ok], :3]
    t = np.einsum("nij,nj->ni", M[ok], res)
    return np.einsum("ni,ni->", res, t) / ok.sum()


def test_pose_is_apply_state_composed_with_the_guess(ref):
    for guess in GUESSES + [gr.pose((-40.0, 12.5, 3.0), (0.3, -0.2, 0.6))]:
        for x in XS + [[1.5, -2.0, 0.3, 0.4, -0.3, 1.1]]:
            T = ref.pose(x, guess)
            assert np.array_equal(T, np_pose(ref.apply_state(x), guess))
            assert np.array_equal(T[3], guess[3])
    # at an identity guess the functor's pose is GICP's applyState(I, x), bit for bit
    for x in XS:
        assert np.array_equal(ref.pose(x, np.eye(4, dtype=np.float32)), ref.apply_state(x))


@pytest.mark.parametrize("gi", range(len(GUESSES)))
def test_cost_and_gradient_match_numpy_and_finite_differences(ref, gi):
    guess = GUESSES[gi]
    tgt = gr.scene(1500, seed=21)
    src = gr.transform(gr.scene(1500, seed=22), np.linalg.inv(guess.astype(np.float64)).astype(np.float32) @ gr.pose((0.15, -0.1, 0.0), (0.0, 0.0, 0.02)))
    scov, tcov = ref.covariances(src), ref.covariances(tgt)
    T_rel = gr.pose((-0.1, 0.05, 0.0), (0.0, 0.0, -0.01))
    corr, M, cnt = ref.correspondences(src, tgt, guess, T_rel, scov=scov, tcov=tcov)
    wc, _, out = np_correspondences(src, tgt, scov, tcov, guess, T_rel)
    assert np.array_equal(corr, wc) and cnt > 500
    for x in XS:
        f, g, m = ref.fdf(src, tgt, guess, T_rel, x, scov=scov, tcov=tcov)
        T = np_pose(ref.apply_state(x), guess)
        wf, wgt, dRsum, tsum = np_cost_omp(T, src, out, tgt, corr, M)
        assert m == cnt
        assert abs(f - wf) <= 1e-9 * abs(wf)
        assert np.max(np.abs(g[:3] - wgt)) <= 1e-9 * np.max(np.abs(wgt))
        wgr = rot_grad(x, 2.0 / m * dRsum)
        assert np.max(np.abs(g[3:] - wgr)) <= 1e-6 * np.max(np.abs(wgr))
        # the 13 cost-pass sums at applyState(guess, x) are the same numbers before scaling
        sums, _ = ref.cost(src, tgt, guess, T_rel, ref.pose(x, guess), scov=scov, tcov=tcov)
        assert abs(sums[0] / m - f) <= 1e-12 * abs(f) and np.allclose(sums[1:4] * 2.0 / m, g[:3], rtol=1e-12, atol=0)
        # central differences of f: the translation gradient always; the rotation gradient once the dR term's t_g (guess p = R_g p +
        # t_g, where d res / d angle = dR R_g p) is taken out, which is pclomp's gradient and not f's own when the guess is translated
        fd = np.zeros(6)
        for a in range(6):
            h = 1e-5
            xp, xm = np.array(x, float), np.array(x, float)
            xp[a] += h
            xm[a] -= h
            fd[a] = (f_smooth(xp, guess, src, tgt, corr, M) - f_smooth(xm, guess, src, tgt, corr, M)) / (2 * h)
        scale = np.max(np.abs(fd))
        assert np.max(np.abs(g[:3] - fd[:3])) <= 1e-3 * scale
        tg = np.asarray(guess, np.float64)[:3, 3]
        exact_rot = g[3:] - rot_grad(x, 2.0 / m * np.outer(tg, tsum))
        assert np.max(np.abs(exact_rot - fd[3:])) <= 1e-3 * scale


def test_functor_is_gicps_at_the_shifted_state(ref, gicp):
    """f_omp(x; guess) = f_gicp(x') with R(x') = R(x) and t(x') = t(x) + t_g - R(x) t_g, to float32 rounding"""
    from scipy.spatial.transform import Rotation
    tgt = gr.scene(2000, seed=23)
    guess = GUESSES[2]
    src = gr.transform(gr.scene(2000, seed=24), np.linalg.inv(guess.astype(np.float64)).astype(np.float32))
    scov, tcov = ref.covariances(src), ref.covariances(tgt)
    T_rel = np.eye(4, dtype=np.float32)
    for x in XS:
        f, _, m = ref.fdf(src, tgt, guess, T_rel, x, scov=scov, tcov=tcov)
        R = Rotation.from_euler("ZYX", [x[5], x[4], x[3]]).as_matrix()
        tg = np.asarray(guess, np.float64)[:3, 3]
        xs = np.r_[np.asarray(x[:3]) + tg - R @ tg, x[3:]]
        fg, _, mg = gicp.fdf(src, tgt, guess, T_rel, xs, scov=scov, tcov=tcov)
        assert m == mg > 500
        assert abs(f - fg) <= 1e-3 * abs(fg) + 1e-9
    # at x = 0 the shift is 0 (R(0) = I): the two functors agree to float32 rounding of the pose products
    f0, _, _ = ref.fdf(src, tgt, guess, T_rel, np.zeros(6), scov=scov, tcov=tcov)
    g0, _, _ = gicp.fdf(src, tgt, guess, T_rel, np.zeros(6), scov=scov, tcov=tcov)
    assert abs(f0 - g0) <= 1e-5 * abs(g0)


def test_identity_guess_align_is_gicps(ref, gicp):
    tgt = gr.scene(6000, seed=25)
    src = gr.transform(gr.scene(6000, seed=26), gr.pose((0.3, -0.2, 0.03), (0.01, 0.0, 0.05)))
    for kw in ({}, dict(max_optimizer_iterations=1, max_iterations=8)):
        a, b = ref.align(src, tgt, **kw), gicp.align(src, tgt, **kw)
        assert np.array_equal(a["T"], b["T"])
        for key in ("converged", "iterations", "corr_passes", "cost_passes", "evaluations", "bfgs_steps"):
            assert a[key] == b[key], key


def test_translated_guess_ends_elsewhere(ref, gicp):
    T_true = gr.pose((4.0, -3.0, 0.2), (0.0, 0.01, 0.3))
    tgt = gr.scene(6000, seed=27)
    src = gr.transform(tgt, np.linalg.inv(T_true.astype(np.float64)).astype(np.float32))
    guess = gr.pose((3.8, -2.9, 0.2), (0.0, 0.0, 0.28))
    a, b = ref.align(src, tgt, guess), gicp.align(src, tgt, guess)
    assert a["converged"] and b["converged"] and a["iterations"] >= 1
    # GICP recovers the transform; pclomp's functor pose leaves its end pose about (R(x*) - I) t_g away
    assert np.max(np.abs(b["T"][:3, 3] - T_true[:3, 3])) <= 5e-3
    assert np.max(np.abs(a["T"] - b["T"])) > 1e-3
    # with the guess's translation taken away, the two end at the same answer (R(x) R_g p and R(x) (R_g p) round differently in
    # float32, so the line searches may part in the last bits: the end-point rule of the GICP tests)
    guess0 = guess.copy()
    guess0[:3, 3] = 0
    src0 = gr.transform(tgt, np.linalg.inv(gr.pose((0.0, 0.0, 0.0), (0.0, 0.01, 0.3)).astype(np.float64)).astype(np.float32))
    a0, b0 = ref.align(src0, tgt, guess0), gicp.align(src0, tgt, guess0)
    assert a0["converged"] and b0["converged"]
    gr.end_point_is_as_good(a0["T"], b0["T"])


def test_too_few_correspondences_and_empty_clouds(ref):
    tgt = gr.scene(800, seed=28)
    src = gr.scene(800, seed=29)
    far = gr.pose((400.0, 0.0, 0.0))
    w = ref.align(src, tgt, far)
    assert not w["converged"] and w["iterations"] == 0 and w["corr_passes"] == 1 and w["cost_passes"] == 0
    assert np.array_equal(w["T"], far)


def test_pcl_entry_points_in_the_omp_library_are_gicps(ref, gicp):
    """the omp library compiles gicp_pcl_ref.cpp with its functor's cost hook: without an omp entry point active, that hook is pcl
    GICP's own cost_sums, so the library's ref_gicp_pcl_* align and fdf give the pcl GICP library's results bit for bit"""
    view = gr.Reference.__new__(gr.Reference)
    view.lib = ref.lib._L
    tgt = gr.scene(4000, seed=30)
    guess = GUESSES[2]
    src = gr.transform(gr.scene(4000, seed=31), np.linalg.inv(guess.astype(np.float64)).astype(np.float32) @ gr.pose((0.1, 0.0, 0.0)))
    a, b = view.align(src, tgt, guess), gicp.align(src, tgt, guess)
    assert np.array_equal(a["T"], b["T"]) and all(a[k] == b[k] for k in ("converged", "iterations", "cost_passes", "evaluations"))
    assert not np.array_equal(ref.align(src, tgt, guess)["T"], b["T"])
    x = XS[1]
    fa, ga, _ = view.fdf(src, tgt, guess, np.eye(4, dtype=np.float32), x)
    fb, gb, _ = gicp.fdf(src, tgt, guess, np.eye(4, dtype=np.float32), x)
    assert fa == fb and np.array_equal(ga, gb)
