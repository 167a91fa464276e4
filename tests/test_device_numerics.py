"""CPU half of the device-numerics tests (tests/device_numerics_harness.cu; the device half is test_device_numerics_gpu.py).

  * PTX / SASS pin: no kernel of the engine holds a float32 fma / mad in its PTX, and in the SASS of the built library every FFMA
    of the kernels with float32 bit-exact contracts comes from a correctly rounded division or square root: the kernels hold as many
    FFMA as the same source built with -fmad=false, where ptxas contracts nothing.
  * class B, host build: the plain-operator helpers the device may contract (ldlt6_solve, se3_exp, mul_iso, inv3, mul3,
    sym_min_eigvec3, sym_cross_eigvec3, gicp_is_converged) within stated error bounds of exact references (mpmath at 50 digits,
    np.longdouble); the same checks run on the device build in the GPU suite.
  * the LM replay's recorded round sequences (the oracle-emulated rounds of lm_harness plus synthetic ones with rho at 0 and steps
    at the convergence epsilons) replay on the host build to the recording's own decisions."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import device_numerics_build as dnb

ROOT = dnb.ROOT
EPS = np.finfo(np.float64).eps

# kernels whose float32 arithmetic is a bit-exact contract (their PTX float32 mul / add / sub all carry .rn)
F32_EXACT = [r"k_transform\w*", r"k_vgicp_cuda_round", r"k_pcl_cov\w*<[^>]*VcudaCov>", r"k_gicp_pcl_cost\w*", r"k_gicp_omp_cost\w*",
             r"k_icp_step", r"k_ransac_\w+", r"k_floor_band", r"k_avg_\w+", r"k_vg_centroid", r"k_map_\w+", r"k_deskew",
             r"k_pair_search<\d>", r"k_fitness\w*"]


@pytest.fixture(scope="module")
def host(oracle, tmp_path_factory):
    return dnb.Harness(dnb.build_host(tmp_path_factory.mktemp("dn_host")))


def _sass_ffma(path):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([cuobjdump, "-sass", path], capture_output=True, text=True, check=True).stdout
    out = {}
    for f in sass.split("Function : ")[1:]:
        name = f.split("\n", 1)[0].strip()
        out[name] = len(re.findall(r"\bFFMA\b", f))
    return out


def _demangle(names):
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return dict(zip(names, r))


@pytest.fixture(scope="module")
def engine_ptx_text(tmp_path_factory):
    from hdl_graph_slam_b200 import build
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    ptx = tmp_path_factory.mktemp("ptx") / "api.ptx"
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC", "-lineinfo")]
    flags = [f.replace("code=sm_90a", "code=compute_90a") for f in flags]
    subprocess.check_call([nvcc] + flags + ["-ptx", "-o", str(ptx), os.path.join(ROOT, "hdl_graph_slam_b200", "csrc", "api.cu")])
    return ptx.read_text()


def test_no_kernel_has_float32_fma(engine_ptx_text):
    bodies = re.findall(r"\.entry (\w+)\((.*?)\n}\n", engine_ptx_text, flags=re.S)
    assert len(bodies) > 100
    fused = [n for n, b in bodies if re.search(r"\b(fma|mad)(\.\w+)*\.f32\b", b)]
    assert not fused, f"float32 fma / mad in {_demangle(fused)}"


def test_exact_float32_kernels_have_no_contracted_ffma(tmp_path):
    """FFMA in the kernels with float32 bit-exact contracts: as many in the library's SASS as with -fmad=false (the FFMA of the
    correctly rounded float32 / float64 division and square root sequences), so ptxas contracted no multiply-add of theirs"""
    from hdl_graph_slam_b200 import build
    build.build_engine()
    so = os.path.join(ROOT, "hdl_graph_slam_b200", "_lib", "libb200reg.so")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cubin = tmp_path / "nofma.cubin"
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    subprocess.check_call([nvcc] + flags + ["-fmad=false", "-cubin", "-o", str(cubin), os.path.join(ROOT, "hdl_graph_slam_b200", "csrc", "api.cu")])
    built, nofma = _sass_ffma(so), _sass_ffma(str(cubin))
    names = _demangle(list(built))
    pat = re.compile(r"b2r::(" + "|".join(F32_EXACT) + r")(?!\w)")
    exact = [m for m, d in names.items() if pat.search(d.replace("b2r::VcudaCov", "VcudaCov"))]
    assert len(exact) >= 25, sorted(names[m] for m in exact)
    for want in ("k_transform", "k_vgicp_cuda_round", "k_icp_step", "k_ransac_samples", "k_floor_band", "k_deskew", "k_pair_search<1>",
                 "k_fitness", "k_pcl_cov<VcudaCov>", "k_pcl_cov_reg<20, VcudaCov>", "k_pcl_cov_reg_batch<20, VcudaCov>"):
        assert any(want in names[m].replace("b2r::VcudaCov", "VcudaCov") for m in exact), want
    contracted = {names[m][:100]: (built[m], nofma.get(m)) for m in exact if built[m] != nofma.get(m)}
    assert not contracted, f"FFMA (built, -fmad=false) differ: {contracted}"


# ------------------------------------------------------------------------------------------------ class B
CLASS_B = {40: "ldlt6_solve", 41: "se3_exp", 42: "mul_iso", 43: "inv3", 44: "mul3", 45: "sym_min_eigvec3", 46: "sym_cross_eigvec3",
           47: "gicp_is_converged"}


def _spd6(rng, n):
    M = rng.standard_normal((n, 6, 6)) * 10.0 ** rng.uniform(-3, 3, (n, 1, 6))
    A = M @ M.transpose(0, 2, 1) + np.eye(6)[None] * 10.0 ** rng.uniform(-8, 0, (n, 1, 1))
    return A * 10.0 ** rng.uniform(-10, 10, (n, 1, 1))


def _se3_inputs(rng, n):
    w = rng.standard_normal((n, 3))
    w /= np.linalg.norm(w, axis=1, keepdims=True)
    th2 = np.concatenate([np.full(n // 8, 1e-10) * (1 - 2.0 ** -52), np.full(n // 8, 1e-10), np.full(n // 8, 1e-10) * (1 + 2.0 ** -52),
                          10.0 ** rng.uniform(-24, -10, n // 8), (np.pi - 10.0 ** rng.uniform(-12, -2, n // 8)) ** 2,
                          np.full(n // 8, np.pi ** 2), 1e-20 * rng.random(n // 8)])
    th2 = np.concatenate([th2, rng.uniform(0, 4 * np.pi ** 2, n - len(th2))])
    om = w * np.sqrt(th2)[:, None]
    return np.c_[om, rng.standard_normal((n, 3)) * 10.0 ** rng.uniform(-3, 2, (n, 1))]


def _iso(rng, n):
    a = _se3_inputs(rng, n)
    T = np.zeros((n, 16))
    for i in range(n):  # rotation from the exact formula, translation random
        th = np.linalg.norm(a[i, :3])
        K = np.array([[0, -a[i, 2], a[i, 1]], [a[i, 2], 0, -a[i, 0]], [-a[i, 1], a[i, 0], 0]])
        R = np.eye(3) + (np.sin(th) / th if th else 1.0) * K + ((1 - np.cos(th)) / th ** 2 if th else 0.5) * (K @ K)
        T[i] = np.r_[np.c_[R, a[i, 3:] * 100], [[0, 0, 0, 1]]].reshape(16)
    return T


def _mp_se3(a):
    import mpmath as mp
    mp.mp.dps = 50
    o = [mp.mpf(float(x)) for x in a[:3]]
    th2 = o[0] ** 2 + o[1] ** 2 + o[2] ** 2
    th = mp.sqrt(th2)
    if th2 == 0:
        imag, real = mp.mpf(0.5), mp.mpf(1)
    else:
        imag, real = mp.sin(th / 2) / th, mp.cos(th / 2)
    q = [real] + [imag * x for x in o]
    w, x, y, z = q
    R = mp.matrix([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                   [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                   [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    Om = mp.matrix([[0, -o[2], o[1]], [o[2], 0, -o[0]], [-o[1], o[0], 0]])
    if float(th) < 1e-10:  # upstream takes V = R there
        V = R
    else:
        V = mp.eye(3) + (1 - mp.cos(th)) / th2 * Om + (th - mp.sin(th)) / (th2 * th) * (Om * Om)
    t = V * mp.matrix([mp.mpf(float(x)) for x in a[3:]])
    return np.array([[float(R[r, c]) for c in range(3)] + [float(t[r])] for r in range(3)])


def _mp_min_eig(A):
    import mpmath as mp
    mp.mp.dps = 50
    E, Q = mp.eigsy(mp.matrix([[mp.mpf(float(A[r * 3 + c])) for c in range(3)] for r in range(3)]))
    ev = [E[i] for i in range(3)]
    i = int(np.argmin([float(e) for e in ev]))
    s = sorted(ev)
    return np.array([float(Q[r, i]) for r in range(3)]), float(s[0]), float(s[1] - s[0]), max(abs(float(e)) for e in ev)


def _eig_inputs(rng, n):
    A = dnb.sym_matrices(rng, n, np.float64)
    keep = np.isfinite(A).all(1) & (np.abs(A).max(1) > 1e-250) & (np.abs(A).max(1) < 1e250)
    return A[keep]


def check_class_b(h, fn, host=None):
    """the error bounds of class-B function fn on harness h (host or device build); with `host`, decisions equal the host build's"""
    rng = np.random.default_rng(7000 + fn)
    if fn == 40:
        n = 100_000
        A, b = _spd6(rng, n), rng.standard_normal((n, 6)) * 10.0 ** rng.uniform(-5, 5, (n, 1))
        A[:50, 0, 0] = 0.0                     # zero first pivot
        A[50:100, 3, 3] = np.nan               # NaN pivot
        A[100:150, 2, 2] = A[100:150, 2, 1] = A[100:150, 1, 2] = A[100:150, 1, 1] = 1.0  # singular leading 3x3: zero pivot at j = 2
        A[100:150, 2, 0] = A[100:150, 0, 2] = A[100:150, 1, 0] = A[100:150, 0, 1] = 0.0
        o = h.run(fn, np.c_[A.reshape(n, 36), b]).view(np.float64)
        ok, x = o[:, 0], o[:, 1:]
        assert (ok[:150] == 0).all() and (ok[150:] == 1).all()
        Al, xl, bl = A[150:].astype(np.longdouble), x[150:].astype(np.longdouble), b[150:].astype(np.longdouble)
        r = np.einsum("nij,nj->ni", Al, xl) - bl
        eta = np.abs(r).max(1) / (np.abs(Al).sum(2).max(1) * np.abs(xl).max(1) + np.abs(bl).max(1))
        assert float(eta.max()) <= 64 * EPS, float(eta.max()) / EPS  # normwise backward error of LDL^T on SPD: O(n eps)
        if host is not None:
            np.testing.assert_array_equal(ok, host.run(fn, np.c_[A.reshape(n, 36), b]).view(np.float64)[:, 0])
    elif fn == 41:
        a = _se3_inputs(rng, 2000)
        o = h.run(fn, a).view(np.float64).reshape(-1, 4, 4)
        for i in range(len(a)):
            ref = _mp_se3(a[i])
            err_r = np.abs(o[i, :3, :3] - ref[:, :3]).max()
            err_t = np.abs(o[i, :3, 3] - ref[:, 3]).max() / max(1.0, np.abs(a[i, 3:]).max())
            # (1 - cos theta) / theta^2 cancels: its absolute error eps / theta^2, times |Omega| = theta, bounds V's error by eps / theta
            th = float(np.linalg.norm(a[i, :3]))
            assert err_r <= 8 * EPS and err_t <= 64 * EPS * max(1.0, 1.0 / th if th >= 1e-10 else 1.0), (a[i].tolist(), err_r / EPS, err_t / EPS)
        assert (o[:, 3] == [0, 0, 0, 1]).all()
    elif fn in (42, 44):
        n = 100_000
        if fn == 42:
            A, B = _iso(rng, n // 10), _iso(rng, n // 10)
            o = h.run(fn, np.c_[A, B]).view(np.float64)
            Al, Bl = A.reshape(-1, 4, 4).astype(np.longdouble), B.reshape(-1, 4, 4).astype(np.longdouble)
        else:
            A = rng.standard_normal((n, 9)) * 10.0 ** rng.uniform(-100, 100, (n, 1))
            B = rng.standard_normal((n, 9)) * 10.0 ** rng.uniform(-100, 100, (n, 1))
            o = h.run(fn, np.c_[A, B]).view(np.float64)
            Al, Bl = A.reshape(-1, 3, 3).astype(np.longdouble), B.reshape(-1, 3, 3).astype(np.longdouble)
        exact = Al @ Bl
        mag = np.abs(Al) @ np.abs(Bl)
        m = exact.shape[1]
        o = o.reshape(exact.shape[0], -1)[:, : m * exact.shape[2]].reshape(exact.shape)
        rows = 3
        err = np.abs(o[:, :rows] - exact[:, :rows]) / np.maximum(mag[:, :rows], np.finfo(np.float64).tiny)
        assert float(err.max()) <= 4 * EPS, float(err.max()) / EPS  # gamma_4 componentwise bound of a 3- / 4-term dot product
    elif fn == 43:
        n = 100_000
        A = rng.standard_normal((n, 9)) * 10.0 ** rng.uniform(-50, 50, (n, 1))
        A[: n // 10] = dnb.sym_matrices(rng, n // 10, np.float64)
        A = A[np.isfinite(A).all(1) & (np.abs(A).max(1) > 1e-90) & (np.abs(A).max(1) < 1e90)]
        o = h.run(fn, A).view(np.float64)
        Al = A.reshape(-1, 3, 3).astype(np.longdouble)
        c00 = Al[:, 1, 1] * Al[:, 2, 2] - Al[:, 1, 2] * Al[:, 2, 1]
        c01 = Al[:, 1, 2] * Al[:, 2, 0] - Al[:, 1, 0] * Al[:, 2, 2]
        c02 = Al[:, 1, 0] * Al[:, 2, 1] - Al[:, 1, 1] * Al[:, 2, 0]
        det = Al[:, 0, 0] * c00 + Al[:, 0, 1] * c01 + Al[:, 0, 2] * c02
        perm = (np.abs(Al[:, 0, :]) * (np.abs(Al[:, 1, [1, 2, 0]] * Al[:, 2, [2, 0, 1]]) + np.abs(Al[:, 1, [2, 0, 1]] * Al[:, 2, [1, 2, 0]]))).sum(1)
        assert float((np.abs(o[:, 9] - det) / np.maximum(perm, np.finfo(np.float64).tiny)).max()) <= 4 * EPS
        good = np.abs(det) > 1e-8 * perm   # condition below 1e8
        inv = np.linalg.inv(A[good].reshape(-1, 3, 3))  # reference to float64; the bound below is far above its error
        kappa = np.abs(A[good].reshape(-1, 3, 3)).sum(2).max(1) * np.abs(inv).sum(2).max(1)
        err = np.abs(o[good, :9].reshape(-1, 3, 3) - inv).max((1, 2)) / np.abs(inv).max((1, 2))
        assert float((err / (kappa * EPS)).max()) <= 16
    elif fn in (45, 46):
        A = _eig_inputs(rng, 4000)[:2000]
        refs = [_mp_min_eig(a) for a in A]
        if fn == 45:
            o = h.run(fn, A).view(np.float64)
        else:
            lam = np.array([r[1] for r in refs])
            o = h.run(fn, np.c_[A[:, [0, 1, 2, 4, 5, 8]], lam]).view(np.float64)
        for a, v, (u, lam0, gap, nrm) in zip(A, o, refs):
            if fn == 45 and a[1] == 0 and a[2] == 0 and a[5] == 0:
                continue  # exactly diagonal: the JacobiSVD axis rule (by |a_ii|), tested in test_diagonal_normals.py
            if not gap > 1e-6 * nrm:
                continue  # near-tied smallest pair: the eigenvector is not determined to more than eps / (gap / |A|)
            s = np.linalg.norm(np.cross(v, u))  # sin of the angle
            assert abs(np.linalg.norm(v) - 1) <= 4 * EPS
            assert s <= 512 * EPS * nrm / gap, (a.tolist(), s, EPS * nrm / gap)
    elif fn == 47:
        n = 100_000
        rot_eps, trans_eps = 10.0 ** rng.uniform(-8, -1, n), 10.0 ** rng.uniform(-8, -1, n)
        D = np.tile(np.eye(4).reshape(1, 16), (n, 1))
        k = rng.integers(0, 12, n)  # entry that sits on its threshold
        on = np.where(k < 9, rot_eps, trans_eps) * rng.choice([1 - EPS, 1.0, 1 + 2 * EPS, 0.5], n)
        rows = np.where(k < 9, (k // 3) * 4 + k % 3, (k - 9) * 4 + 3)
        D[np.arange(n), rows] += on * rng.choice([-1.0, 1.0], n)
        o = h.run(fn, np.c_[D, rot_eps, trans_eps]).view(np.float64)[:, 0]
        R = D.reshape(n, 4, 4)
        mr = ((1.0 / rot_eps)[:, None, None] * np.abs(R[:, :3, :3] - np.eye(3)[None])).max((1, 2))
        mt = ((1.0 / trans_eps)[:, None] * np.abs(R[:, :3, 3])).max(1)
        np.testing.assert_array_equal(o, (np.maximum(mr, mt) < 1).astype(np.float64))
        assert 0.1 < o.mean() < 0.9
    else:
        raise ValueError(fn)


@pytest.mark.parametrize("fn", sorted(CLASS_B), ids=lambda f: CLASS_B[f])
def test_class_b_host_within_bounds(host, fn):
    check_class_b(host, fn)


# ------------------------------------------------------------------------------------------------ LM replay inputs
def lm_cases():
    return ["odometry", "loop_perturbed", "iteration_cap", "far_guess", "tight_epsilon", "synthetic_rho_zero", "synthetic_delta_at_eps"]


def lm_rounds(host, synth, case):
    """(R rounds x 29, x0[12], (rot_eps, trans_eps, max_iterations)) of one LM run: recorded from the oracle-emulated rounds of
    lm_harness, or synthetic sums whose trial cost equals the model cost to the last bit (rho = +-0 or one ulp below) or whose
    steps land on the translation epsilon"""
    from common import perturb
    if not case.startswith("synthetic"):
        tgt = synth.scan("vlp16_16k", frame=5, stride=4)
        src = synth.scan("vlp16_16k", frame=7 if case != "loop_perturbed" else 9, stride=4)
        max_it, eps, dist = 64, 0.01, 2.5
        guess = np.eye(4)
        if case == "loop_perturbed":
            guess = np.linalg.inv(synth.pose_matrix(5)) @ synth.pose_matrix(9) @ perturb(3, 0.5, 3.0)
        elif case == "iteration_cap":
            max_it = 2
        elif case == "far_guess":
            guess = perturb(11, 2.0, 8.0)
        elif case == "tight_epsilon":
            eps = 1e-5
        g = np.ascontiguousarray(guess, np.float32)
        R = np.zeros((2000, 29))
        nr = host.lib.dn_lm_record(src.ctypes.data, len(src) // 4, tgt.ctypes.data, len(tgt) // 4, 4, max_it, eps, dist, g.ctypes.data,
                                   R.ctypes.data, len(R))
        assert 1 < nr < len(R)
        return R[:nr], g.astype(np.float64)[:3].reshape(12), (2e-3, eps, max_it)
    rng = np.random.default_rng(31 if case.endswith("zero") else 37)
    rounds, trans_eps = 200, 1e-3
    M = rng.standard_normal((6, 6))
    H = M @ M.T + np.eye(6)
    R = np.zeros((rounds, 29))
    R[:, :21] = H[np.triu_indices(6)]
    Y = 10.0
    R[:, 27] = Y
    if case.endswith("zero"):
        R[:, 21:27] = rng.standard_normal((rounds, 6)) * 1e-2
        R[:, 28] = Y * (1 + rng.choice([-EPS, 0.0, EPS], rounds))  # rho = +-tiny or exactly 0
    else:
        d = np.zeros((rounds, 6))
        d[:, 3] = trans_eps * (1 + rng.choice([-1.0, 1.0], rounds, p=[0.03, 0.97]) * 10.0 ** rng.uniform(-4, -3, rounds))
        R[:, 21:27] = -(d @ H.T)  # (H + lambda I) d ~ -b, lambda ~ 1e-9 |H|: the step lands within 1e-3 of the epsilon
        R[:, 28] = Y - 1e-3
    return R, np.eye(4)[:3].reshape(12), (2e-3, trans_eps, 10_000)


@pytest.mark.parametrize("case", ["odometry", "far_guess", "synthetic_rho_zero", "synthetic_delta_at_eps"])
def test_lm_replay_host_reproduces_the_recording(host, synth, case):
    """the replay entry point, on the host build, walks the recorded sequence to its end (mode DONE exactly at the last round for
    a recording) and both synthetic sequences exercise rejections (li > 0) and acceptances"""
    R, x0, cfg = lm_rounds(host, synth, case)
    o = host.lm_replay(R, x0, *cfg)
    if not case.startswith("synthetic"):
        assert (o[:-1, 0] != 5).all() and o[-1, 0] == 5  # PM_DONE at the last recorded round, never before
    else:
        live = o[o[:, 0] >= 0]
        if case.endswith("zero"):
            assert len(live) > 10 and (live[:, 1] > 0).any()
        else:
            assert len(live) >= 2 and (live[:, 3] == 0).any()


# ------------------------------------------------------------------------------------------------ the shared atan2
def test_atan2_rn_is_within_an_ulp_of_glibc_and_exact(host):
    """atan2_rn (csrc/atan2_rn.cuh), the float64 atan2 that pcl_eigen33 and tests/floor_ref.cpp share, against glibc's atan2 on 1e6
    pairs (<= 2 ulp) and mpmath at 40 digits on 3000 (<= 1.5 ulp), and C99's special values exactly"""
    import mpmath as mp
    rng = np.random.default_rng(11)
    n = 1_000_000
    y = (rng.standard_normal(n) * 10.0 ** rng.uniform(-30, 30, n)).astype(np.float32).astype(np.float64)
    x = (rng.standard_normal(n) * 10.0 ** rng.uniform(-30, 30, n)).astype(np.float32).astype(np.float64)
    y[: n // 2], x[: n // 2] = np.abs(rng.standard_normal(n // 2)), rng.standard_normal(n // 2)  # the pairs computeRoots meets
    o = host.run(64, np.c_[y, x]).view(np.float64)[:, 0]
    g = np.arctan2(y, x)
    assert float((np.abs(o - g) / np.spacing(np.abs(g))).max()) <= 2.0
    mp.mp.dps = 40
    worst = max(float(abs(mp.mpf(float(o[i])) - mp.atan2(mp.mpf(float(y[i])), mp.mpf(float(x[i])))) / np.spacing(abs(g[i])))
                for i in range(3000))
    assert worst <= 1.5, worst
    sp = np.array([(0.0, 1.0), (0.0, -1.0), (-0.0, -1.0), (-0.0, 1.0), (1.0, 0.0), (-1.0, -0.0), (0.0, 0.0), (0.0, -0.0), (-0.0, -0.0),
                   (np.inf, np.inf), (np.inf, -np.inf), (-np.inf, np.inf), (1.0, np.inf), (1.0, -np.inf), (-1.0, -np.inf), (np.inf, 1.0),
                   (np.nan, 1.0), (1.0, np.nan), (5e-324, -1.0), (1e300, 1e-300)])
    o = host.run(64, sp).view(np.float64)[:, 0]
    g = np.arctan2(sp[:, 0], sp[:, 1])
    assert ((o == g) & (np.signbit(o) == np.signbit(g)) | (np.isnan(o) & np.isnan(g))).all(), np.c_[sp, o, g]


def test_class_a_inputs_take_every_branch(host):
    """the class-A inputs reach the branches the device tests must cover: pcl_compute_roots' |c0| < FLT_EPSILON quadratic, the
    a_over_3 and q clamps and the r0 <= 0 fallback; icp_umeyama's rank-2 path and det < 0; ndt_voxel_gaussian's fewer-than-6-point
    voxels and invalidated voxels (numpy restatement of the branch conditions on the inputs, host outputs)"""
    rng = np.random.default_rng(1018)
    A = dnb.class_a_inputs(18, rng, 200_000).view(np.float32)
    _, quad, a3c, qc = dnb.compute_roots_args(A, scale=False)
    r = host.run(18, A).view(np.float32)
    fallback = (r[:, 0] == 0) & ~quad
    counts = dict(quad=int(quad.sum()), a_over_3_clamp=int(a3c.sum()), q_clamp=int(qc.sum()), fallback=int(fallback.sum()))
    assert min(counts.values()) >= 200, counts
    rng = np.random.default_rng(1015)
    sig = dnb.class_a_inputs(15, rng, 100_000).view(np.float32)
    d = host.run(13, np.ascontiguousarray(sig[:, :9])).view(np.float32)[:, 9:12]
    rank = (~(np.abs(d) <= np.abs(d[:, :1]) * np.float32(1e-5))).sum(1)
    det = host.run(14, np.ascontiguousarray(sig[:, :9])).view(np.float32)[:, 0]
    assert (rank == 2).sum() >= 1000 and (det < 0).sum() >= 1000
    rng = np.random.default_rng(1012)
    vox = dnb.class_a_inputs(12, rng, 100_000)
    o = host.run(12, vox).view(np.float64)
    cnt = vox.view(np.float64)[:, 0]
    assert (cnt < 6).sum() >= 1000 and (o[:, 0] == -1).sum() >= 1000 and ((o[:, 0] >= 6)).sum() >= 1000
