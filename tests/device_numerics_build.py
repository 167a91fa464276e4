"""The two builds of tests/device_numerics_harness.cu and their ctypes view.

device build: nvcc with the library's NVCC_FLAGS unchanged (so contraction decisions are the product's) + OpenMP for the host side
              of the libm sweeps.
host build:   nvcc host code with -ffp-contract=off, as the other host harnesses; linked with the oracle for the LM recordings.
Both export dn_info / dn_run / dn_lm_replay over the same records."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "device_numerics_harness.cu")
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def build_device(out_dir):
    from hdl_graph_slam_b200 import build
    so = os.path.join(str(out_dir), "dn_device.so")
    subprocess.check_call([_nvcc()] + build.NVCC_FLAGS + ["-DDN_DEVICE", "-w", "-Xcompiler", "-fopenmp", "-ccbin", GXX, "-o", so, SRC, "-lgomp"])
    return so


def build_host(out_dir):
    so = os.path.join(str(out_dir), "dn_host.so")
    orc = os.path.join(ROOT, "oracle")
    subprocess.check_call([_nvcc(), "-O2", "-std=c++17", "-w", "-Wno-deprecated-gpu-targets", "-shared", "-DDN_ORACLE", "-gencode", "arch=compute_90a,code=sm_90a", "-ccbin", GXX,
                           "-Xcompiler", "-fPIC,-ffp-contract=off,-fopenmp", "-o", so, SRC, "-L" + orc, "-loracle",
                           "-Xlinker", "-rpath=" + orc, "-lgomp"])
    return so


class Harness:
    def __init__(self, so):
        self.lib = C.CDLL(so)
        self.lib.dn_run.argtypes = [C.c_int, C.c_void_p, C.c_longlong, C.c_void_p]
        self.lib.dn_lm_replay.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        if hasattr(self.lib, "dn_libm_sweep"):
            self.lib.dn_libm_sweep.argtypes = [C.c_int, C.c_ulonglong, C.c_longlong, C.c_int, C.c_void_p]
            self.lib.dn_libm_sweep.restype = C.c_longlong
        if hasattr(self.lib, "dn_lm_record"):
            self.lib.dn_lm_record.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_double, C.c_double,
                                              C.c_void_p, C.c_void_p, C.c_int]

    def words(self, fn):
        i, o = C.c_int(), C.c_int()
        assert self.lib.dn_info(fn, C.byref(i), C.byref(o)) == 0, fn
        return i.value, o.value

    def run(self, fn, rec):
        """rec: (n, in_words) array of any 4- or 8-byte dtype, or a float64 (n, in_words / 2) array -> (n, out_words) uint32"""
        iw, ow = self.words(fn)
        raw = np.ascontiguousarray(rec).view(np.uint32).reshape(len(rec), -1)
        assert raw.shape[1] == iw, (fn, raw.shape, iw)
        out = np.zeros((len(rec), ow), np.uint32)
        rc = self.lib.dn_run(fn, raw.ctypes.data, len(rec), out.ctypes.data)
        assert rc == 0, f"dn_run({fn}) = {rc}"
        return out

    def lm_replay(self, R, x0, rot_eps, trans_eps, max_it):
        R = np.ascontiguousarray(R, np.float64)
        x0 = np.ascontiguousarray(x0, np.float64).reshape(12)
        cfg = np.array([rot_eps, trans_eps], np.float64)
        out = np.zeros((len(R), 22), np.float64)
        assert self.lib.dn_lm_replay(R.ctypes.data, len(R), x0.ctypes.data, cfg.ctypes.data, max_it, out.ctypes.data) == 0
        return out

    def libm_sweep(self, fn, first, count, keep=16):
        bad = np.full((keep, 4), 0xFFFFFFFF, np.uint32)
        n = self.lib.dn_libm_sweep(fn, first, count, keep, bad.ctypes.data)
        assert n >= 0, f"dn_libm_sweep({fn}) = {n}"
        return n, bad[bad[:, 0] != 0xFFFFFFFF].view(np.float32)


# output words of class-A functions that are integers (keys, indices, flags, generator words): compared raw, never as NaNs
INT_WORDS = {7: [0, 1], 8: [0], 20: list(range(8)), 21: [8 * t + i for t in range(4) for i in (0, 1, 2, 7)], 22: [0]}


def same_bits(a, b, fn=None):
    """per-record equality of uint32 words; a float word that is NaN equals any NaN (payload and sign ignored), the integer words
    of function fn (INT_WORDS) must be equal"""
    a = np.asarray(a, np.uint32)
    b = np.asarray(b, np.uint32)
    nan_a = (a & 0x7F800000) == 0x7F800000
    nan_a &= (a & 0x007FFFFF) != 0
    nan_b = (b & 0x7F800000) == 0x7F800000
    nan_b &= (b & 0x007FFFFF) != 0
    both_nan = nan_a & nan_b
    both_nan[:, INT_WORDS.get(fn, [])] = False
    return ((a == b) | both_nan).all(axis=1)


def same_bits64(a, b):
    """the same for records of float64 fields"""
    a = np.ascontiguousarray(a).view(np.float64)
    b = np.ascontiguousarray(b).view(np.float64)
    return ((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))).all(axis=1)


# ------------------------------------------------------------------------------------------------ inputs
F32_SPECIAL = np.array([0.0, -0.0, 1.0, -1.0, 0.5, 3.0, np.float32(1.0) + np.finfo(np.float32).eps, 1e-45, -1e-45, 1.1754942e-38,
                        1.17549435e-38, 3.4028235e38, -3.4028235e38, np.inf, -np.inf, np.nan], np.float32)


def f32_values(rng, n):
    """n float32 values: sign * 10^U(-20, 20) * U(1, 10), with the special values (+-0, subnormals, FLT_MIN, FLT_MAX, +-inf, NaN)"""
    v = (rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(-20, 20, n) * rng.uniform(1, 10, n)).astype(np.float32)
    k = min(n // 50, 20000)
    v[:k] = rng.choice(F32_SPECIAL, k)
    return v


def sym_matrices(rng, n, dtype):
    """(n, 9) row-major symmetric 3x3: generic ones at one scale 10^U(-20, 20) per matrix and at mixed per-entry scales, and the
    structured kinds where eigen-solvers branch: diagonal, multiples of I, exact rank 1 and rank 2 on a 1/8 grid, tied and 1-ulp
    separated eigenvalues, +-0 and subnormal entries, a non-finite entry"""
    kinds = 12
    k = rng.integers(0, kinds, n)
    M = np.zeros((n, 3, 3))
    s = 10.0 ** rng.uniform(-20, 20, n)
    g = lambda *sh: rng.integers(-16, 17, sh) / 8.0  # noqa: E731  1/8 grid
    G = rng.standard_normal((n, 3, 3))
    gen = (G + G.transpose(0, 2, 1)) * s[:, None, None]
    mixed = (G + G.transpose(0, 2, 1)) * 10.0 ** rng.uniform(-6, 6, (n, 1, 1)) * 10.0 ** rng.uniform(-3, 3, (n, 3, 3))
    mixed = 0.5 * (mixed + mixed.transpose(0, 2, 1))
    d = rng.standard_normal((n, 3)) * s[:, None]
    u, v = g(n, 3), g(n, 3)
    r1 = u[:, :, None] * u[:, None, :]
    r2 = r1 + v[:, :, None] * v[:, None, :]
    M[k == 0] = gen[k == 0]
    M[k == 1] = mixed[k == 1]
    M[k == 2] = np.einsum("ni,ij->nij", d, np.eye(3))[k == 2]
    M[k == 3] = (np.eye(3)[None] * d[:, :1, None])[k == 3]
    M[k == 4] = r1[k == 4]
    M[k == 5] = r2[k == 5]
    M[k == 6] = (r1 * s[:, None, None])[k == 6]
    M[k == 7] = (r2 * s[:, None, None])[k == 7]
    # tied eigenvalues: a I + b w w^T with w a signed axis or (1, 1, 0) / (1, 1, 1) direction on the grid
    w = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [1, -1, 1]], np.float64)[rng.integers(0, 5, n)]
    tied = np.eye(3)[None] * g(n)[:, None, None] + g(n)[:, None, None] * w[:, :, None] * w[:, None, :]
    M[k == 8] = tied[k == 8]
    # 1-ulp separated diagonal, then a grid rotation-free shear in the off-diagonals of 0
    a = np.abs(rng.standard_normal(n)) + 0.5
    one_ulp = np.zeros((n, 3, 3))
    one_ulp[:, 0, 0] = a
    one_ulp[:, 1, 1] = np.nextafter(a.astype(dtype), dtype(np.inf)).astype(np.float64)
    one_ulp[:, 2, 2] = a * 2
    one_ulp[:, 0, 1] = one_ulp[:, 1, 0] = np.where(rng.random(n) < 0.5, 0.0, 2.0 ** -30)
    M[k == 9] = one_ulp[k == 9]
    tiny = gen / s[:, None, None] * (1e-40 if dtype == np.float32 else 1e-310)
    tiny[:, 0, 1] = tiny[:, 1, 0] = -0.0
    M[k == 10] = tiny[k == 10]
    bad = gen.copy()
    bad[:, 1, 2] = bad[:, 2, 1] = rng.choice([np.inf, -np.inf, np.nan], n)
    M[k == 11] = bad[k == 11]
    return M.reshape(n, 9).astype(dtype)


def _u32(a):
    return np.ascontiguousarray(a).view(np.uint32).reshape(len(a), -1)


def _grid_points(rng, n, m, offset_scale):
    """(n, m, 3) float32 points: on a 1/64 grid around an offset 10^U(0, offset_scale), a third of the sets collinear or coplanar"""
    off = (rng.choice([-1.0, 1.0], (n, 1, 3)) * 10.0 ** rng.uniform(0, offset_scale, (n, 1, 1))).round()
    p = rng.integers(-64, 65, (n, m, 3)) / 64.0
    kind = rng.integers(0, 3, n)
    t = rng.integers(-64, 65, (n, m, 1)) / 64.0
    p[kind == 1] = (t * np.array([1.0, 0.5, -0.25]))[kind == 1]        # collinear
    p[kind == 2, :, 2] = 0.25                                             # coplanar z = const
    return (p + off).astype(np.float32)


def class_a_inputs(fn, rng, n):
    """n input records of class-A function fn (see the DN_FN table of the harness)"""
    f32 = lambda *sh: f32_values(rng, int(np.prod(sh))).reshape(sh)  # noqa: E731
    if fn in (0, 1, 2, 3, 4):
        return _u32(f32(n, 2))
    if fn == 5:
        return _u32(f32(n, 6))
    if fn == 6:
        return _u32(f32(n, 7))
    if fn == 7:
        d2 = np.abs(f32(n))
        return np.c_[d2.view(np.uint32), rng.integers(0, 2 ** 31, n).astype(np.uint32)]
    if fn == 8:
        return rng.integers(0, 2 ** 32, (n, 3), dtype=np.uint64).astype(np.uint32)
    if fn in (9, 10):
        return _u32(sym_matrices(rng, n, np.float64) if fn == 9 else np.where(rng.random((n, 1)) < 0.5, sym_matrices(rng, n, np.float64),
                    rng.standard_normal((n, 9)) * 10.0 ** rng.uniform(-20, 20, (n, 1))))
    if fn == 11:
        return _u32(np.c_[sym_matrices(rng, n, np.float64), rng.standard_normal((n, 9)) * 10.0 ** rng.uniform(-20, 20, (n, 1))])
    if fn == 12:
        # voxels of 1..15 points on planes, lines, single points and generic sets, near the origin and far from it
        m = 15
        p = _grid_points(rng, n, m, 4).astype(np.float64)
        cnt = rng.integers(1, m + 1, n)
        p[np.arange(m)[None, :] >= cnt[:, None]] = 0.0
        S = p.sum(1)
        S2 = np.einsum("nki,nkj->nij", p, p).reshape(n, 9)
        return _u32(np.c_[cnt.astype(np.float64), S, S2])
    if fn in (13, 14, 18, 19, 24):
        A = sym_matrices(rng, n, np.float32)
        if fn in (13, 14):  # general (non-symmetric) matrices too
            G = f32(n, 9)
            A = np.where(rng.random((n, 1)) < 0.5, A, (rng.standard_normal((n, 9)) * 10.0 ** rng.uniform(-20, 20, (n, 1))).astype(np.float32))
            A[: n // 20] = G[: n // 20]
        return _u32(A)
    if fn == 15:
        # sigma: generic, rank 2 (two outer products on the grid, so the rank-2 branch decides S[2]), reflections (det < 0)
        g = lambda *sh: rng.integers(-16, 17, sh) / 8.0  # noqa: E731
        k = rng.integers(0, 3, n)
        gen = rng.standard_normal((n, 3, 3))
        r2 = g(n, 3)[:, :, None] * g(n, 3)[:, None, :] + g(n, 3)[:, :, None] * g(n, 3)[:, None, :]
        refl = gen.copy()
        refl[:, :, 0] *= -np.sign(np.linalg.det(gen))[:, None]
        sig = np.where((k == 0)[:, None, None], gen, np.where((k == 1)[:, None, None], r2, refl)) * 10.0 ** rng.uniform(-6, 6, (n, 1, 1))
        means = rng.standard_normal((n, 6)) * 10.0 ** rng.uniform(-2, 4, (n, 1))
        return _u32(np.c_[sig.reshape(n, 9), means].astype(np.float32))
    if fn == 16:
        # poses near I whose rotation / translation tests sit exactly on the thresholds, and MSE pairs around 1e-12 apart
        T = np.tile(np.eye(4).reshape(1, 16), (n, 1))
        eps = 10.0 ** rng.uniform(-12, -2, n)
        ang = rng.choice([0.0, 1.0, 0.5], n) * np.sqrt(2 * eps)
        T[:, 0] = T[:, 5] = np.cos(ang).astype(np.float32)
        T[:, 1] = -np.sin(ang).astype(np.float32)
        T[:, 4] = np.sin(ang).astype(np.float32)
        T[:, 3] = np.sqrt(eps * rng.choice([0.5, 1.0, 2.0], n)).astype(np.float32)
        T = T.astype(np.float32).astype(np.float64)
        cos_angle = 0.5 * ((T[:, 0].astype(np.float32) + T[:, 5].astype(np.float32) + T[:, 10].astype(np.float32)) - np.float32(1)).astype(np.float64)
        tsq = (T[:, 3].astype(np.float32) * T[:, 3].astype(np.float32)).astype(np.float64)
        rot = np.where(rng.random(n) < 0.3, cos_angle, 1.0 - eps)
        trans = np.where(rng.random(n) < 0.3, tsq, eps)
        it = rng.integers(0, 4, n).astype(np.float64)
        mse = rng.uniform(0, 1, n)
        prev = mse + rng.choice([1e-12, -1e-12, 0.9999999e-12, 1.0000001e-12, 0.0, 1.0], n)
        return _u32(np.c_[T, it, np.full(n, 3.0), rot, trans, mse, prev])
    if fn == 17:
        bc = f32(n, 2)
        with np.errstate(over="ignore"):
            bc[n // 2:, 1] = (bc[n // 2:, 0].astype(np.float64) ** 2 / 4).astype(np.float32)  # discriminant at 0
        return _u32(bc)
    if fn == 20:
        return np.c_[rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32), rng.integers(0, 1500, n).astype(np.uint32)]
    if fn == 21:
        pts = _grid_points(rng, n, 16, 3)
        same = rng.random(n) < 0.1
        pts[same] = pts[same, :1, :]  # every draw of these is collinear
        hdr = np.c_[rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32), rng.integers(0, 17, n).astype(np.uint32)]
        return np.c_[hdr, pts.reshape(n, 48).view(np.uint32)]
    if fn == 22:
        c = rng.standard_normal((n, 3))
        c /= np.linalg.norm(c, axis=1, keepdims=True)
        p = rng.standard_normal((n, 3)) * 30
        d = -(c * p).sum(1) + rng.choice([0.1, -0.1, 0.0999999, 0.1000001], n)
        return _u32(np.c_[c, d, p].astype(np.float32))
    if fn == 23:
        return _u32((rng.standard_normal((n, 32)) * 10.0 ** rng.uniform(-3, 4, (n, 1))).astype(np.float32))
    if fn == 25:
        pts = _grid_points(rng, n, 20, 5)
        pts += (rng.standard_normal(pts.shape) * 0.01).astype(np.float32) * (rng.random((n, 1, 1)) < 0.5)
        kk = rng.integers(1, 21, n).astype(np.uint32)
        return np.c_[kk, pts.reshape(n, 60).view(np.uint32)]
    raise ValueError(fn)


CLASS_A = {0: "fmul", 1: "fadd", 2: "fsub", 3: "fdiv_rn", 4: "fsqrt_rn", 5: "dist2_f32", 6: "xform_row", 7: "nn_key", 8: "hilbert30",
           9: "sym_eigen3", 10: "inv3_rn", 11: "mul3_rn", 12: "ndt_voxel_gaussian", 13: "icp_jacobi_svd3", 14: "icp_det3f",
           15: "icp_umeyama", 16: "icp_has_converged", 17: "pcl_compute_roots2", 18: "pcl_compute_roots", 19: "pcl_eigen33",
           20: "mt19937", 21: "ransac_draw", 22: "ransac_inlier", 23: "gicp_pcl_mul4f", 24: "vcuda_eigen3", 25: "raw_moment_cov_f32"}


# ------------------------------------------------------------------------------------------------ pcl::eigen33's atan2 arguments
def compute_roots_args(A, scale=True):
    """numpy float32 restatement of pcl_eigen33's scaling and pcl_compute_roots up to its atan2 (every float32 step correctly rounded,
    in linalg.cuh's order; scale=False restates pcl_compute_roots alone): returns (a, b) = (sqrt(-q), half_b) per matrix, NaN where the quadratic branch |c0| < FLT_EPSILON is
    taken, and the branch flags (quadratic, a_over_3 clamped, q clamped)"""
    f = np.float32
    A = np.asarray(A, f).reshape(-1, 9)
    with np.errstate(all="ignore"):
        s = np.abs(A).max(1)
        s = np.where((s <= f(1.17549435e-38)) | (not scale), f(1), s).astype(f)
        S = (A / s[:, None]).astype(f)
        m00, m01, m02, m11, m12, m22 = (S[:, i] for i in (0, 1, 2, 4, 5, 8))
        two, half, inv3 = f(2), f(0.5), f(1.0 / 3.0)
        c0 = (((m00 * m11 * m22 + two * m01 * m02 * m12) - m00 * m12 * m12) - m11 * m02 * m02) - m22 * m01 * m01
        c1 = ((((m00 * m11 - m01 * m01) + m00 * m22) - m02 * m02) + m11 * m22) - m12 * m12
        c2 = (m00 + m11) + m22
        quad = np.abs(c0) < f(1.1920929e-07)
        c2o3 = c2 * inv3
        a3 = (c1 - c2 * c2o3) * inv3
        a3_clamped = a3 > 0
        a3 = np.where(a3_clamped, f(0), a3).astype(f)
        hb = half * (c0 + c2o3 * ((two * c2o3) * c2o3 - c1))
        q = hb * hb + (a3 * a3) * a3
        q_clamped = q > 0
        q = np.where(q_clamped, f(0), q).astype(f)
        a = np.sqrt(-q).astype(f)
    a = np.where(quad, f(np.nan), a)
    hb = np.where(quad, f(np.nan), hb)
    return np.c_[a, hb].astype(f), quad, a3_clamped & ~quad, q_clamped & ~quad


FLOOR_SCANS = [("vlp16", 2), ("hdl32e", 2), ("kitti", 2), ("vlp16", 5), ("hdl32e", 5), ("kitti", 5), ("vlp16", 3), ("hdl32e", 7)]


def floor_scan_covariances(host, synth):
    """the float32 raw-moment covariances floor detection's normal filter computes on the floor tests' scans (stride 8, tilt 0) for
    the two launch files that filter normals: the height band ((0 x + 0 y) + 1 z >= -(float)(h + r) and not >= -(float)(h - r)),
    k = 10 neighbours in the band (itself included) in ascending (float32 d2, index) order, moments by the harness (class A holds
    host == device)"""
    from scipy.spatial import cKDTree
    f = np.float32
    out = []
    for sensor, frame in FLOOR_SCANS:
        c = synth.scan(sensor, frame=frame, stride=8)
        for h, r in ((2.0, 1.0), (1.5, 0.5)):
            z = c[:, 2].astype(f)
            band = c[(z >= -f(h + r)) & ~(z >= -f(h - r)) & np.isfinite(c[:, :3]).all(1), :3].astype(f)
            if len(band) < 10:
                continue
            _, cand = cKDTree(band.astype(np.float64)).query(band.astype(np.float64), k=min(16, len(band)))
            d = band[cand] - band[:, None, :]
            d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
            order = np.lexsort((cand, d2), axis=1)[:, :10]
            nb = band[np.take_along_axis(cand, order, 1)]
            rec = np.zeros((len(band), 61), np.uint32)
            rec[:, 0] = 10
            rec[:, 1:31] = np.ascontiguousarray(nb.reshape(len(band), 30)).view(np.uint32)
            out.append(host.run(25, rec).view(np.float32))
    return np.concatenate(out)
