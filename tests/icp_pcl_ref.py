"""Shared by the pcl ICP tests: the sequential CPU reference of pcl::IterativeClosestPoint (tests/icp_pcl_ref.cpp) and the host build of
the device's step (tests/icp_pcl_harness.cu), both compiled into a temporary directory."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_VP, _SZ, _D, _I = C.c_void_p, C.c_size_t, C.c_double, C.c_int


def _cxx():
    return "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")


def _p(a):
    return a.ctypes.data if a is not None else None


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def _row(T):
    return np.ascontiguousarray(T, np.float32).reshape(16)


def _step_api(L, prefix):
    getattr(L, prefix + "svd").argtypes = [_VP] * 4
    getattr(L, prefix + "umeyama").argtypes = [_VP] * 4
    f = getattr(L, prefix + "has_converged")
    f.argtypes = [_VP, _I, _I, _D, _D, _D, _VP]
    f.restype = _I


class Step:
    """svd / umeyama / has_converged of one implementation (the reference's or the device source built for the host)"""

    def __init__(self, lib, prefix):
        self.lib, self.prefix = lib, prefix

    def svd(self, A):
        A = _f32(A).reshape(9)
        U, d, V = np.empty(9, np.float32), np.empty(3, np.float32), np.empty(9, np.float32)
        getattr(self.lib, self.prefix + "svd")(_p(A), _p(U), _p(d), _p(V))
        return U.reshape(3, 3), d, V.reshape(3, 3)

    def umeyama(self, sigma, sm, dm):
        s, a, b = _f32(sigma).reshape(9), _f32(sm), _f32(dm)
        Rt = np.empty(16, np.float32)
        getattr(self.lib, self.prefix + "umeyama")(_p(s), _p(a), _p(b), _p(Rt))
        return Rt.reshape(4, 4)

    def has_converged(self, T, iterations, max_iterations, eps, mse, prev):
        t = _row(T)
        pv = np.array([prev], np.float64)
        r = getattr(self.lib, self.prefix + "has_converged")(_p(t), int(iterations), int(max_iterations), 1.0 - eps, float(eps), float(mse), _p(pv))
        return bool(r), float(pv[0])


class Reference(Step):
    def __init__(self, tmpdir):
        so = os.path.join(str(tmpdir), "libicp_pcl_ref.so")
        subprocess.check_call([_cxx(), "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-Wall", "-o", so,
                               os.path.join(ROOT, "tests", "icp_pcl_ref.cpp")])
        L = C.CDLL(so)
        _step_api(L, "ref_icp_")
        cloud = [_VP, _SZ, _SZ, _VP, _SZ, _SZ]
        L.ref_icp_correspondences.restype = _SZ
        L.ref_icp_correspondences.argtypes = cloud + [_VP, _D, _I, _VP, _VP]
        L.ref_icp_estimate.restype = _SZ
        L.ref_icp_estimate.argtypes = cloud + [_VP, _D, _I, _VP, _VP]
        L.ref_icp_align.restype = _SZ
        L.ref_icp_align.argtypes = cloud + [_VP, _D, _D, _I, _I, _VP, _VP, _VP, _SZ]
        super().__init__(L, "ref_icp_")

    @staticmethod
    def _clouds(src, tgt):
        s, t = _f32(src), _f32(tgt)
        return (s, t), [_p(s), s.shape[0], s.shape[1], _p(t), t.shape[0], t.shape[1]]

    def correspondences(self, src, tgt, T, max_dist=2.5, reciprocal=False):
        keep, args = self._clouds(src, tgt)
        n = keep[0].shape[0]
        corr, d2 = np.empty(n, np.int32), np.empty(n, np.float32)
        cnt = self.lib.ref_icp_correspondences(*args, _p(_row(T)), float(max_dist), int(reciprocal), _p(corr), _p(d2))
        return corr, d2, cnt

    def estimate(self, src, tgt, T, max_dist=2.5, reciprocal=False):
        keep, args = self._clouds(src, tgt)
        Rt, sums = np.full(16, np.nan, np.float32), np.full(17, np.nan)
        cnt = self.lib.ref_icp_estimate(*args, _p(_row(T)), float(max_dist), int(reciprocal), _p(Rt), _p(sums))
        return Rt.reshape(4, 4), sums, cnt

    def align(self, src, tgt, guess=None, max_iterations=64, transformation_epsilon=0.01, max_dist=2.5, reciprocal=False):
        keep, args = self._clouds(src, tgt)
        g = _row(np.eye(4) if guess is None else guess)
        T = np.empty(16, np.float32)
        stats = np.zeros(2, np.int64)
        cap = 4096
        counts = np.zeros(cap, np.int64)
        passes = self.lib.ref_icp_align(*args, _p(g), float(transformation_epsilon), float(max_dist), int(max_iterations), int(reciprocal), _p(T),
                                        _p(stats), _p(counts), cap)
        return dict(T=T.reshape(4, 4), converged=bool(stats[0]), iterations=int(stats[1]), counts=counts[:min(passes, cap)].copy())


class DeviceStep(Step):
    """the device's step source (csrc/linalg.cuh) built for the host"""

    def __init__(self, tmpdir):
        so = os.path.join(str(tmpdir), "libicp_pcl_harness.so")
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        subprocess.check_call([nvcc, "-O2", "-std=c++17", "-w", "-Wno-deprecated-gpu-targets", "-shared", "-Xcompiler", "-fPIC,-ffp-contract=off", "-ccbin", _cxx(), "-o", so,
                               os.path.join(ROOT, "tests", "icp_pcl_harness.cu")])
        L = C.CDLL(so)
        _step_api(L, "dev_icp_")
        super().__init__(L, "dev_icp_")
