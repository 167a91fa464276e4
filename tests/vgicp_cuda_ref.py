"""Shared by the FastVGICPCuda tests: the sequential CPU reference of fast_gicp::FastVGICPCuda (tests/vgicp_cuda_ref.cpp, compiled into a
temporary directory) with its own float32 covariances.  The clouds come from vgicp_ref.py."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "vgicp_cuda_ref.cpp")
_VP = C.c_void_p
_SZ = C.c_size_t


class Reference:
    def __init__(self, tmpdir):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
        so = os.path.join(str(tmpdir), "libvgicp_cuda_ref.so")
        subprocess.check_call([cxx, "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-Wall", "-o", so, SRC])
        L = C.CDLL(so)
        L.ref_vcuda_covariances.argtypes = [_VP, _SZ, _SZ, C.c_int, _VP]
        L.ref_vcuda_map.restype = _VP
        L.ref_vcuda_map.argtypes = [_VP, _SZ, _SZ, _VP, C.c_double, _VP]
        L.ref_vcuda_free.argtypes = [_VP]
        L.ref_vcuda_voxels.restype = _SZ
        L.ref_vcuda_voxels.argtypes = [_VP, _VP, _VP, _VP, _VP]
        L.ref_vcuda_linearize.restype = C.c_double
        L.ref_vcuda_linearize.argtypes = [_VP, _VP, _SZ, _SZ, _VP, _VP, _VP, _VP, _VP]
        L.ref_vcuda_error.restype = C.c_double
        L.ref_vcuda_error.argtypes = [_VP, _VP, _SZ, _SZ, _VP, _VP, _VP]
        L.ref_vcuda_align.argtypes = [_VP, _VP, _SZ, _SZ, _VP, _VP, _VP, _VP, _VP, _VP, _VP]
        self.lib = L

    def covariances(self, pts, k=20):
        """(n, 3, 3): float32 raw moments + PLANE, widened; NaN rows for non-finite points"""
        a = np.ascontiguousarray(pts, np.float32)
        out = np.empty((a.shape[0], 3, 3))
        self.lib.ref_vcuda_covariances(a.ctypes.data, a.shape[0], a.shape[1], k, out.ctypes.data)
        return out

    def map(self, tgt, resolution, cov=None, k=20):
        return VcudaMap(self, tgt, resolution, cov, k)


class VcudaMap:
    """the target's float32 Gaussian voxel map (status 1 = a finite point beyond the 21-bit cell range)"""

    def __init__(self, ref, tgt, resolution, cov=None, k=20):
        self.ref = ref
        self.lib = ref.lib
        self.k = k
        self.tgt = np.ascontiguousarray(tgt, np.float32)
        self.cov = np.ascontiguousarray(ref.covariances(self.tgt, k) if cov is None else cov, np.float64)
        st = C.c_int()
        self._m = _VP(self.lib.ref_vcuda_map(self.tgt.ctypes.data, self.tgt.shape[0], self.tgt.shape[1], self.cov.ctypes.data, float(resolution),
                                             C.addressof(st)))
        self.status = st.value

    def __del__(self):
        try:
            self.lib.ref_vcuda_free(self._m)
        except Exception:
            pass

    def voxels(self):
        V = self.lib.ref_vcuda_voxels(self._m, None, None, None, None)
        cells = np.empty((V, 3), np.int32)
        counts = np.empty(V, np.int32)
        mean = np.empty((V, 3))
        cov = np.empty((V, 3, 3))
        self.lib.ref_vcuda_voxels(self._m, cells.ctypes.data, counts.ctypes.data, mean.ctypes.data, cov.ctypes.data)
        return dict(cells=cells, counts=counts, mean=mean, cov=cov)

    def _src(self, src, scov):
        s = np.ascontiguousarray(src, np.float32)
        return s, np.ascontiguousarray(self.ref.covariances(s, self.k) if scov is None else scov, np.float64)

    def linearize(self, src, T, scov=None):
        s, sc = self._src(src, scov)
        T = np.ascontiguousarray(T, np.float64)
        H = np.empty((6, 6))
        b = np.empty(6)
        vox = np.empty(max(s.shape[0], 1), np.int32)
        cost = self.lib.ref_vcuda_linearize(self._m, s.ctypes.data, s.shape[0], s.shape[1], sc.ctypes.data, T.ctypes.data, H.ctypes.data, b.ctypes.data,
                                            vox.ctypes.data)
        return H, b, cost, vox[:s.shape[0]]

    def error(self, src, T1, T2, scov=None):
        s, sc = self._src(src, scov)
        T1 = np.ascontiguousarray(T1, np.float64)
        T2 = np.ascontiguousarray(T2, np.float64)
        return self.lib.ref_vcuda_error(self._m, s.ctypes.data, s.shape[0], s.shape[1], sc.ctypes.data, T1.ctypes.data, T2.ctypes.data)

    def align(self, src, guess=None, scov=None, max_iterations=64, transformation_epsilon=0.01, rotation_epsilon=2e-3):
        s, sc = self._src(src, scov)
        g = np.ascontiguousarray(np.eye(4) if guess is None else guess, np.float32)
        d = np.array([transformation_epsilon, rotation_epsilon], np.float64)
        i = np.array([max_iterations], np.int32)
        T = np.empty((4, 4), np.float32)
        T64 = np.empty((4, 4))
        out = np.zeros(3, np.int32)
        self.lib.ref_vcuda_align(self._m, s.ctypes.data, s.shape[0], s.shape[1], sc.ctypes.data, d.ctypes.data, i.ctypes.data, g.ctypes.data,
                                 T.ctypes.data, out.ctypes.data, T64.ctypes.data)
        return dict(T=T, T64=T64, converged=bool(out[0]), iterations=int(out[1]), lm_failed=bool(out[2]))
