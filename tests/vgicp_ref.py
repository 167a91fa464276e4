"""Shared by the VGICP tests: the sequential CPU reference of fast_gicp::FastVGICP (tests/vgicp_ref.cpp, compiled into a temporary
directory), fed with the oracle's FastGICP covariances, and the clouds the tests use."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "vgicp_ref.cpp")
_VP = C.c_void_p


def covariances(pts, k=20):
    """FastGICP covariances (n, 3, 3) of the finite points, computed among the finite points only; NaN rows for the others"""
    pts = np.ascontiguousarray(pts, np.float32)
    fin = np.isfinite(pts[:, :3]).all(axis=1)
    out = np.full((pts.shape[0], 3, 3), np.nan)
    if fin.any():
        out[fin] = orc.gicp_covariances(np.ascontiguousarray(pts[fin]), k)
    return out


class Reference:
    def __init__(self, tmpdir):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
        so = os.path.join(str(tmpdir), "libvgicp_ref.so")
        subprocess.check_call([cxx, "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-Wall", "-o", so, SRC])
        L = C.CDLL(so)
        L.ref_vgicp_map.restype = _VP
        L.ref_vgicp_map.argtypes = [_VP, C.c_size_t, C.c_size_t, _VP, C.c_double, _VP]
        L.ref_vgicp_free.argtypes = [_VP]
        L.ref_vgicp_voxels.restype = C.c_size_t
        L.ref_vgicp_voxels.argtypes = [_VP, _VP, _VP, _VP, _VP]
        L.ref_vgicp_linearize.restype = C.c_double
        L.ref_vgicp_linearize.argtypes = [_VP, _VP, C.c_size_t, C.c_size_t, _VP, _VP, _VP, _VP, _VP]
        L.ref_vgicp_error.restype = C.c_double
        L.ref_vgicp_error.argtypes = [_VP, _VP, C.c_size_t, C.c_size_t, _VP, _VP, _VP]
        L.ref_vgicp_align.argtypes = [_VP, _VP, C.c_size_t, C.c_size_t, _VP, _VP, _VP, _VP, _VP, _VP, _VP]
        self.lib = L

    def map(self, tgt, resolution, cov=None):
        return VgicpMap(self, tgt, resolution, cov)


class VgicpMap:
    """the target's Gaussian voxel map (status 1 = a finite point beyond the 21-bit cell range)"""

    def __init__(self, ref, tgt, resolution, cov=None):
        self.lib = ref.lib
        self.tgt = np.ascontiguousarray(tgt, np.float32)
        self.cov = np.ascontiguousarray(covariances(self.tgt) if cov is None else cov, np.float64)
        st = C.c_int()
        self._m = _VP(self.lib.ref_vgicp_map(self.tgt.ctypes.data, self.tgt.shape[0], self.tgt.shape[1], self.cov.ctypes.data, float(resolution),
                                             C.addressof(st)))
        self.status = st.value

    def __del__(self):
        try:
            self.lib.ref_vgicp_free(self._m)
        except Exception:
            pass

    def voxels(self):
        V = self.lib.ref_vgicp_voxels(self._m, None, None, None, None)
        cells = np.empty((V, 3), np.int32)
        counts = np.empty(V, np.int32)
        mean = np.empty((V, 3))
        cov = np.empty((V, 3, 3))
        self.lib.ref_vgicp_voxels(self._m, cells.ctypes.data, counts.ctypes.data, mean.ctypes.data, cov.ctypes.data)
        return dict(cells=cells, counts=counts, mean=mean, cov=cov)

    def linearize(self, src, T, scov=None):
        s = np.ascontiguousarray(src, np.float32)
        sc = np.ascontiguousarray(covariances(s) if scov is None else scov, np.float64)
        T = np.ascontiguousarray(T, np.float64)
        H = np.empty((6, 6))
        b = np.empty(6)
        vox = np.empty(max(s.shape[0], 1), np.int32)
        cost = self.lib.ref_vgicp_linearize(self._m, s.ctypes.data, s.shape[0], s.shape[1], sc.ctypes.data, T.ctypes.data, H.ctypes.data, b.ctypes.data,
                                            vox.ctypes.data)
        return H, b, cost, vox[:s.shape[0]]

    def error(self, src, T1, T2, scov=None):
        s = np.ascontiguousarray(src, np.float32)
        sc = np.ascontiguousarray(covariances(s) if scov is None else scov, np.float64)
        T1 = np.ascontiguousarray(T1, np.float64)
        T2 = np.ascontiguousarray(T2, np.float64)
        return self.lib.ref_vgicp_error(self._m, s.ctypes.data, s.shape[0], s.shape[1], sc.ctypes.data, T1.ctypes.data, T2.ctypes.data)

    def align(self, src, guess=None, scov=None, max_iterations=64, transformation_epsilon=0.01, rotation_epsilon=2e-3):
        s = np.ascontiguousarray(src, np.float32)
        sc = np.ascontiguousarray(covariances(s) if scov is None else scov, np.float64)
        g = np.ascontiguousarray(np.eye(4) if guess is None else guess, np.float32)
        d = np.array([transformation_epsilon, rotation_epsilon], np.float64)
        i = np.array([max_iterations], np.int32)
        T = np.empty((4, 4), np.float32)
        T64 = np.empty((4, 4))
        out = np.zeros(3, np.int32)
        self.lib.ref_vgicp_align(self._m, s.ctypes.data, s.shape[0], s.shape[1], sc.ctypes.data, d.ctypes.data, i.ctypes.data, g.ctypes.data,
                                 T.ctypes.data, out.ctypes.data, T64.ctypes.data)
        return dict(T=T, T64=T64, converged=bool(out[0]), iterations=int(out[1]), lm_failed=bool(out[2]))


def records(xyz):
    xyz = np.asarray(xyz, np.float32)
    return np.c_[xyz, np.ones(xyz.shape[0], np.float32)].astype(np.float32)


def room(n, seed=0):
    """floor, two walls and a box with sensor noise"""
    rng = np.random.default_rng(seed)
    k = n // 4
    floor = np.c_[rng.uniform(-6, 6, k), rng.uniform(-6, 6, k), rng.normal(0, 0.01, k)]
    wall1 = np.c_[rng.uniform(-6, 6, k), np.full(k, 5.0) + rng.normal(0, 0.01, k), rng.uniform(0, 3, k)]
    wall2 = np.c_[np.full(k, -5.0) + rng.normal(0, 0.01, k), rng.uniform(-6, 6, k), rng.uniform(0, 3, k)]
    r = n - 3 * k
    box = np.c_[rng.uniform(1, 2.5, r), rng.uniform(-1, 0.5, r), rng.uniform(0, 1.2, r)]
    return records(np.r_[floor, wall1, wall2, box])


def rigid(rz, t):
    c, s = np.cos(rz), np.sin(rz)
    T = np.eye(4)
    T[:2, :2] = [[c, -s], [s, c]]
    T[:3, 3] = t
    return T


def moved(cloud, T):
    """the cloud seen from pose T: T^-1 applied to its points (float32 records)"""
    Ti = np.linalg.inv(T)
    p = cloud[:, :3].astype(np.float64) @ Ti[:3, :3].T + Ti[:3, 3]
    return records(p)
