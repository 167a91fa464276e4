"""Shared by the NDT_OMP KDTREE tests: the sequential CPU reference of pclomp::NormalDistributionsTransform with reg_nn_search_method =
KDTREE (tests/ndt_kdtree_ref.cpp, compiled into a temporary directory).  It is the oracle's NDT_OMP (oracle/ndt.cpp) over ndt_pcl_ref.cpp's
radius neighbourhood; both are compiled into the one library unchanged, so the pcl NDT entry points (ref_pcl_centroids /
ref_pcl_neighbors) and the oracle's are available beside the ref_kd_* ones."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "ndt_kdtree_ref.cpp")
_VP = C.c_void_p
_SZ = C.c_size_t


class Reference:
    def __init__(self, tmpdir):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
        so = os.path.join(str(tmpdir), "libndt_kdtree_ref.so")
        # -ffp-contract=off as for the oracle: the reference is built without FMA
        subprocess.check_call([cxx, "-O2", "-fopenmp", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-variable",
                               "-o", so, SRC])
        L = C.CDLL(so)
        L.ref_kd_map.restype = _VP
        L.ref_kd_map.argtypes = [_VP, _SZ, _SZ, C.c_float]
        L.ref_kd_free.argtypes = [_VP]
        L.ref_kd_voxels.restype = _VP
        L.ref_kd_voxels.argtypes = [_VP]
        L.ref_kd_search.restype = _VP
        L.ref_kd_search.argtypes = [_VP]
        L.ref_kd_derivatives.restype = C.c_double
        L.ref_kd_derivatives.argtypes = [_VP, _VP, _SZ, _SZ, _VP, _VP, _VP, _VP, _VP]
        L.ref_kd_hessian_at.argtypes = [_VP, _VP, _SZ, _SZ, _VP, _VP, _VP]
        L.ref_kd_align.argtypes = [_VP, _VP, _SZ, _SZ, _VP, _VP, _VP]
        L.orc_ndt_dump.restype = _SZ
        L.orc_ndt_dump.argtypes = [_VP] * 8
        L.ref_pcl_centroids.restype = _SZ
        L.ref_pcl_centroids.argtypes = [_VP, _VP, _VP]
        L.ref_pcl_neighbors.restype = _SZ
        L.ref_pcl_neighbors.argtypes = [_VP, _VP, _SZ, _SZ, _VP, _VP, _VP, _VP, _VP, _SZ]
        self.lib = L

    def map(self, tgt, resolution):
        return KdMap(self, tgt, resolution)


def _src(src):
    s = np.ascontiguousarray(src, np.float32)
    if s.ndim != 2 or s.shape[0] == 0:
        s = np.zeros((0, 4), np.float32) if s.size == 0 else s
    return s


class KdMap:
    """NDT_OMP target with the KDTREE neighbourhood: the oracle's voxel map and the centroid cloud on top of it"""

    def __init__(self, ref, tgt, resolution):
        self.lib = ref.lib
        self.tgt = np.ascontiguousarray(tgt, np.float32)
        self.resolution = float(resolution)
        self._m = _VP(self.lib.ref_kd_map(self.tgt.ctypes.data, self.tgt.shape[0], self.tgt.shape[1], C.c_float(resolution)))

    def __del__(self):
        try:
            self.lib.ref_kd_free(self._m)
        except Exception:
            pass

    def _cfg(self, **kw):
        return orc.NdtConfig(kw.get("max_iterations", 64), kw.get("transformation_epsilon", 0.01), kw.get("step_size", 0.1), kw.get("outlier_ratio", 0.55),
                             self.resolution, 7, kw.get("threads", 0), kw.get("mt_interval_flag", 0), kw.get("fixed_iterations", 0))

    def voxels(self):
        """the oracle's dump of the NDT_OMP voxel map (keys, npts, mean, cov, icov, min_b, div_b)"""
        om = self.lib.ref_kd_voxels(self._m)
        minb = np.zeros(3, np.int32)
        divb = np.zeros(3, np.int32)
        V = self.lib.orc_ndt_dump(om, None, None, None, None, None, minb.ctypes.data, divb.ctypes.data)
        keys = np.empty(V, np.int64)
        npts = np.empty(V, np.int32)
        mean = np.empty((V, 3))
        cov = np.empty((V, 3, 3))
        icov = np.empty((V, 3, 3))
        self.lib.orc_ndt_dump(om, keys.ctypes.data, npts.ctypes.data, mean.ctypes.data, cov.ctypes.data, icov.ctypes.data, minb.ctypes.data, divb.ctypes.data)
        return dict(keys=keys, npts=npts, mean=mean, cov=cov, icov=icov, min_b=minb, div_b=divb)

    def centroids(self):
        pm = self.lib.ref_kd_search(self._m)
        c = self.lib.ref_pcl_centroids(pm, None, None)
        keys = np.empty(c, np.int64)
        xyz = np.empty((c, 3), np.float32)
        self.lib.ref_pcl_centroids(pm, keys.ctypes.data, xyz.ctypes.data)
        return keys, xyz

    def neighbors(self, src, p):
        """radius neighbours of every source point at p: counts, and the leaf keys ascending within each point"""
        pm = self.lib.ref_kd_search(self._m)
        s = _src(src)
        d = np.array([self.resolution, 0.1, 0.55, 0.01], np.float64)
        i = np.array([64, 0, 0, 0], np.int32)
        p = np.ascontiguousarray(p, np.float64)
        counts = np.zeros(max(s.shape[0], 1), np.uint32)
        total = self.lib.ref_pcl_neighbors(pm, s.ctypes.data, s.shape[0], s.shape[1], d.ctypes.data, i.ctypes.data, p.ctypes.data, counts.ctypes.data, None, 0)
        keys = np.empty(max(total, 1), np.int64)
        self.lib.ref_pcl_neighbors(pm, s.ctypes.data, s.shape[0], s.shape[1], d.ctypes.data, i.ctypes.data, p.ctypes.data, counts.ctypes.data,
                                   keys.ctypes.data, total)
        return counts[:s.shape[0]], keys[:total]

    def derivatives(self, src, p, **kw):
        s = _src(src)
        cfg = self._cfg(**kw)
        p = np.ascontiguousarray(p, np.float64)
        g = np.empty(6)
        H = np.empty((6, 6))
        npairs = C.c_uint64()
        score = self.lib.ref_kd_derivatives(self._m, s.ctypes.data, s.shape[0], s.shape[1], C.addressof(cfg), p.ctypes.data, g.ctypes.data,
                                            H.ctypes.data, C.addressof(npairs))
        return dict(score=score, g=g, H=H, n_pairs=npairs.value)

    def hessian_at(self, src, p, **kw):
        s = _src(src)
        cfg = self._cfg(**kw)
        p = np.ascontiguousarray(p, np.float64)
        H = np.empty((6, 6))
        self.lib.ref_kd_hessian_at(self._m, s.ctypes.data, s.shape[0], s.shape[1], C.addressof(cfg), p.ctypes.data, H.ctypes.data)
        return H

    def align(self, src, guess=None, **kw):
        s = _src(src)
        cfg = self._cfg(**kw)
        g = np.ascontiguousarray(np.eye(4) if guess is None else guess, np.float32)
        res = orc.NdtResult()
        self.lib.ref_kd_align(self._m, s.ctypes.data, s.shape[0], s.shape[1], C.addressof(cfg), g.ctypes.data, C.addressof(res))
        return dict(T=np.array(res.T, np.float32).reshape(4, 4), converged=bool(res.converged), iterations=res.iterations, p=np.array(res.p),
                    derivative_passes=res.derivative_passes, hessian_passes=res.hessian_passes)
