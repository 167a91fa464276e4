"""Shared by the pcl NDT tests: the sequential CPU reference of pcl::NormalDistributionsTransform (tests/ndt_pcl_ref.cpp, compiled into
a temporary directory) on top of the oracle's voxel map, and the clouds the tests use."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "ndt_pcl_ref.cpp")
_VP = C.c_void_p


class Reference:
    def __init__(self, tmpdir):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
        so = os.path.join(str(tmpdir), "libndt_pcl_ref.so")
        # -ffp-contract=off as for the oracle: the reference is built without FMA
        subprocess.check_call([cxx, "-O2", "-fopenmp", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-variable",
                               "-o", so, SRC])
        L = C.CDLL(so)
        L.ref_pcl_map.restype = _VP
        L.ref_pcl_map.argtypes = [_VP, C.c_size_t, C.c_size_t, C.c_float, C.c_size_t, _VP, _VP, _VP, _VP, _VP, _VP]
        L.ref_pcl_free.argtypes = [_VP]
        L.ref_pcl_centroids.restype = C.c_size_t
        L.ref_pcl_centroids.argtypes = [_VP, _VP, _VP]
        L.ref_pcl_neighbors.restype = C.c_size_t
        L.ref_pcl_neighbors.argtypes = [_VP, _VP, C.c_size_t, C.c_size_t, _VP, _VP, _VP, _VP, _VP, C.c_size_t]
        L.ref_pcl_derivatives.restype = C.c_double
        L.ref_pcl_derivatives.argtypes = [_VP, _VP, C.c_size_t, C.c_size_t, _VP, _VP, _VP, _VP, _VP, _VP]
        L.ref_pcl_align.argtypes = [_VP, _VP, C.c_size_t, C.c_size_t, _VP, _VP, _VP, _VP, _VP, _VP]
        self.lib = L

    def map(self, tgt, resolution):
        return PclMap(self, tgt, resolution)


class PclMap:
    """pcl NDT target: the oracle's voxel map plus the searchable centroid cloud"""

    def __init__(self, ref, tgt, resolution):
        self.lib = ref.lib
        self.tgt = np.ascontiguousarray(tgt, np.float32)
        self.resolution = float(resolution)
        d = orc.NdtMap(self.tgt, resolution).dump()
        self.voxels = d
        self._keep = [np.ascontiguousarray(d[k]) for k in ("keys", "npts", "mean", "icov", "min_b", "div_b")]
        k, npts, mean, icov, minb, divb = self._keep
        self._m = _VP(self.lib.ref_pcl_map(self.tgt.ctypes.data, self.tgt.shape[0], self.tgt.shape[1], C.c_float(resolution), k.shape[0],
                                           k.ctypes.data, npts.ctypes.data, mean.ctypes.data, icov.ctypes.data, minb.ctypes.data, divb.ctypes.data))

    def __del__(self):
        try:
            self.lib.ref_pcl_free(self._m)
        except Exception:
            pass

    def _cfg(self, **kw):
        d = np.array([self.resolution, kw.get("step_size", 0.1), kw.get("outlier_ratio", 0.55), kw.get("transformation_epsilon", 0.01)], np.float64)
        i = np.array([kw.get("max_iterations", 64), kw.get("mt_interval_flag", 0), kw.get("fixed_iterations", 0), kw.get("threads", 0)], np.int32)
        return d, i

    def centroids(self):
        c = self.lib.ref_pcl_centroids(self._m, None, None)
        keys = np.empty(c, np.int64)
        xyz = np.empty((c, 3), np.float32)
        self.lib.ref_pcl_centroids(self._m, keys.ctypes.data, xyz.ctypes.data)
        return keys, xyz

    def neighbors(self, src, p, **kw):
        s = np.ascontiguousarray(src, np.float32)
        d, i = self._cfg(**kw)
        p = np.ascontiguousarray(p, np.float64)
        counts = np.zeros(max(s.shape[0], 1), np.uint32)
        total = self.lib.ref_pcl_neighbors(self._m, s.ctypes.data, s.shape[0], s.shape[1], d.ctypes.data, i.ctypes.data, p.ctypes.data,
                                           counts.ctypes.data, None, 0)
        keys = np.empty(max(total, 1), np.int64)
        self.lib.ref_pcl_neighbors(self._m, s.ctypes.data, s.shape[0], s.shape[1], d.ctypes.data, i.ctypes.data, p.ctypes.data,
                                   counts.ctypes.data, keys.ctypes.data, total)
        return counts[:s.shape[0]], keys[:total]

    def derivatives(self, src, p, **kw):
        s = np.ascontiguousarray(src, np.float32)
        d, i = self._cfg(**kw)
        p = np.ascontiguousarray(p, np.float64)
        g = np.empty(6)
        H = np.empty((6, 6))
        npairs = C.c_uint64()
        score = self.lib.ref_pcl_derivatives(self._m, s.ctypes.data, s.shape[0], s.shape[1], d.ctypes.data, i.ctypes.data, p.ctypes.data,
                                             g.ctypes.data, H.ctypes.data, C.addressof(npairs))
        return dict(score=score, g=g, H=H, n_pairs=npairs.value)

    def align(self, src, guess=None, **kw):
        s = np.ascontiguousarray(src, np.float32)
        d, i = self._cfg(**kw)
        g = np.ascontiguousarray(np.eye(4) if guess is None else guess, np.float32)
        T = np.empty((4, 4), np.float32)
        out = np.zeros(4, np.int32)
        p = np.zeros(6)
        self.lib.ref_pcl_align(self._m, s.ctypes.data, s.shape[0], s.shape[1], d.ctypes.data, i.ctypes.data, g.ctypes.data, T.ctypes.data,
                               out.ctypes.data, p.ctypes.data)
        return dict(T=T, converged=bool(out[0]), iterations=int(out[1]), derivative_passes=int(out[2]), hessian_passes=int(out[3]), p=p)


def records(xyz):
    """(n, 3) -> (n, 4) float32 x y z 1"""
    xyz = np.asarray(xyz, np.float32)
    return np.c_[xyz, np.ones(xyz.shape[0], np.float32)].astype(np.float32)


def room(n, seed=0):
    """a small structured scene: floor, two walls and a box, with sensor noise (planar and linear voxels included)"""
    rng = np.random.default_rng(seed)
    k = n // 4
    floor = np.c_[rng.uniform(-6, 6, k), rng.uniform(-6, 6, k), rng.normal(0, 0.01, k)]
    wall1 = np.c_[rng.uniform(-6, 6, k), np.full(k, 5.0) + rng.normal(0, 0.01, k), rng.uniform(0, 3, k)]
    wall2 = np.c_[np.full(k, -5.0) + rng.normal(0, 0.01, k), rng.uniform(-6, 6, k), rng.uniform(0, 3, k)]
    r = n - 3 * k
    box = np.c_[rng.uniform(1, 2.5, r), rng.uniform(-1, 0.5, r), rng.uniform(0, 1.2, r)]
    return records(np.r_[floor, wall1, wall2, box])


def pose_matrix(p):
    """(tx, ty, tz, rx, ry, rz) -> row-major 4x4 float32, Translation * Rx * Ry * Rz"""
    cx, cy, cz = np.cos(p[3:]); sx, sy, sz = np.sin(p[3:])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    T = np.eye(4)
    T[:3, :3] = Rx @ Ry @ Rz
    T[:3, 3] = p[:3]
    return T.astype(np.float32)


def outside_cell_voxel(leaf=0.1, start=3):
    """(x, n, k): n points at x = the largest float32 of cell k - 1 (floor(x * (1/leaf)) in float32) whose float32 centroid
    (sequential sum / n) lands in cell k, found by search"""
    f32 = np.float32
    inv = f32(1) / f32(leaf)
    for k in range(start, start + 400):
        x = f32(k * leaf)
        while np.floor(x * inv) >= k:
            x = np.nextafter(x, f32(-np.inf))
        while np.floor(np.nextafter(x, f32(np.inf)) * inv) < k:
            x = np.nextafter(x, f32(np.inf))
        for n in range(6, 120):
            c = np.add.accumulate(np.full(n, x, np.float32), dtype=np.float32)[-1] / f32(n)
            if np.floor(c * inv) >= k:
                return x, n, k
    raise AssertionError("no such voxel found")


def outside_scene(leaf=0.1, seed=0):
    """a target holding a voxel whose centroid lies in the next cell, on a noisy wall; and queries around that centroid"""
    x, n, k = outside_cell_voxel(leaf)
    rng = np.random.default_rng(seed)
    vox = np.c_[np.full(n, x, np.float32), rng.uniform(0.01, 0.09, n), rng.uniform(0.01, 0.09, n)]
    wall = np.c_[rng.uniform(-1, 1, 4000), rng.uniform(-1, 1, 4000), np.full(4000, 0.3) + rng.normal(0, 0.005, 4000)]
    c = np.float32(k * leaf)
    q = np.c_[c + rng.uniform(-1.5 * leaf, 1.5 * leaf, 3000), rng.uniform(-0.1, 0.2, 3000), rng.uniform(-0.1, 0.2, 3000)]
    return records(np.r_[vox, wall]), records(q), (x, n, k)
