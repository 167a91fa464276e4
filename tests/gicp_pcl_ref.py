"""Shared by the pcl GICP tests: the sequential CPU reference of pcl::GeneralizedIterativeClosestPoint (tests/gicp_pcl_ref.cpp,
compiled into a temporary directory) and the clouds the tests use."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "gicp_pcl_ref.cpp")
_VP = C.c_void_p
_SZ = C.c_size_t


def _p(a):
    return a.ctypes.data if a is not None else None


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def _row(T):
    return np.ascontiguousarray(T, np.float32).reshape(16)


class Reference:
    def __init__(self, tmpdir):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
        so = os.path.join(str(tmpdir), "libgicp_pcl_ref.so")
        subprocess.check_call([cxx, "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-variable", "-o", so, SRC])
        L = C.CDLL(so)
        L.ref_gicp_pcl_covariances.argtypes = [_VP, _SZ, _SZ, C.c_int, _VP]
        pair = [_VP, _SZ, _SZ, _VP, _VP, _SZ, _SZ, _VP, _VP]
        L.ref_gicp_pcl_correspondences.restype = _SZ
        L.ref_gicp_pcl_correspondences.argtypes = pair + [_VP, C.c_double, _VP, _VP]
        L.ref_gicp_pcl_cost.restype = _SZ
        L.ref_gicp_pcl_cost.argtypes = pair + [_VP, C.c_double, _VP, _VP]
        L.ref_gicp_pcl_fdf.restype = _SZ
        L.ref_gicp_pcl_fdf.argtypes = pair + [_VP, C.c_double, _VP, _VP, _VP]
        L.ref_gicp_pcl_apply_state.argtypes = [_VP, _VP]
        L.ref_gicp_pcl_align.restype = _SZ
        L.ref_gicp_pcl_align.argtypes = pair + [_VP, _VP, _VP, _VP, _VP, _SZ]
        self.lib = L

    def covariances(self, pts, k=20):
        a = _f32(pts)
        out = np.empty((a.shape[0], 3, 3))
        self.lib.ref_gicp_pcl_covariances(_p(a), a.shape[0], a.shape[1], k, _p(out))
        return out

    def _pair(self, src, scov, tgt, tcov, k):
        s, t = _f32(src), _f32(tgt)
        sc = np.ascontiguousarray(self.covariances(s, k) if scov is None else scov, np.float64)
        tc = np.ascontiguousarray(self.covariances(t, k) if tcov is None else tcov, np.float64)
        return (s, sc, t, tc), [_p(s), s.shape[0], s.shape[1], _p(sc), _p(t), t.shape[0], t.shape[1], _p(tc)]

    def correspondences(self, src, tgt, guess, T_rel, corr_dist=2.5, scov=None, tcov=None, k=20):
        keep, args = self._pair(src, scov, tgt, tcov, k)
        n = keep[0].shape[0]
        corr = np.empty(n, np.int32)
        M = np.empty((n, 3, 3))
        g, t = _row(guess), _row(T_rel)
        cnt = self.lib.ref_gicp_pcl_correspondences(*args, _p(g), _p(t), float(corr_dist), _p(corr), _p(M))
        return corr, M, cnt

    def cost(self, src, tgt, guess, T_rel, T, corr_dist=2.5, scov=None, tcov=None, k=20):
        keep, args = self._pair(src, scov, tgt, tcov, k)
        g, t, TT = _row(guess), _row(T_rel), _row(T)
        sums = np.empty(13)
        cnt = self.lib.ref_gicp_pcl_cost(*args, _p(g), _p(t), float(corr_dist), _p(TT), _p(sums))
        return sums, cnt

    def fdf(self, src, tgt, guess, T_rel, x, corr_dist=2.5, scov=None, tcov=None, k=20):
        keep, args = self._pair(src, scov, tgt, tcov, k)
        g, t = _row(guess), _row(T_rel)
        xv = np.ascontiguousarray(x, np.float64)
        f = np.empty(1)
        gr = np.empty(6)
        m = self.lib.ref_gicp_pcl_fdf(*args, _p(g), _p(t), float(corr_dist), _p(xv), _p(f), _p(gr))
        return f[0], gr, m

    def apply_state(self, x):
        xv = np.ascontiguousarray(x, np.float64)
        T = np.empty((4, 4), np.float32)
        self.lib.ref_gicp_pcl_apply_state(_p(xv), _p(T))
        return T

    def align(self, src, tgt, guess=None, max_iterations=64, max_optimizer_iterations=20, transformation_epsilon=0.01, rotation_epsilon=2e-3,
              corr_dist=2.5, k=20, scov=None, tcov=None, trace=False):
        keep, args = self._pair(src, scov, tgt, tcov, k)
        g = _row(np.eye(4) if guess is None else guess)
        cfg = np.array([transformation_epsilon, rotation_epsilon, corr_dist], np.float64)
        icfg = np.array([max_iterations, max_optimizer_iterations], np.int32)
        T = np.empty((4, 4), np.float32)
        stats = np.zeros(6, np.int64)
        cap = 5 * 4096 if trace else 0
        tr = np.empty(max(cap, 1))
        w = self.lib.ref_gicp_pcl_align(*args, _p(g), _p(cfg), _p(icfg), _p(T), _p(stats), _p(tr) if trace else None, cap)
        out = dict(T=T, converged=bool(stats[0]), iterations=int(stats[1]), corr_passes=int(stats[2]), cost_passes=int(stats[3]),
                   evaluations=int(stats[4]), bfgs_steps=int(stats[5]))
        if trace:
            out["trace"] = tr[:min(w, cap)].reshape(-1, 5)
        return out


def rot(rx, ry, rz):
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def pose(t=(0, 0, 0), r=(0, 0, 0)):
    T = np.eye(4)
    T[:3, :3] = rot(*r)
    T[:3, 3] = t
    return T.astype(np.float32)


def scene(n, seed=0, offset=(0.0, 0.0, 0.0)):
    """a small structured scene (floor, two walls, a box) of n points with 16 bytes per point"""
    rng = np.random.default_rng(seed)
    k = n // 4
    floor = np.c_[rng.uniform(-10, 10, k), rng.uniform(-10, 10, k), rng.normal(0, 0.01, k)]
    wall1 = np.c_[rng.uniform(-10, 10, k), np.full(k, 8.0) + rng.normal(0, 0.01, k), rng.uniform(0, 3, k)]
    wall2 = np.c_[np.full(k, -7.0) + rng.normal(0, 0.01, k), rng.uniform(-10, 10, k), rng.uniform(0, 3, k)]
    r = n - 3 * k
    box = np.c_[rng.uniform(1, 3, r), rng.uniform(-2, 0, r), rng.uniform(0, 2, r)]
    p = np.vstack([floor, wall1, wall2, box]) + np.asarray(offset)
    return np.c_[p, np.ones(n)].astype(np.float32)


def transform(pts, T):
    p = pts[:, :3].astype(np.float64) @ np.asarray(T, np.float64)[:3, :3].T + np.asarray(T, np.float64)[:3, 3]
    out = pts.copy()
    out[:, :3] = p.astype(np.float32)
    return out



def end_point_is_as_good(T, T_ref):
    """an engine align's end pose T against the reference's T_ref after the same outer iterations: equal to 1e-5, or, where the two
    BFGS line searches part in the last bits (fixed-tree against index-order sums), within 2e-3 in translation and rotation.  The
    outer loop only stops once a whole iteration moves the pose by less than transformation_epsilon (0.01 m) and rotation_epsilon
    (2e-3), so end points that far apart are the same answer to the stopping rule's resolution; a wrong optimiser step is larger."""
    dt = float(np.max(np.abs(np.asarray(T)[:3, 3] - np.asarray(T_ref)[:3, 3])))
    dr = float(np.max(np.abs(np.asarray(T)[:3, :3] - np.asarray(T_ref)[:3, :3])))
    assert (dt <= 1e-5 and dr <= 1e-5) or (dt <= 2e-3 and dr <= 2e-3), (dt, dr)
