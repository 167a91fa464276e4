"""ctypes wrapper of oracle/liboracle.so — TEST INFRASTRUCTURE ONLY (see oracle/oracle.h).

Importable only from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
All matrices row-major numpy; clouds float32 (n, stride)."""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATH = os.path.join(_HERE, "liboracle.so")
_lib = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("gicp.cpp", "ndt.cpp", "oracle.h", "kdtree.hpp", "linalg.hpp", "Makefile")]
    if force or not os.path.exists(_PATH) or any(os.path.getmtime(s) > os.path.getmtime(_PATH) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _PATH


class GicpConfig(C.Structure):
    _fields_ = [("max_iterations", C.c_int), ("transformation_epsilon", C.c_double), ("rotation_epsilon", C.c_double),
                ("max_corr_dist", C.c_double), ("k_correspondences", C.c_int), ("num_threads", C.c_int)]


class GicpResult(C.Structure):
    _fields_ = [("T", C.c_float * 16), ("T64", C.c_double * 16), ("converged", C.c_int), ("iterations", C.c_int), ("lm_failed", C.c_int),
                ("last_error", C.c_double), ("total_inner", C.c_int)]


class NdtConfig(C.Structure):
    _fields_ = [("max_iterations", C.c_int), ("transformation_epsilon", C.c_double), ("step_size", C.c_double), ("outlier_ratio", C.c_double),
                ("resolution", C.c_double), ("search_method", C.c_int), ("num_threads", C.c_int), ("mt_interval_flag", C.c_int),
                ("fixed_iterations", C.c_int)]


class NdtResult(C.Structure):
    _fields_ = [("T", C.c_float * 16), ("converged", C.c_int), ("iterations", C.c_int), ("trans_probability", C.c_double), ("p", C.c_double * 6),
                ("derivative_passes", C.c_uint64), ("hessian_passes", C.c_uint64)]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            build()
        _lib = C.CDLL(_PATH)
        _lib.orc_gicp_linearize.restype = C.c_double
        _lib.orc_gicp_error.restype = C.c_double
        _lib.orc_ndt_derivatives.restype = C.c_double
        _lib.orc_ndt_build.restype = C.c_void_p
        _lib.orc_ndt_dump.restype = C.c_size_t
        _lib.orc_max_threads.restype = C.c_int
        _lib.orc_gicp_target_create.restype = C.c_void_p
        _lib.orc_gicp_target_fitness.restype = C.c_double
    return _lib


def _f32(a):
    a = np.ascontiguousarray(a, np.float32)
    return a, a.ctypes.data_as(C.c_void_p), a.shape[0], a.shape[1]


def max_threads():
    return lib().orc_max_threads()


def knn(pts, queries, k, threads=0):
    p, pp, n, s = _f32(pts)
    q, qp, nq, qs = _f32(queries)
    idx = np.empty((nq, k), np.int32)
    d2 = np.empty((nq, k), np.float32)
    lib().orc_knn(pp, C.c_size_t(n), C.c_size_t(s), qp, C.c_size_t(nq), C.c_size_t(qs), k, idx.ctypes.data_as(C.c_void_p), d2.ctypes.data_as(C.c_void_p), threads)
    return idx, d2


def gicp_covariances(pts, k=20, threads=0):
    p, pp, n, s = _f32(pts)
    cov = np.empty((n, 3, 3), np.float64)
    lib().orc_gicp_covariances(pp, C.c_size_t(n), C.c_size_t(s), k, cov.ctypes.data_as(C.c_void_p), threads)
    return cov


def gicp_linearize(src, src_cov, tgt, tgt_cov, T, max_corr_dist=2.5, threads=0):
    sa, sp, n, ss = _f32(src)
    ta, tp, m, ts = _f32(tgt)
    T = np.ascontiguousarray(T, np.float64)
    sc = np.ascontiguousarray(src_cov, np.float64)
    tc = np.ascontiguousarray(tgt_cov, np.float64)
    corr = np.empty(n, np.int32)
    d2 = np.empty(n, np.float32)
    mahal = np.zeros((n, 3, 3), np.float64)
    H = np.empty((6, 6), np.float64)
    b = np.empty(6, np.float64)
    vp = C.c_void_p
    e = lib().orc_gicp_linearize(sp, C.c_size_t(n), C.c_size_t(ss), sc.ctypes.data_as(vp), tp, C.c_size_t(m), C.c_size_t(ts), tc.ctypes.data_as(vp),
                                 T.ctypes.data_as(vp), C.c_double(max_corr_dist), corr.ctypes.data_as(vp), d2.ctypes.data_as(vp), mahal.ctypes.data_as(vp),
                                 H.ctypes.data_as(vp), b.ctypes.data_as(vp), threads)
    return dict(corr=corr, d2=d2, mahal=mahal, H=H, b=b, err=e)


def gicp_error(src, tgt, corr, mahal, T, threads=0):
    sa, sp, n, ss = _f32(src)
    ta, tp, m, ts = _f32(tgt)
    T = np.ascontiguousarray(T, np.float64)
    vp = C.c_void_p
    return lib().orc_gicp_error(sp, C.c_size_t(n), C.c_size_t(ss), tp, C.c_size_t(ts), np.ascontiguousarray(corr, np.int32).ctypes.data_as(vp),
                                np.ascontiguousarray(mahal, np.float64).ctypes.data_as(vp), T.ctypes.data_as(vp), threads)


def gicp_align(src, tgt, guess=None, max_iterations=64, transformation_epsilon=0.01, rotation_epsilon=2e-3, max_corr_dist=2.5, k=20,
               threads=0, src_cov=None, tgt_cov=None, trace=False):
    sa, sp, n, ss = _f32(src)
    ta, tp, m, ts = _f32(tgt)
    cfg = GicpConfig(max_iterations, transformation_epsilon, rotation_epsilon, max_corr_dist, k, threads)
    g = np.ascontiguousarray(np.eye(4) if guess is None else guess, np.float32)
    res = GicpResult()
    vp = C.c_void_p
    corr = np.empty(max(n, 1), np.int32)
    tH = np.zeros((max_iterations, 6, 6)) if trace else None
    tb = np.zeros((max_iterations, 6)) if trace else None
    ty = np.zeros(max_iterations) if trace else None
    scp = np.ascontiguousarray(src_cov, np.float64).ctypes.data_as(vp) if src_cov is not None else None
    tcp = np.ascontiguousarray(tgt_cov, np.float64).ctypes.data_as(vp) if tgt_cov is not None else None
    lib().orc_gicp_align(sp, C.c_size_t(n), C.c_size_t(ss), scp, tp, C.c_size_t(m), C.c_size_t(ts), tcp, C.byref(cfg), g.ctypes.data_as(vp), C.byref(res),
                         tH.ctypes.data_as(vp) if trace else None, tb.ctypes.data_as(vp) if trace else None, ty.ctypes.data_as(vp) if trace else None,
                         corr.ctypes.data_as(vp))
    out = dict(T=np.array(res.T, np.float32).reshape(4, 4), T64=np.array(res.T64).reshape(4, 4), converged=bool(res.converged), iterations=res.iterations,
               lm_failed=bool(res.lm_failed), last_error=res.last_error, total_inner=res.total_inner, corr=corr[:n])
    if trace:
        out.update(trace_H=tH, trace_b=tb, trace_y=ty)
    return out


class GicpTarget:
    """a kept target (kd-tree + covariances built once), as fast_gicp keeps it while the same target cloud stays set"""

    def __init__(self, tgt, k=20, threads=0):
        ta, tp, m, ts = _f32(tgt)
        self._keep = ta
        self._t = C.c_void_p(lib().orc_gicp_target_create(tp, C.c_size_t(m), C.c_size_t(ts), k, threads))

    def __del__(self):
        try:
            lib().orc_gicp_target_free(self._t)
        except Exception:
            pass

    def align(self, src, guess=None, max_iterations=64, transformation_epsilon=0.01, rotation_epsilon=2e-3, max_corr_dist=2.5, k=20, threads=0,
              src_cov=None):
        sa, sp, n, ss = _f32(src)
        cfg = GicpConfig(max_iterations, transformation_epsilon, rotation_epsilon, max_corr_dist, k, threads)
        g = np.ascontiguousarray(np.eye(4) if guess is None else guess, np.float32)
        res = GicpResult()
        vp = C.c_void_p
        corr = np.empty(max(n, 1), np.int32)
        scp = np.ascontiguousarray(src_cov, np.float64).ctypes.data_as(vp) if src_cov is not None else None
        lib().orc_gicp_align_to(self._t, sp, C.c_size_t(n), C.c_size_t(ss), scp, C.byref(cfg), g.ctypes.data_as(vp), C.byref(res), corr.ctypes.data_as(vp))
        return dict(T=np.array(res.T, np.float32).reshape(4, 4), converged=bool(res.converged), iterations=res.iterations, corr=corr[:n])

    def fitness(self, src, T, max_range=np.finfo(np.float64).max, threads=0):
        sa, sp, n, ss = _f32(src)
        T = np.ascontiguousarray(T, np.float32)
        return lib().orc_gicp_target_fitness(self._t, sp, C.c_size_t(n), C.c_size_t(ss), T.ctypes.data_as(C.c_void_p), C.c_double(max_range), threads)


def fitness(tgt, src, T, max_range=np.finfo(np.float64).max, inlier_thresh_sq=0.25, threads=0, want_nn=False):
    ta, tp, m, ts = _f32(tgt)
    sa, sp, n, ss = _f32(src)
    T = np.ascontiguousarray(T, np.float32)
    score, nr, inl = C.c_double(), C.c_uint32(), C.c_uint32()
    idx = np.empty(max(n, 1), np.int32)
    d2 = np.empty(max(n, 1), np.float32)
    vp = C.c_void_p
    lib().orc_fitness(tp, C.c_size_t(m), C.c_size_t(ts), sp, C.c_size_t(n), C.c_size_t(ss), T.ctypes.data_as(vp), C.c_double(max_range),
                      C.c_float(inlier_thresh_sq), C.byref(score), C.byref(nr), C.byref(inl), idx.ctypes.data_as(vp), d2.ctypes.data_as(vp), threads)
    if want_nn:
        return score.value, nr.value, inl.value, idx[:n], d2[:n]
    return score.value, nr.value, inl.value


def voxelgrid(cloud, leaf):
    a, ap, n, s = _f32(cloud)
    out = np.zeros((max(n, 1), 4), np.float32)
    keys = np.empty(max(n, 1), np.int32)
    counts = np.empty(max(n, 1), np.int32)
    n_out = C.c_size_t()
    vp = C.c_void_p
    rc = lib().orc_voxelgrid(ap, C.c_size_t(n), C.c_size_t(s), C.c_float(leaf), out.ctypes.data_as(vp), keys.ctypes.data_as(vp), counts.ctypes.data_as(vp), C.byref(n_out))
    m = n_out.value
    return out[:m], keys[:m], counts[:m], rc


def distance_filter(cloud, near, far):
    a, ap, n, s = _f32(cloud)
    keep = np.zeros(max(n, 1), np.uint8)
    lib().orc_distance_filter(ap, C.c_size_t(n), C.c_size_t(s), C.c_double(near), C.c_double(far), keep.ctypes.data_as(C.c_void_p))
    return keep[:n].astype(bool)


def radius_outlier(cloud, radius, min_neighbors, threads=0):
    a, ap, n, s = _f32(cloud)
    keep = np.zeros(max(n, 1), np.uint8)
    lib().orc_radius_outlier(ap, C.c_size_t(n), C.c_size_t(s), C.c_double(radius), int(min_neighbors), keep.ctypes.data_as(C.c_void_p), threads)
    return keep[:n].astype(bool)


def statistical_outlier(cloud, mean_k, stddev_mul, threads=0):
    a, ap, n, s = _f32(cloud)
    keep = np.zeros(max(n, 1), np.uint8)
    dist = np.zeros(max(n, 1), np.float32)
    lib().orc_statistical_outlier(ap, C.c_size_t(n), C.c_size_t(s), int(mean_k), C.c_double(stddev_mul), keep.ctypes.data_as(C.c_void_p),
                                  dist.ctypes.data_as(C.c_void_p), threads)
    return keep[:n].astype(bool), dist[:n]


def deskew(cloud, scan_period, angular_velocity):
    a, ap, n, s = _f32(cloud)
    out = np.zeros_like(a)
    w = np.ascontiguousarray(angular_velocity, np.float32)
    lib().orc_deskew(ap, C.c_size_t(n), C.c_size_t(s), C.c_double(scan_period), w.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    return out


def map_cloud_generate(keyframes, resolution):
    """MapCloudGenerator::generate (/root/reference/src/hdl_graph_slam/map_cloud_generator.cpp:13-51) restated with numpy, including
    pcl::octree::OctreePointCloud's SEQUENTIAL bounding-box growth (adoptBoundingBoxToPoint, UPSTREAM-RECALL of PCL 1.10): the box
    starts at p0 -+ resolution/2 and doubles towards each violating point; keys are (point - min) / resolution in float64; centres
    (key + 0.5) * resolution + min with the FINAL min.  Returns the concatenated cloud (n, 5: x y z 1 intensity) when
    resolution <= 0, else the occupied voxel centres (m, 3) as float32, in ascending lexicographic order."""
    pts = []
    for cloud, pose in keyframes:
        c = np.asarray(cloud, np.float32)
        P = np.asarray(pose, np.float64).astype(np.float32)
        x, y, z = c[:, 0], c[:, 1], c[:, 2]
        o = np.zeros((c.shape[0], 5), np.float32)
        for r in range(3):  # ((m0 x + m1 y) + m2 z) + m3, float32
            o[:, r] = ((P[r, 0] * x + P[r, 1] * y).astype(np.float32) + (P[r, 2] * z).astype(np.float32)).astype(np.float32) + P[r, 3]
        o[:, 3] = 1.0
        o[:, 4] = c[:, 4] if c.shape[1] > 4 else 0.0
        pts.append(o)
    cloud = np.concatenate(pts) if pts else np.zeros((0, 5), np.float32)
    if not (resolution > 0):
        return cloud
    res = float(resolution)
    eps = float(np.finfo(np.float32).eps)
    mn, mx, depth, defined = np.zeros(3), np.zeros(3), 0, False
    xyz = cloud[:, :3].astype(np.float64)
    finite = np.isfinite(xyz).all(axis=1)
    # points that violate the current box are rare after the first few: scan in chunks and only loop over violators
    i, n = 0, xyz.shape[0]
    while i < n:
        if not finite[i]:
            i += 1
            continue
        p = xyz[i]
        while True:
            lower, upper = p < mn, p >= mx
            if defined and not (lower.any() or upper.any()):
                break
            if defined:
                side = float(1 << depth) * res
                mn = np.where(~upper, mn - side, mn)
                depth += 1
                side = float(1 << depth) * res - eps
                mx = mn + side
            else:
                mn, mx, defined = p - res / 2, p + res / 2, True
        # skip ahead to the next violator
        rest = xyz[i + 1:]
        bad = ((rest < mn) | (rest >= mx)).any(axis=1) & finite[i + 1:]
        nxt = np.flatnonzero(bad)
        i = i + 1 + (int(nxt[0]) if nxt.size else rest.shape[0])
    keys = np.floor((xyz[finite] - mn) / res).astype(np.int64)
    uniq = np.unique(keys, axis=0)
    centres = ((uniq.astype(np.float64) + 0.5) * res + mn).astype(np.float32)
    order = np.lexsort((centres[:, 0], centres[:, 1], centres[:, 2]))
    return centres[order]


class NdtMap:
    def __init__(self, tgt, resolution):
        ta, tp, m, ts = _f32(tgt)
        self._keep = ta
        self._m = C.c_void_p(lib().orc_ndt_build(tp, C.c_size_t(m), C.c_size_t(ts), C.c_float(resolution)))
        self.resolution = resolution

    def __del__(self):
        try:
            lib().orc_ndt_free(self._m)
        except Exception:
            pass

    def dump(self):
        vp = C.c_void_p
        minb = np.zeros(3, np.int32)
        divb = np.zeros(3, np.int32)
        V = lib().orc_ndt_dump(self._m, None, None, None, None, None, minb.ctypes.data_as(vp), divb.ctypes.data_as(vp))
        keys = np.empty(V, np.int64)
        npts = np.empty(V, np.int32)
        mean = np.empty((V, 3))
        cov = np.empty((V, 3, 3))
        icov = np.empty((V, 3, 3))
        lib().orc_ndt_dump(self._m, keys.ctypes.data_as(vp), npts.ctypes.data_as(vp), mean.ctypes.data_as(vp), cov.ctypes.data_as(vp), icov.ctypes.data_as(vp),
                           minb.ctypes.data_as(vp), divb.ctypes.data_as(vp))
        return dict(keys=keys, npts=npts, mean=mean, cov=cov, icov=icov, min_b=minb, div_b=divb)

    def _cfg(self, **kw):
        return NdtConfig(kw.get("max_iterations", 64), kw.get("transformation_epsilon", 0.01), kw.get("step_size", 0.1), kw.get("outlier_ratio", 0.55),
                         self.resolution, kw.get("search_method", 7), kw.get("threads", 0), kw.get("mt_interval_flag", 0), kw.get("fixed_iterations", 0))

    def derivatives(self, src, p, **kw):
        sa, sp, n, ss = _f32(src)
        cfg = self._cfg(**kw)
        p = np.ascontiguousarray(p, np.float64)
        g = np.empty(6)
        H = np.empty((6, 6))
        npairs = C.c_uint64()
        cells = np.empty(max(n, 1), np.uint8)
        vp = C.c_void_p
        score = lib().orc_ndt_derivatives(self._m, sp, C.c_size_t(n), C.c_size_t(ss), C.byref(cfg), p.ctypes.data_as(vp), g.ctypes.data_as(vp), H.ctypes.data_as(vp),
                                          C.byref(npairs), cells.ctypes.data_as(vp))
        return dict(score=score, g=g, H=H, n_pairs=npairs.value, cells=cells[:n])

    def hessian_at(self, src, p, **kw):
        """the float64 computeHessian pass alone at p: H (6, 6)"""
        sa, sp, n, ss = _f32(src)
        cfg = self._cfg(**kw)
        p = np.ascontiguousarray(p, np.float64)
        H = np.empty((6, 6))
        vp = C.c_void_p
        lib().orc_ndt_hessian_at(self._m, sp, C.c_size_t(n), C.c_size_t(ss), C.byref(cfg), p.ctypes.data_as(vp), H.ctypes.data_as(vp))
        return H

    def align(self, src, guess=None, trace=False, **kw):
        sa, sp, n, ss = _f32(src)
        cfg = self._cfg(**kw)
        g = np.ascontiguousarray(np.eye(4) if guess is None else guess, np.float32)
        res = NdtResult()
        tp = np.zeros((cfg.max_iterations + 4, 6)) if trace else None
        lib().orc_ndt_align(self._m, sp, C.c_size_t(n), C.c_size_t(ss), C.byref(cfg), g.ctypes.data_as(C.c_void_p), C.byref(res),
                            tp.ctypes.data_as(C.c_void_p) if trace else None)
        out = dict(T=np.array(res.T, np.float32).reshape(4, 4), converged=bool(res.converged), iterations=res.iterations,
                   trans_probability=res.trans_probability, p=np.array(res.p), derivative_passes=res.derivative_passes,
                   hessian_passes=res.hessian_passes)
        if trace:
            out["trace_p"] = tp
        return out
