"""Host-side mirror of the reference's registration interface, as thin wrappers over the C ABI (libb200reg.so).

Names follow the reference so that tests read like its call sites:
  select_registration_method   <- src/hdl_graph_slam/registrations.cpp:22-124
  Registration.setInputTarget / setInputSource / align / hasConverged / getFinalTransformation / getFitnessScore
                               <- pcl::Registration<PointXYZI,PointXYZI> as used at
                                  apps/scan_matching_odometry_nodelet.cpp:172,177,210,214,220,246,307 and
                                  include/hdl_graph_slam/loop_detector.hpp:122,136,143,146,147,153
  ScanMatchingOdometry.matching <- apps/scan_matching_odometry_nodelet.cpp:165-262
  ScanMatchingOdometry.aligned  <- its aligned_points cloud (:254-259)
  LoopDetector.matching         <- include/hdl_graph_slam/loop_detector.hpp:117-171
  VoxelGrid.filter              <- pcl::VoxelGrid as set up at apps/prefiltering_nodelet.cpp:54-58
  approximateVoxelGridFilter    <- pcl::ApproximateVoxelGrid as set up at apps/prefiltering_nodelet.cpp:61-63

Clouds are float32 numpy arrays of shape (n, 4) [x,y,z,1] or (n, 8) [pcl::PointXYZI record]; 4x4 poses are ordinary
row-major numpy matrices (the wrapper converts to the ABI's column-major layout).  All arithmetic happens in the CUDA
library; nothing here computes.
"""
import ctypes as C
import numpy as np
from . import _capi
from ._capi import Config, Result, Pair, OdometryParams, OdometryStatus, Stats, check, B2R_METHOD_GICP, B2R_METHOD_NDT, B2R_METHOD_NDT_PCL, B2R_METHOD_VGICP, B2R_METHOD_GICP_PCL, B2R_METHOD_ICP_PCL, B2R_METHOD_VGICP_CUDA, B2R_METHOD_GICP_OMP, B2R_METHOD_NDT_KDTREE  # noqa: F401


def _cloud(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.ndim != 2 or a.shape[1] < 3:
        raise ValueError("cloud must be (n, >=3) float32")
    return a, a.shape[0], a.shape[1] * 4


def _colmajor(T, dtype=np.float32):
    return np.ascontiguousarray(np.asarray(T, dtype=dtype).T.reshape(-1))


def _from_colmajor(buf):
    return np.array(buf, dtype=np.float32).reshape(4, 4).T.copy()


def default_config(method):
    lib = _capi.load()
    cfg = Config()
    check(lib.b2r_config_default(C.byref(cfg), method))
    return cfg


class Registration:
    """One registration handle (== one pcl::Registration object of the reference)."""

    def __init__(self, cfg=None, _handle=None):
        self._lib = _capi.load()
        self._h = C.c_void_p()
        if _handle is not None:
            self._h = _handle
        else:
            check(self._lib.b2r_create(C.byref(cfg), C.byref(self._h)))
        self._res = Result()
        self._res.converged = 0
        self._keep = {}

    def close(self):
        if self._h:
            self._lib.b2r_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def config(self):
        cfg = Config()
        check(self._lib.b2r_get_config(self._h, C.byref(cfg)))
        return cfg

    # --- pcl::Registration surface
    def setInputTarget(self, cloud):
        a, n, s = _cloud(cloud)
        self._keep["t"] = a
        check(self._lib.b2r_set_target(self._h, a.ctypes.data_as(C.c_void_p), n, s))

    def setInputSource(self, cloud):
        a, n, s = _cloud(cloud)
        self._keep["s"] = a
        check(self._lib.b2r_set_source(self._h, a.ctypes.data_as(C.c_void_p), n, s))

    def setInputTargetDevice(self, ptr, n, stride_bytes):
        check(self._lib.b2r_set_target_device(self._h, C.c_void_p(ptr), n, stride_bytes))

    def setInputSourceDevice(self, ptr, n, stride_bytes):
        check(self._lib.b2r_set_source_device(self._h, C.c_void_p(ptr), n, stride_bytes))

    def setInputTargetRaw(self, ptr, n, stride_bytes):
        """host pointer variant (e.g. pinned memory owned by the caller)"""
        check(self._lib.b2r_set_target(self._h, C.c_void_p(ptr), n, stride_bytes))

    def setInputSourceRaw(self, ptr, n, stride_bytes):
        check(self._lib.b2r_set_source(self._h, C.c_void_p(ptr), n, stride_bytes))

    def prefetchSourceRaw(self, ptr, n, stride_bytes, device=False):
        fn = self._lib.b2r_prefetch_source_device if device else self._lib.b2r_prefetch_source
        check(fn(self._h, C.c_void_p(ptr), n, stride_bytes))

    def prefetchSource(self, cloud):
        a, n, s = _cloud(cloud)
        self._keep["p"] = a
        check(self._lib.b2r_prefetch_source(self._h, a.ctypes.data_as(C.c_void_p), n, s))

    def synchronize(self):
        check(self._lib.b2r_synchronize(self._h))

    def setProfiling(self, on):
        check(self._lib.b2r_set_profiling(self._h, int(bool(on))))

    def getStats(self, reset=False):
        st = Stats()
        check(self._lib.b2r_get_stats(self._h, C.byref(st), int(reset)))
        names = [self._lib.b2r_kernel_class_name(i).decode() for i in range(st.n_classes)]
        return dict(h2d_bytes=int(st.h2d_bytes), d2h_bytes=int(st.d2h_bytes),
                    launches={n: int(st.launches[i]) for i, n in enumerate(names)},
                    calls={n: int(st.calls[i]) for i, n in enumerate(names)},
                    ms={n: float(st.ms[i]) for i, n in enumerate(names)})

    def getStream(self):
        p = C.c_void_p()
        check(self._lib.b2r_get_stream(self._h, C.byref(p)))
        return p.value

    def promoteSourceToTarget(self):
        check(self._lib.b2r_promote_source_to_target(self._h))

    def align(self, guess=None, want_aligned=False):
        g = _colmajor(np.eye(4) if guess is None else guess)
        check(self._lib.b2r_align(self._h, g.ctypes.data_as(C.POINTER(C.c_float)), C.byref(self._res)))
        if want_aligned:
            return self.getAligned()
        return None

    def getAligned(self):
        src = self._keep.get("s")
        if src is None:
            raise RuntimeError("getAligned needs a host source cloud")
        out = src.copy()
        check(self._lib.b2r_get_aligned(self._h, out.ctypes.data_as(C.c_void_p), out.shape[0], out.shape[1] * 4))
        return out

    def hasConverged(self):
        return bool(self._res.converged)

    def getFinalTransformation(self):
        return _from_colmajor(self._res.T)

    @property
    def nr_iterations(self):
        return int(self._res.iterations)

    def getFitnessScore(self, max_range=np.finfo(np.float64).max, T=None, inlier_thresh_sq=0.25, full=False):
        score, used, inl = C.c_double(), C.c_uint32(), C.c_uint32()
        tp = None
        if T is not None:
            t = _colmajor(T)
            tp = t.ctypes.data_as(C.POINTER(C.c_float))
        check(self._lib.b2r_fitness(self._h, tp, max_range, inlier_thresh_sq, C.byref(score), C.byref(used), C.byref(inl)))
        if full:
            return score.value, used.value, inl.value
        return score.value

    def nearestKSearch(self, queries):
        """getSearchMethodTarget()->nearestKSearch(pt, 1, ...) for many points: (indices, squared distances)"""
        a, n, s = _cloud(queries)
        idx = np.empty(n, np.int32)
        d2 = np.empty(n, np.float32)
        check(self._lib.b2r_target_nearest(self._h, a.ctypes.data_as(C.c_void_p), n, s, idx.ctypes.data_as(C.POINTER(C.c_int32)),
                                           d2.ctypes.data_as(C.POINTER(C.c_float))))
        return idx, d2

    # --- parity taps
    def getCorrespondences(self, n):
        out = np.empty(n, np.int32)
        check(self._lib.b2r_get_correspondences(self._h, out.ctypes.data_as(C.POINTER(C.c_int32)), n))
        return out

    def getCovariances(self, which, n):
        out = np.empty((n, 3, 3), np.float64)
        check(self._lib.b2r_get_covariances(self._h, which, out.ctypes.data_as(C.POINTER(C.c_double)), n))
        return out

    def gicpLinearizeAt(self, T):
        t = _colmajor(T, np.float64)
        H = np.empty((6, 6), np.float64)
        b = np.empty(6, np.float64)
        e = C.c_double()
        dp = C.POINTER(C.c_double)
        check(self._lib.b2r_gicp_linearize_at(self._h, t.ctypes.data_as(dp), H.ctypes.data_as(dp), b.ctypes.data_as(dp), C.byref(e)))
        return H, b, e.value

    def gicpErrorAt(self, T):
        t = _colmajor(T, np.float64)
        e = C.c_double()
        check(self._lib.b2r_gicp_error_at(self._h, t.ctypes.data_as(C.POINTER(C.c_double)), C.byref(e)))
        return e.value

    def ndtGetVoxels(self):
        nv = C.c_size_t()
        minb = np.zeros(3, np.int32)
        divb = np.zeros(3, np.int32)
        ip = C.POINTER(C.c_int32)
        check(self._lib.b2r_ndt_get_voxels(self._h, 0, C.byref(nv), None, None, None, None, minb.ctypes.data_as(ip), divb.ctypes.data_as(ip)))
        V = nv.value
        keys = np.empty(V, np.int64)
        npts = np.empty(V, np.int32)
        mean = np.empty((V, 3), np.float64)
        icov = np.empty((V, 3, 3), np.float64)
        dp = C.POINTER(C.c_double)
        check(self._lib.b2r_ndt_get_voxels(self._h, V, C.byref(nv), keys.ctypes.data_as(C.POINTER(C.c_int64)), npts.ctypes.data_as(ip),
                                           mean.ctypes.data_as(dp), icov.ctypes.data_as(dp), minb.ctypes.data_as(ip), divb.ctypes.data_as(ip)))
        return dict(keys=keys, npts=npts, mean=mean, icov=icov, min_b=minb, div_b=divb)

    def ndtDerivativesAt(self, p):
        p = np.ascontiguousarray(p, np.float64)
        g = np.empty(6, np.float64)
        H = np.empty((6, 6), np.float64)
        score = C.c_double()
        npairs = C.c_uint64()
        dp = C.POINTER(C.c_double)
        check(self._lib.b2r_ndt_derivatives_at(self._h, p.ctypes.data_as(dp), C.byref(score), g.ctypes.data_as(dp), H.ctypes.data_as(dp), C.byref(npairs)))
        return score.value, g, H, npairs.value

    def ndtHessianAt(self, p):
        """the float64 Hessian pass alone (computeHessian, run after an active More-Thuente line search) at p: H (6, 6)"""
        p = np.ascontiguousarray(p, np.float64)
        H = np.empty((6, 6), np.float64)
        dp = C.POINTER(C.c_double)
        check(self._lib.b2r_ndt_hessian_at(self._h, p.ctypes.data_as(dp), H.ctypes.data_as(dp)))
        return H

    def ndtGetCentroids(self):
        """(pcl NDT) the searchable centroid cloud of the target: (leaf keys (m,) int64 ascending, centroids (m, 3) float32)"""
        nc = C.c_size_t()
        check(self._lib.b2r_ndt_get_centroids(self._h, 0, C.byref(nc), None, None))
        keys = np.empty(nc.value, np.int64)
        xyz = np.empty((nc.value, 3), np.float32)
        check(self._lib.b2r_ndt_get_centroids(self._h, nc.value, C.byref(nc), keys.ctypes.data_as(C.POINTER(C.c_int64)),
                                              xyz.ctypes.data_as(C.POINTER(C.c_float))))
        return keys, xyz

    def ndtNeighborsAt(self, p, n_source):
        """(pcl NDT) radius neighbours of every source point at p: (counts (n,) uint32, leaf keys (sum counts,) int64, CSR)"""
        p = np.ascontiguousarray(p, np.float64)
        dp = C.POINTER(C.c_double)
        counts = np.zeros(max(n_source, 1), np.uint32)
        total = C.c_size_t()
        check(self._lib.b2r_ndt_neighbors_at(self._h, p.ctypes.data_as(dp), counts.ctypes.data_as(C.POINTER(C.c_uint32)), 0, None, C.byref(total)))
        keys = np.empty(max(total.value, 1), np.int64)
        check(self._lib.b2r_ndt_neighbors_at(self._h, p.ctypes.data_as(dp), counts.ctypes.data_as(C.POINTER(C.c_uint32)), total.value,
                                             keys.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(total)))
        return counts[:n_source], keys[:total.value]

    def vgicpGetVoxels(self):
        """(VGICP, VGICP_CUDA) the target's Gaussian voxel map, cells ascending: dict(cells (V, 3) int32, counts (V,), mean (V, 3), cov (V, 3, 3))"""
        nv = C.c_size_t()
        check(self._lib.b2r_vgicp_get_voxels(self._h, 0, C.byref(nv), None, None, None, None))
        V = nv.value
        cells = np.empty((V, 3), np.int32)
        counts = np.empty(V, np.int32)
        mean = np.empty((V, 3), np.float64)
        cov = np.empty((V, 3, 3), np.float64)
        ip, dp = C.POINTER(C.c_int32), C.POINTER(C.c_double)
        check(self._lib.b2r_vgicp_get_voxels(self._h, V, C.byref(nv), cells.ctypes.data_as(ip), counts.ctypes.data_as(ip), mean.ctypes.data_as(dp),
                                             cov.ctypes.data_as(dp)))
        return dict(cells=cells, counts=counts, mean=mean, cov=cov)

    def vgicpLinearizeAt(self, T, n_source):
        """(VGICP, VGICP_CUDA) one voxel-correspondence update + linearisation at T: (H (6, 6), b (6,), cost, correspondence count, voxel of every
        source point (n,) int32, -1 = none)"""
        t = _colmajor(T, np.float64)
        H = np.empty((6, 6), np.float64)
        b = np.empty(6, np.float64)
        cost = C.c_double()
        nc = C.c_uint64()
        vox = np.empty(max(n_source, 1), np.int32)
        dp = C.POINTER(C.c_double)
        check(self._lib.b2r_vgicp_linearize_at(self._h, t.ctypes.data_as(dp), H.ctypes.data_as(dp), b.ctypes.data_as(dp), C.byref(cost), C.byref(nc),
                                               vox.ctypes.data_as(C.POINTER(C.c_int32)), n_source))
        return H, b, cost.value, nc.value, vox[:n_source]

    def gicpPclCorrespondencesAt(self, guess, T_rel, n_source):
        """(pcl GICP, pclomp GICP) one correspondence pass at (guess, T_rel): (target index of every source point (n,) int32, -1 = none,
        Mahalanobis matrices (n, 3, 3), NaN where there is none, accepted count)"""
        g = _colmajor(guess, np.float32)
        t = _colmajor(T_rel, np.float32)
        corr = np.empty(max(n_source, 1), np.int32)
        M = np.empty((max(n_source, 1), 3, 3), np.float64)
        nc = C.c_uint64()
        fp = C.POINTER(C.c_float)
        check(self._lib.b2r_gicp_pcl_correspondences_at(self._h, g.ctypes.data_as(fp), t.ctypes.data_as(fp), corr.ctypes.data_as(C.POINTER(C.c_int32)),
                                                        M.ctypes.data_as(C.POINTER(C.c_double)), C.byref(nc)))
        return corr[:n_source], M[:n_source], nc.value

    def gicpPclCostAt(self, T):
        """(pcl GICP, pclomp GICP: T moves the raw source point) one cost pass at T over the last correspondences: (sum res^T M res, sum M res (3,), sum p (M res)^T (3, 3))"""
        t = _colmajor(T, np.float32)
        f = C.c_double()
        g = np.empty(3, np.float64)
        dR = np.empty((3, 3), np.float64)
        dp = C.POINTER(C.c_double)
        check(self._lib.b2r_gicp_pcl_cost_at(self._h, t.ctypes.data_as(C.POINTER(C.c_float)), C.byref(f), g.ctypes.data_as(dp), dR.ctypes.data_as(dp)))
        return f.value, g, dR

    def icpPclCorrespondencesAt(self, T, n_source):
        """(pcl ICP) one correspondence pass with the source transformed once by T, forward or reciprocal as configured: (target index of
        every source point (n,) int32, -1 = none, squared distance (n,) float32, NaN where there is none, accepted count)"""
        t = _colmajor(T, np.float32)
        corr = np.empty(max(n_source, 1), np.int32)
        d2 = np.empty(max(n_source, 1), np.float32)
        nc = C.c_uint64()
        check(self._lib.b2r_icp_pcl_correspondences_at(self._h, t.ctypes.data_as(C.POINTER(C.c_float)), corr.ctypes.data_as(C.POINTER(C.c_int32)),
                                                       d2.ctypes.data_as(C.POINTER(C.c_float)), C.byref(nc)))
        return corr[:n_source], d2[:n_source], nc.value

    def icpPclEstimateAt(self, T):
        """(pcl ICP) the same pass, then pcl::umeyama on it: (transformation_ (4, 4) float32, sums (17,): count, sum d2, sum src (3),
        sum tgt (3), demeaned cross products (9))"""
        t = _colmajor(T, np.float32)
        out = np.empty(16, np.float32)
        sums = np.empty(17, np.float64)
        check(self._lib.b2r_icp_pcl_estimate_at(self._h, t.ctypes.data_as(C.POINTER(C.c_float)), out.ctypes.data_as(C.POINTER(C.c_float)),
                                                sums.ctypes.data_as(C.POINTER(C.c_double))))
        return _from_colmajor(out), sums

    # --- companion / prefilter chain
    def _filter(self, fn, cloud, *args):
        a, n, s = _cloud(cloud)
        out = np.zeros_like(a)
        n_out = C.c_size_t()
        check(fn(self._h, a.ctypes.data_as(C.c_void_p), n, s, *args, out.ctypes.data_as(C.c_void_p), C.byref(n_out)))
        return out[: n_out.value]

    def distanceFilter(self, cloud, near, far):
        return self._filter(self._lib.b2r_distance_filter, cloud, float(near), float(far))

    def radiusOutlierRemoval(self, cloud, radius, min_neighbors):
        return self._filter(self._lib.b2r_radius_outlier_removal, cloud, float(radius), int(min_neighbors))

    def statisticalOutlierRemoval(self, cloud, mean_k, stddev_mul):
        return self._filter(self._lib.b2r_statistical_outlier_removal, cloud, int(mean_k), float(stddev_mul))

    def deskew(self, cloud, scan_period, angular_velocity):
        a, n, s = _cloud(cloud)
        out = np.zeros_like(a)
        w = np.ascontiguousarray(angular_velocity, np.float32)
        check(self._lib.b2r_deskew(self._h, a.ctypes.data_as(C.c_void_p), n, s, float(scan_period), w.ctypes.data_as(C.POINTER(C.c_float)),
                                   out.ctypes.data_as(C.c_void_p)))
        return out

    def prefilter(self, cloud, want_host=True, **params):
        """PrefilteringNodelet::cloud_callback in one call (b2r_prefilter): returns (host array or None, device pointer, count)"""
        a, n, s = _cloud(cloud)
        p = _capi.PrefilterParams()
        check(self._lib.b2r_prefilter_params_default(C.byref(p)))
        for k, v in params.items():
            if k in ("angular_velocity", "base_link_transform"):
                arr = getattr(p, k)
                vals = _colmajor(v) if k == "base_link_transform" else np.asarray(v, np.float32)
                for i, x in enumerate(vals):
                    arr[i] = float(x)
            else:
                setattr(p, k, v)
        out = np.zeros_like(a) if want_host else None
        dptr, m = C.c_void_p(), C.c_size_t()
        check(self._lib.b2r_prefilter(self._h, a.ctypes.data_as(C.c_void_p), n, s, 0, C.byref(p), out.ctypes.data_as(C.c_void_p) if want_host else None,
                                      C.byref(dptr), C.byref(m)))
        return (out[: m.value] if want_host else None), dptr.value, m.value

    def prefilter_raw(self, ptr, n, stride_bytes, device=False, **params):
        """b2r_prefilter on a raw (host or device) pointer; the result stays in HBM: returns (None, device pointer, count)"""
        p = _capi.PrefilterParams()
        check(self._lib.b2r_prefilter_params_default(C.byref(p)))
        for k, v in params.items():
            setattr(p, k, v)
        dptr, m = C.c_void_p(), C.c_size_t()
        check(self._lib.b2r_prefilter(self._h, C.c_void_p(ptr), n, stride_bytes, int(device), C.byref(p), None, C.byref(dptr), C.byref(m)))
        return None, dptr.value, m.value

    def floor_detect(self, cloud=None, ptr=None, n=0, stride_bytes=32, device=False, want_host=True, **params):
        """FloorDetectionNodelet::detect (b2r_floor_detect) on a host array `cloud`, or on `n` records at `ptr` (a device pointer when
        device=True).  Returns a dict: detected, reason (name), coeffs, n_filtered, n_inliers, ransac_iterations, model_indices,
        ransac_batches, ransac_hypotheses, readbacks, the filtered and inlier clouds as host arrays (when want_host) and their device pointers."""
        if cloud is not None:
            a, n, stride_bytes = _cloud(cloud)
            ptr, device = a.ctypes.data, False
        p = _capi.FloorParams()
        check(self._lib.b2r_floor_params_default(C.byref(p)))
        for k, v in params.items():
            if not hasattr(p, k):
                raise TypeError(f"unknown floor parameter {k}")
            setattr(p, k, v)
        r = _capi.FloorResult()
        sf = stride_bytes // 4
        filt = np.zeros((max(n, 1), sf), np.float32) if want_host else None
        inl = np.zeros((max(n, 1), sf), np.float32) if want_host else None
        df, di = C.c_void_p(), C.c_void_p()
        check(self._lib.b2r_floor_detect(self._h, C.c_void_p(ptr), n, stride_bytes, int(device), C.byref(p), C.byref(r),
                                         filt.ctypes.data_as(C.c_void_p) if want_host else None, inl.ctypes.data_as(C.c_void_p) if want_host else None,
                                         C.byref(df), C.byref(di)))
        return {"detected": bool(r.detected), "reason": _capi.FLOOR_REASONS[r.reason], "coeffs": np.array(r.coeffs[:], np.float32),
                "n_filtered": r.n_filtered, "n_inliers": r.n_inliers, "ransac_iterations": r.ransac_iterations,
                "model_indices": tuple(r.model_indices[:]), "ransac_batches": r.ransac_batches, "ransac_hypotheses": r.ransac_hypotheses,
                "readbacks": r.readbacks,
                "filtered": filt[: r.n_filtered] if want_host else None, "inliers": inl[: r.n_inliers] if want_host else None,
                "d_filtered": df.value, "d_inliers": di.value}

    def ingestPointCloud2(self, blob, n_points, point_step, off_x=0, off_y=4, off_z=8, off_intensity=0xffffffff, intensity_datatype=7, is_bigendian=False):
        """sensor_msgs/PointCloud2 data[] -> device PointXYZI records (b2r_ingest_pointcloud2); returns the device pointer"""
        buf = np.frombuffer(blob, np.uint8) if not isinstance(blob, np.ndarray) else blob.view(np.uint8).reshape(-1)
        self._keep["pc2"] = buf
        L = _capi.PointLayout(point_step, off_x, off_y, off_z, off_intensity, intensity_datatype, int(is_bigendian))
        out = C.c_void_p()
        check(self._lib.b2r_ingest_pointcloud2(self._h, buf.ctypes.data_as(C.c_void_p), n_points, C.byref(L), C.byref(out)))
        return out.value

    def ingestPointCloud2Rows(self, blob, width, height, row_step, point_step, off_x=0, off_y=4, off_z=8, off_intensity=0xffffffff,
                              intensity_datatype=7, is_bigendian=False):
        """organized sensor_msgs/PointCloud2 data[] with rows of row_step bytes (padding after width * point_step allowed) -> device
        PointXYZI records, width * height of them (b2r_ingest_pointcloud2_rows); returns the device pointer"""
        buf = np.frombuffer(blob, np.uint8) if not isinstance(blob, np.ndarray) else blob.view(np.uint8).reshape(-1)
        if width * height and buf.size < height * row_step:
            raise ValueError("blob is shorter than height * row_step")
        self._keep["pc2"] = buf
        L = _capi.PointLayout(point_step, off_x, off_y, off_z, off_intensity, intensity_datatype, int(is_bigendian))
        out = C.c_void_p()
        check(self._lib.b2r_ingest_pointcloud2_rows(self._h, buf.ctypes.data_as(C.c_void_p), width, height, row_step, C.byref(L), C.byref(out)))
        return out.value

    def ingestPcd(self, path):
        """binary PCD file -> (device pointer to PointXYZI records, point count) (b2r_ingest_pcd)"""
        out, n = C.c_void_p(), C.c_size_t()
        check(self._lib.b2r_ingest_pcd(self._h, str(path).encode(), C.byref(out), C.byref(n)))
        return out.value, n.value

    def mapCloudGenerate(self, keyframes, resolution):
        """MapCloudGenerator::generate: keyframes = list of (cloud, 4x4 pose) -> map cloud (b2r_map_cloud_generate); None if empty"""
        arrs = [_cloud(c)[0] for c, _ in keyframes]
        kf = (_capi.KeyframeSnapshot * max(len(arrs), 1))()
        for i, (a, (_, pose)) in enumerate(zip(arrs, keyframes)):
            kf[i].points, kf[i].n = a.ctypes.data, a.shape[0]
            pc = _colmajor(pose)
            for k in range(16):
                kf[i].pose[k] = pc[k]
        total = sum(a.shape[0] for a in arrs)
        stride_f = arrs[0].shape[1] if arrs else 8
        out = np.zeros((max(total, 1), stride_f), np.float32)
        m = C.c_size_t()
        rc = check(self._lib.b2r_map_cloud_generate(self._h, kf, len(arrs), stride_f * 4, float(resolution), out.ctypes.data_as(C.c_void_p), total, C.byref(m)))
        return None if rc == 1 else out[: m.value]

    def voxelGridFilterDevice(self, d_ptr, n, stride_bytes, leaf):
        """device pointer in -> (device pointer out, voxel count, rc): the result stays in HBM (b2r_voxelgrid_device)"""
        out, m = C.c_void_p(), C.c_size_t()
        rc = check(self._lib.b2r_voxelgrid_device(self._h, C.c_void_p(d_ptr), n, stride_bytes, leaf, C.byref(out), C.byref(m)))
        return out.value, m.value, rc

    def voxelGridFilter(self, cloud, leaf, with_keys=False):
        a, n, s = _cloud(cloud)
        out = np.zeros_like(a)
        n_out = C.c_size_t()
        keys = np.empty(max(n, 1), np.int32)
        counts = np.empty(max(n, 1), np.int32)
        ip = C.POINTER(C.c_int32)
        rc = check(self._lib.b2r_voxelgrid(self._h, a.ctypes.data_as(C.c_void_p), n, s, leaf, out.ctypes.data_as(C.c_void_p), C.byref(n_out),
                                           keys.ctypes.data_as(ip), counts.ctypes.data_as(ip)))
        m = n_out.value
        if with_keys:
            return out[:m], keys[:m], counts[:m], rc
        return out[:m]

    def approximateVoxelGridFilter(self, cloud, leaf, with_counts=False):
        """pcl::ApproximateVoxelGrid::filter (b2r_approximate_voxelgrid): the outputs in PCL's order; with_counts also returns the
        number of points behind each output"""
        a, n, s = _cloud(cloud)
        out = np.zeros_like(a)
        n_out = C.c_size_t()
        counts = np.empty(max(n, 1), np.int32)
        check(self._lib.b2r_approximate_voxelgrid(self._h, a.ctypes.data_as(C.c_void_p), n, s, leaf, out.ctypes.data_as(C.c_void_p), C.byref(n_out),
                                                  counts.ctypes.data_as(C.POINTER(C.c_int32))))
        m = n_out.value
        if with_counts:
            return out[:m], counts[:m]
        return out[:m]

    def approximateVoxelGridFilterDevice(self, d_ptr, n, stride_bytes, leaf):
        """device pointer in -> (device pointer out, output count): the result stays in HBM (b2r_approximate_voxelgrid_device)"""
        out, m = C.c_void_p(), C.c_size_t()
        check(self._lib.b2r_approximate_voxelgrid_device(self._h, C.c_void_p(d_ptr), n, stride_bytes, leaf, C.byref(out), C.byref(m)))
        return out.value, m.value


def select_registration_method(params=None, device_id=0):
    """Mirror of hdl_graph_slam::select_registration_method(ros::NodeHandle&): `params` plays the private rosparam
    namespace (same keys, same defaults).  Raises B2RError(B2R_EUNSUPPORTED) for methods this engine does not re-create."""
    lib = _capi.load()
    params = params or {}
    keys = [str(k).encode() for k in params.keys()]
    vals = [(("true" if v else "false") if isinstance(v, bool) else str(v)).encode() for v in params.values()]
    n = len(keys)
    ka = (C.c_char_p * max(n, 1))(*keys)
    va = (C.c_char_p * max(n, 1))(*vals)
    h = C.c_void_p()
    check(lib.b2r_select_registration_method(ka, va, n, device_id, C.byref(h)))
    return Registration(_handle=h)


class ScanMatchingOdometry:
    """Mirror of ScanMatchingOdometryNodelet's matching() state machine (keyframe, prev_trans, thresholds).

    downsample_method / downsample_resolution are the odometry nodelet's own downsample (:83-103): B2R_DOWNSAMPLE_VOXELGRID or
    B2R_DOWNSAMPLE_APPROX_VOXELGRID filter every cloud on the device before it is registered; B2R_DOWNSAMPLE_NONE (the default here,
    and what every shipped launch file sets) and unknown values register the cloud as given."""

    def __init__(self, registration, keyframe_delta_trans=0.25, keyframe_delta_angle=0.15, keyframe_delta_time=1.0,
                 transform_thresholding=False, max_acceptable_trans=1.0, max_acceptable_angle=1.0, publish_status=False,
                 downsample_method=_capi.B2R_DOWNSAMPLE_NONE, downsample_resolution=0.1):
        self._lib = _capi.load()
        self.registration = registration
        p = OdometryParams(keyframe_delta_trans, keyframe_delta_angle, keyframe_delta_time, int(transform_thresholding),
                           max_acceptable_trans, max_acceptable_angle, int(publish_status), int(downsample_method), float(downsample_resolution))
        self._o = C.c_void_p()
        check(self._lib.b2r_odometry_create(registration._h, C.byref(p), C.byref(self._o)))
        self._keep = []

    def close(self):
        if self._o:
            self._lib.b2r_odometry_destroy(self._o)
            self._o = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def matching(self, stamp, cloud, msf_delta=None):
        a, n, s = _cloud(cloud)
        return self.matching_raw(stamp, a.ctypes.data, n, s, msf_delta)

    def prefetch_raw(self, ptr, n, stride_bytes, device=False):
        check(self._lib.b2r_odometry_prefetch(self._o, C.c_void_p(ptr), n, stride_bytes, int(device)))

    def matching_raw(self, stamp, ptr, n, stride_bytes, msf_delta=None, device=False):
        st = OdometryStatus()
        dp = None
        if msf_delta is not None:
            d = _colmajor(msf_delta)
            dp = d.ctypes.data_as(C.POINTER(C.c_float))
        fn = self._lib.b2r_odometry_matching_device if device else self._lib.b2r_odometry_matching
        check(fn(self._o, float(stamp), C.c_void_p(ptr), n, stride_bytes, dp, C.byref(st)))
        return _odometry_status(st)

    def matching_ros(self, sec, nsec, cloud, msf_delta=None, want_status=False):
        """matching() with a ros::Time stamp (sec, nsec): the keyframe test takes roscpp's exact (stamp - keyframe_stamp).toSec(), and
        the status (matching_error, inlier_fraction) is computed only when want_status is set"""
        a, n, s = _cloud(cloud)
        return self.matching_ros_raw(sec, nsec, a.ctypes.data, n, s, msf_delta, want_status)

    def matching_ros_raw(self, sec, nsec, ptr, n, stride_bytes, msf_delta=None, want_status=False, device=False):
        st = OdometryStatus()
        dp = None
        if msf_delta is not None:
            d = _colmajor(msf_delta)
            dp = d.ctypes.data_as(C.POINTER(C.c_float))
        check(self._lib.b2r_odometry_matching_ros(self._o, int(sec), int(nsec), C.c_void_p(ptr), n, stride_bytes, int(device), dp,
                                                  int(bool(want_status)), C.byref(st)))
        return _odometry_status(st)

    def aligned(self, n, stride_bytes=32, is_dense=True):
        """aligned_points of the last matching call: its raw cloud (n records of stride_bytes) under odom, as (n, stride_bytes / 4)
        float32; raises after a first or rejected frame"""
        out = np.zeros((n, stride_bytes // 4), np.float32)
        check(self._lib.b2r_odometry_aligned(self._o, int(bool(is_dense)), out.ctypes.data, n, stride_bytes))
        return out


def _odometry_status(st):
    return dict(odom=_from_colmajor(st.odom), trans=_from_colmajor(st.trans), converged=bool(st.converged), iterations=st.iterations,
                keyframe_updated=bool(st.keyframe_updated), frame_rejected=bool(st.frame_rejected), matching_error=st.matching_error,
                inlier_fraction=st.inlier_fraction)


class LoopDetector:
    """Mirror of LoopDetector::matching: align each candidate to the new keyframe, keep the best converged fitness."""

    def __init__(self, registration, fitness_score_max_range=np.finfo(np.float64).max, fitness_score_thresh=0.5):
        self._lib = _capi.load()
        self.registration = registration
        self.fitness_score_max_range = fitness_score_max_range
        self.fitness_score_thresh = fitness_score_thresh

    def matching(self, candidate_clouds, new_keyframe_cloud, guesses):
        nk, n_new, s = _cloud(new_keyframe_cloud)
        cands = [_cloud(c)[0] for c in candidate_clouds]
        m = len(cands)
        ptrs = (C.c_void_p * max(m, 1))(*[c.ctypes.data for c in cands])
        ns = (C.c_size_t * max(m, 1))(*[c.shape[0] for c in cands])
        g = np.ascontiguousarray(np.stack([_colmajor(x) for x in guesses]) if m else np.zeros((1, 16), np.float32), np.float32)
        res = (Result * max(m, 1))()
        best = C.c_int32(-1)
        check(self._lib.b2r_loop_matching(self.registration._h, nk.ctypes.data_as(C.c_void_p), n_new, s, ptrs, ns, m,
                                          g.ctypes.data_as(C.POINTER(C.c_float)), self.fitness_score_max_range, self.fitness_score_thresh,
                                          res, C.byref(best)))
        results = [dict(T=_from_colmajor(r.T), fitness=r.fitness, converged=bool(r.converged), iterations=r.iterations) for r in res[:m]]
        return best.value, results


def _result_dict(r):
    return dict(T=_from_colmajor(r.T), fitness=r.fitness, converged=bool(r.converged), iterations=r.iterations)


def _keyframe_states(keyframes):
    """keyframes: sequence of (accum_distance, 4x4 estimate) -> ctypes array of b2r_keyframe_state"""
    arr = (_capi.KeyframeState * max(len(keyframes), 1))()
    for i, (acc, est) in enumerate(keyframes):
        arr[i].accum_distance = float(acc)
        e = np.asarray(est, np.float64).T.reshape(-1)  # column-major
        for k in range(16):
            arr[i].estimate[k] = e[k]
    return arr


class LoopClosureGate:
    """Host mirror of the gating half of hdl_graph_slam's LoopDetector (loop_detector.hpp:39-46,57-68,81-109,137-142): rosparams,
    find_candidates, the initial guess, and detect() as plan -> batched matching -> sequential replay.  Nothing here computes on the
    device; `detect` drives a RegistrationBatch for the matching."""

    def __init__(self, **params):
        self._lib = _capi.load()
        self.params = _capi.LoopParams()
        check(self._lib.b2r_loop_params_default(C.byref(self.params)))
        for k, v in params.items():
            setattr(self.params, k, v)
        self.last_edge_accum_distance = 0.0  # loop_detector.hpp:48

    def find_candidates(self, keyframes, new_keyframe):
        ks, nk = _keyframe_states(keyframes), _keyframe_states([new_keyframe])
        out = (C.c_int32 * max(len(keyframes), 1))()
        n = C.c_size_t()
        check(self._lib.b2r_loop_find_candidates(C.byref(self.params), ks, len(keyframes), nk, self.last_edge_accum_distance, out, len(keyframes), C.byref(n)))
        return list(out[: n.value])

    def guess(self, new_keyframe_estimate, candidate_estimate):
        a = np.ascontiguousarray(np.asarray(new_keyframe_estimate, np.float64).T).reshape(-1)
        b = np.ascontiguousarray(np.asarray(candidate_estimate, np.float64).T).reshape(-1)
        g = np.empty(16, np.float32)
        check(self._lib.b2r_loop_guess(a.ctypes.data_as(C.POINTER(C.c_double)), b.ctypes.data_as(C.POINTER(C.c_double)), g.ctypes.data_as(C.POINTER(C.c_float))))
        return g.reshape(4, 4).T.copy()

    def plan(self, keyframes, new_keyframes):
        """-> (candidate_index[n_pairs], guesses[n_pairs, 4, 4], group_first[n_new + 1]) under the gate as it stands now"""
        ks, nks = _keyframe_states(keyframes), _keyframe_states(new_keyframes)
        cap = max(len(keyframes) * len(new_keyframes), 1)
        idx = (C.c_int32 * cap)()
        g = np.empty((cap, 16), np.float32)
        gf = (C.c_int64 * (len(new_keyframes) + 1))()
        n = C.c_size_t()
        check(self._lib.b2r_loop_detect_plan(C.byref(self.params), ks, len(keyframes), nks, len(new_keyframes), self.last_edge_accum_distance, idx,
                                             g.ctypes.data_as(C.POINTER(C.c_float)), cap, gf, C.byref(n)))
        guesses = g[: n.value].reshape(-1, 4, 4).transpose(0, 2, 1).copy()
        return list(idx[: n.value]), guesses, list(gf)

    def replay(self, new_keyframes, group_first, best, planned_last_edge):
        """the sequential walk of detect() over the batch's per-group answers -> accepted[g] (index inside the group or -1); updates
        last_edge_accum_distance like loop_detector.hpp:166"""
        nks = _keyframe_states(new_keyframes)
        gf = (C.c_int64 * len(group_first))(*[int(x) for x in group_first])
        b = (C.c_int32 * max(len(best), 1))(*[int(x) for x in best])
        acc = (C.c_int32 * max(len(best), 1))()
        last = C.c_double(self.last_edge_accum_distance)
        check(self._lib.b2r_loop_detect_replay(C.byref(self.params), nks, len(new_keyframes), gf, b, float(planned_last_edge), C.byref(last), acc))
        self.last_edge_accum_distance = last.value
        return list(acc[: len(new_keyframes)])

    def detect(self, batch, keyframes, keyframe_cloud_ids, new_keyframes, new_keyframe_cloud_ids):
        """LoopDetector::detect for all new keyframes at once on a RegistrationBatch (its communicator shards the groups over the GPUs).
        Returns [(new keyframe index, candidate keyframe index, relative pose 4x4)] of the registered loops, in the reference's order."""
        planned_last = self.last_edge_accum_distance
        cand, guesses, gf = self.plan(keyframes, new_keyframes)
        pairs = []
        for g in range(len(new_keyframes)):
            for j in range(gf[g], gf[g + 1]):
                pairs.append((keyframe_cloud_ids[cand[j]], new_keyframe_cloud_ids[g], guesses[j]))
        best, results = batch.loopDetect(pairs, gf, self.params.fitness_score_max_range, self.params.fitness_score_thresh)
        accepted = self.replay(new_keyframes, gf, best, planned_last)
        loops = []
        for g, a in enumerate(accepted):
            if a >= 0:
                loops.append((g, cand[gf[g] + a], results[gf[g] + a]["T"]))
        return loops


def shard_range(n_groups, world, rank):
    """contiguous block of groups owned by `rank` (b2r_shard_range)"""
    g0, g1 = C.c_size_t(), C.c_size_t()
    check(_capi.load().b2r_shard_range(n_groups, world, rank, C.byref(g0), C.byref(g1)))
    return g0.value, g1.value


def loop_argmin(results, fitness_score_thresh):
    """LoopDetector::matching's selection over one group's Result records (b2r_loop_argmin)"""
    arr = (Result * max(len(results), 1))(*results)
    best = C.c_int32(-1)
    check(_capi.load().b2r_loop_argmin(arr, len(results), fitness_score_thresh, C.byref(best)))
    return best.value


class RegistrationBatch:
    """Batched, device-resident GICP or NDT registration (include/b200reg.h: b2r_batch_*): keyframe clouds are registered once and many
    (source, target, guess) pairs are aligned per launch — the candidate loop of LoopDetector::matching
    (include/hdl_graph_slam/loop_detector.hpp:135-154) for one or many new keyframes."""

    def __init__(self, cfg=None, params=None, device_id=0):
        self._lib = _capi.load()
        if cfg is None:
            reg = select_registration_method(params or {"registration_method": "FAST_GICP"}, device_id=device_id)
            cfg = reg.config
            reg.close()
        self._b = C.c_void_p()
        check(self._lib.b2r_batch_create(C.byref(cfg), C.byref(self._b)))
        eng = C.c_void_p()
        check(self._lib.b2r_batch_get_engine(self._b, C.byref(eng)))
        self.engine = Registration(_handle=eng)
        self.engine.close = lambda: None  # owned by the batch
        self._keep = {}
        self._sizes = {}  # cloud id -> point count: the capacity of a host map cloud

    def close(self):
        if self._b:
            self.engine._h = C.c_void_p()
            self._lib.b2r_batch_destroy(self._b)
            self._b = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def addCloud(self, cloud):
        a, n, s = _cloud(cloud)
        cid = C.c_int32(-1)
        check(self._lib.b2r_batch_add_cloud(self._b, a.ctypes.data_as(C.c_void_p), n, s, C.byref(cid)))
        self._keep[cid.value] = a
        self._sizes[cid.value] = n
        return cid.value

    def addCloudRaw(self, ptr, n, stride_bytes, device=False):
        cid = C.c_int32(-1)
        fn = self._lib.b2r_batch_add_cloud_device if device else self._lib.b2r_batch_add_cloud
        check(fn(self._b, C.c_void_p(ptr), n, stride_bytes, C.byref(cid)))
        self._sizes[cid.value] = n
        return cid.value

    def removeCloud(self, cid):
        check(self._lib.b2r_batch_remove_cloud(self._b, cid))
        self._keep.pop(cid, None)
        self._sizes.pop(cid, None)

    def cloudCount(self):
        return self._lib.b2r_batch_cloud_count(self._b)

    def synchronize(self):
        check(self._lib.b2r_batch_synchronize(self._b))

    @staticmethod
    def _pairs(pairs):
        arr = (Pair * max(len(pairs), 1))()
        for i, (s, t, g) in enumerate(pairs):
            arr[i].source, arr[i].target = int(s), int(t)
            gc = _colmajor(np.eye(4) if g is None else g)
            for k in range(16):
                arr[i].guess[k] = gc[k]
        return arr

    def align(self, pairs, want_fitness=True, fitness_max_range=np.finfo(np.float64).max, raw=False):
        """pairs: list of (source id, target id, 4x4 guess) -> list of result dicts (or the ctypes Result array when raw)"""
        arr = pairs if isinstance(pairs, C.Array) else self._pairs(pairs)
        n = len(arr) if isinstance(pairs, C.Array) else len(pairs)
        res = (Result * max(n, 1))()
        check(self._lib.b2r_batch_align(self._b, arr, n, int(bool(want_fitness)), fitness_max_range, res))
        if raw:
            return res
        return [_result_dict(r) for r in res[:n]]

    def calcFitnessScore(self, edges, max_range=np.finfo(np.float64).max):
        """InformationMatrixCalculator::calc_fitness_score for many edges: edges = list of (cloud1 id, cloud2 id, relpose 4x4) -> scores"""
        arr = self._pairs([(c2, c1, rel) for c1, c2, rel in edges])
        out = np.empty(max(len(edges), 1), np.float64)
        check(self._lib.b2r_batch_calc_fitness_score(self._b, arr, len(edges), max_range, out.ctypes.data_as(C.POINTER(C.c_double))))
        return out[: len(edges)]

    def mapCloudGenerate(self, ids, poses, resolution, stride_bytes=32, device=False):
        """MapCloudGenerator::generate over cached clouds: keyframe k = cloud ids[k] at the 4x4 pose poses[k] -> map cloud of
        stride_bytes records (b2r_batch_map_cloud_generate); device=True returns (engine-owned device pointer, record count)
        instead.  None if ids is empty."""
        ids = [int(i) for i in ids]
        if len(poses) != len(ids):
            raise ValueError("one pose per id")
        idarr = (C.c_int32 * max(len(ids), 1))(*ids)
        P = np.ascontiguousarray(np.concatenate([_colmajor(p) for p in poses]) if ids else np.zeros(16, np.float32))
        Pp = P.ctypes.data_as(C.POINTER(C.c_float))
        m = C.c_size_t()
        if device:
            dptr = C.c_void_p()
            rc = check(self._lib.b2r_batch_map_cloud_generate(self._b, idarr, Pp, len(ids), float(resolution), stride_bytes, None, 0, C.byref(dptr), C.byref(m)))
            return None if rc == 1 else (dptr.value, m.value)
        cap = sum(self._sizes.get(i, 0) for i in ids)
        out = np.zeros((max(cap, 1), stride_bytes // 4), np.float32)
        rc = check(self._lib.b2r_batch_map_cloud_generate(self._b, idarr, Pp, len(ids), float(resolution), stride_bytes, out.ctypes.data_as(C.c_void_p),
                                                          cap, None, C.byref(m)))
        return None if rc == 1 else out[: m.value]

    def lastRounds(self):
        a, b = C.c_uint64(), C.c_uint64()
        check(self._lib.b2r_batch_last_rounds(self._b, C.byref(a), C.byref(b)))
        return a.value, b.value

    # --- multi-GPU
    @staticmethod
    def ncclUniqueId():
        buf = (C.c_char * 128)()
        check(_capi.load().b2r_nccl_unique_id(buf, 128))
        return bytes(buf)

    def commInit(self, unique_id, rank, world):
        buf = (C.c_char * 128).from_buffer_copy(unique_id)
        check(self._lib.b2r_batch_comm_init(self._b, buf, rank, world))

    def loopDetect(self, pairs, group_first, fitness_score_max_range=np.finfo(np.float64).max, fitness_score_thresh=0.5, raw=False):
        """LoopDetector::matching for many new keyframes, sharded over the communicator's ranks (b2r_batch_loop_detect)"""
        arr = pairs if isinstance(pairs, C.Array) else self._pairs(pairs)
        n = int(group_first[-1])
        gf = (C.c_int64 * len(group_first))(*[int(x) for x in group_first])
        ng = len(group_first) - 1
        res = (Result * max(n, 1))()
        best = (C.c_int32 * max(ng, 1))()
        check(self._lib.b2r_batch_loop_detect(self._b, arr, n, gf, ng, fitness_score_max_range, fitness_score_thresh, res, best))
        if raw:
            return list(best[:ng]), res
        return list(best[:ng]), [_result_dict(r) for r in res[:n]]


def information_from_fitness(fitness_score, **params):
    """InformationMatrixCalculator::calc_information_matrix after the fitness score: diagonal of the 6x6 information matrix"""
    lib = _capi.load()
    p = _capi.InformationParams()
    check(lib.b2r_information_params_default(C.byref(p)))
    for k, v in params.items():
        setattr(p, k, v)
    out = np.empty(6, np.float64)
    check(lib.b2r_information_from_fitness(C.byref(p), float(fitness_score), out.ctypes.data_as(C.POINTER(C.c_double))))
    return out
