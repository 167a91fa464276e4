"""The registration branches the factory serves, as the rosparams that select them, each with its own sequential reference align and
that method's pose tolerance.  Shared by tests/test_backend_methods_gpu.py and tests/test_odometry_methods_gpu.py.

Every reference is built once per test module (References) and takes the engine handle's own configuration (b2r_get_config), so the
reference runs with exactly the parameters the factory gave the handle."""
import numpy as np

import hdl_graph_slam_b200 as pkg
import gicp_omp_ref
import gicp_pcl_ref
import icp_pcl_ref
import ndt_kdtree_ref
import ndt_pcl_ref
import vgicp_cuda_ref
import vgicp_ref
from common import rot_err, trans_err

# case id -> rosparams.  The VGICP branches default reg_resolution to 1.0 and the NDT branches to 0.5; the launch files set 1.0
METHODS = {
    "FAST_GICP": {"registration_method": "FAST_GICP"},
    "GICP": {"registration_method": "GICP"},
    "B200_GICP_OMP": {"registration_method": "B200_GICP_OMP"},
    "B200_ICP": {"registration_method": "B200_ICP", "reg_use_reciprocal_correspondences": "false"},
    "B200_ICP_reciprocal": {"registration_method": "B200_ICP", "reg_use_reciprocal_correspondences": "true"},
    "FAST_VGICP": {"registration_method": "FAST_VGICP"},
    "B200_VGICP_CUDA": {"registration_method": "B200_VGICP_CUDA", "reg_resolution": "1.0"},
    "NDT": {"registration_method": "NDT", "reg_resolution": "1.0"},
    "B200_NDT_KDTREE": {"registration_method": "B200_NDT_KDTREE", "reg_resolution": "1.0"},
    "NDT_OMP": {"registration_method": "NDT_OMP", "reg_resolution": "1.0"},
    "NDT_OMP_DIRECT1": {"registration_method": "NDT_OMP", "reg_resolution": "1.0", "reg_nn_search_method": "DIRECT1"},
}
NDT_FAMILY = {"NDT", "B200_NDT_KDTREE", "NDT_OMP", "NDT_OMP_DIRECT1"}

COMMON = dict(reg_maximum_iterations="5", reg_transformation_epsilon="0.005")
NON_DEFAULT = {  # every reg_* key each branch reads (registrations.cpp:22-124), each away from its default
    "FAST_GICP": dict(COMMON, registration_method="FAST_GICP", reg_max_correspondence_distance="1.75", reg_correspondence_randomness="10"),
    "GICP": dict(COMMON, registration_method="GICP", reg_max_correspondence_distance="1.75", reg_correspondence_randomness="10",
                 reg_max_optimizer_iterations="3"),
    "B200_GICP_OMP": dict(COMMON, registration_method="B200_GICP_OMP", reg_max_correspondence_distance="1.75",
                          reg_correspondence_randomness="10", reg_max_optimizer_iterations="3"),
    "B200_ICP": dict(COMMON, registration_method="B200_ICP", reg_max_correspondence_distance="1.75", reg_use_reciprocal_correspondences="true"),
    "FAST_VGICP": dict(COMMON, registration_method="FAST_VGICP", reg_resolution="2.0", reg_correspondence_randomness="10"),
    "B200_VGICP_CUDA": dict(COMMON, registration_method="B200_VGICP_CUDA", reg_resolution="2.0", reg_correspondence_randomness="10"),
    "NDT": dict(COMMON, registration_method="NDT", reg_resolution="2.0"),
    "NDT_OMP": dict(COMMON, registration_method="NDT_OMP", reg_resolution="2.0", reg_nn_search_method="DIRECT1"),
    "B200_NDT_KDTREE": dict(COMMON, registration_method="B200_NDT_KDTREE", reg_resolution="2.0"),
}


def pose_tolerance(case):
    """the per-entry pose tolerance of pose_close, as one number"""
    if case == "B200_GICP_OMP":
        return 2e-3
    if case in ("GICP", "B200_ICP", "B200_ICP_reciprocal"):
        return 1e-5
    return 1e-4 if case in NDT_FAMILY else 1e-6


def pose_close(case, T, T_ref):
    """the end pose of an engine align against its reference's, at the tolerance that method's own tests hold it to: FastGICP and both
    VGICP methods 1e-6 (DESIGN §2), pcl GICP and pcl ICP 1e-5 per entry (test_gicp_pcl_gpu, test_icp_pcl_gpu: fixed-tree against
    index-order sums), pclomp GICP gicp_pcl_ref.end_point_is_as_good, the NDT family 1e-4 m / rad"""
    T, T_ref = np.asarray(T, np.float64), np.asarray(T_ref, np.float64)
    if case == "B200_GICP_OMP":
        gicp_pcl_ref.end_point_is_as_good(T, T_ref)
        return True
    if case in ("GICP", "B200_ICP", "B200_ICP_reciprocal"):
        return float(np.max(np.abs(T - T_ref))) <= 1e-5
    tol = 1e-4 if case in NDT_FAMILY else 1e-6
    return trans_err(T, T_ref) < tol and rot_err(T, T_ref) < tol


class References:
    """the sequential reference of every method, each library compiled on first use into its own directory"""

    def __init__(self, tmp_path_factory, oracle):
        self.tmp, self.oracle, self._libs, self._cov = tmp_path_factory, oracle, {}, {}

    def close(self):
        for h in self._cov.values():
            h.close()
        self._cov = {}

    def _lib(self, name, cls):
        if name not in self._libs:
            self._libs[name] = cls(self.tmp.mktemp(name))
        return self._libs[name]

    def align(self, case, cfg, src, tgt, guess):
        """align(src -> tgt from guess) with `case`'s reference under the handle configuration cfg -> dict(T, converged, iterations)"""
        g = np.asarray(guess, np.float32)
        if case == "FAST_GICP":
            o = self.oracle.gicp_align(src, tgt, g, max_iterations=cfg.max_iterations, transformation_epsilon=cfg.transformation_epsilon,
                                       rotation_epsilon=cfg.rotation_epsilon, max_corr_dist=cfg.max_correspondence_distance,
                                       k=cfg.k_correspondences)
        elif case in ("GICP", "B200_GICP_OMP"):
            # fed the engine's covariances, as test_gicp_pcl_gpu does: the BFGS line search compares f values that agree to the last
            # bits, so covariances one ulp apart may change the iteration count (the covariances are pinned apart, bit for bit)
            if cfg.k_correspondences not in self._cov:
                self._cov[cfg.k_correspondences] = pkg.select_registration_method(
                    {"registration_method": "GICP", "reg_correspondence_randomness": cfg.k_correspondences})
            h = self._cov[cfg.k_correspondences]
            h.setInputTarget(tgt)
            h.setInputSource(src)
            ref = self._lib(case, gicp_pcl_ref.Reference if case == "GICP" else gicp_omp_ref.Reference)
            o = ref.align(src, tgt, g, scov=h.getCovariances(0, src.shape[0]), tcov=h.getCovariances(1, tgt.shape[0]), max_iterations=cfg.max_iterations, max_optimizer_iterations=cfg.max_optimizer_iterations,
                          transformation_epsilon=cfg.transformation_epsilon, rotation_epsilon=cfg.rotation_epsilon,
                          corr_dist=cfg.max_correspondence_distance, k=cfg.k_correspondences)
        elif case in ("B200_ICP", "B200_ICP_reciprocal"):
            o = self._lib("icp", icp_pcl_ref.Reference).align(src, tgt, g, max_iterations=cfg.max_iterations,
                                                                transformation_epsilon=cfg.transformation_epsilon,
                                                                max_dist=cfg.max_correspondence_distance,
                                                                reciprocal=bool(cfg.use_reciprocal_correspondences))
        elif case in ("FAST_VGICP", "B200_VGICP_CUDA"):
            if case == "FAST_VGICP":
                m = self._lib(case, vgicp_ref.Reference).map(tgt, cfg.ndt_resolution)
            else:
                m = self._lib(case, vgicp_cuda_ref.Reference).map(tgt, cfg.ndt_resolution, k=cfg.k_correspondences)
            o = m.align(src, g, max_iterations=cfg.max_iterations, transformation_epsilon=cfg.transformation_epsilon,
                        rotation_epsilon=cfg.rotation_epsilon)
        else:
            kw = dict(max_iterations=cfg.max_iterations, transformation_epsilon=cfg.transformation_epsilon, step_size=cfg.ndt_step_size,
                      outlier_ratio=cfg.ndt_outlier_ratio, mt_interval_flag=cfg.ndt_mt_interval_flag, fixed_iterations=cfg.ndt_fixed_iterations)
            if case == "NDT":
                m = self._lib(case, ndt_pcl_ref.Reference).map(tgt, cfg.ndt_resolution)
            elif case == "B200_NDT_KDTREE":
                m = self._lib(case, ndt_kdtree_ref.Reference).map(tgt, cfg.ndt_resolution)
            else:
                m = self.oracle.NdtMap(tgt, cfg.ndt_resolution)
                kw["search_method"] = cfg.ndt_search_method
            o = m.align(src, g, **kw)
        return dict(T=np.asarray(o["T"], np.float32), converged=bool(o["converged"]), iterations=int(o["iterations"]))
