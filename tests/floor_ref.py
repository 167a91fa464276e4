"""Shared by the floor-detection tests: the sequential reference of FloorDetectionNodelet::detect (tests/floor_ref.cpp, compiled into a
temporary directory), the launch files' parameter sets and the scans they run on."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from hdl_graph_slam_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "floor_ref.cpp")

# launch/hdl_graph_slam_{400,501,kitti}.launch; floor_normal_thresh is never set there (default 10)
LAUNCH = {
    "hdl": dict(tilt_deg=0.0, sensor_height=2.0, height_clip_range=1.0, floor_pts_thresh=512, use_normal_filtering=1, normal_filter_thresh=20.0),
    "501": dict(tilt_deg=0.0, sensor_height=1.5, height_clip_range=0.5, floor_pts_thresh=256, use_normal_filtering=1, normal_filter_thresh=20.0),
    "kitti": dict(tilt_deg=0.0, sensor_height=3.0, height_clip_range=1.0, floor_pts_thresh=512, use_normal_filtering=0, normal_filter_thresh=20.0),
}

HYP = np.dtype([("idx", np.int32, 3), ("c", np.float32, 4), ("ok", np.int32)])


def params(**kw):
    p = _capi.FloorParams(tilt_deg=0.0, sensor_height=2.0, height_clip_range=1.0, floor_pts_thresh=512, use_normal_filtering=1,
                          floor_normal_thresh=10.0, normal_filter_thresh=20.0)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


class Reference:
    def __init__(self, tmpdir):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
        so = os.path.join(str(tmpdir), "libfloor_ref.so")
        subprocess.check_call([cxx, "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-Wall", "-o", so, SRC])
        self.lib = C.CDLL(so)
        self.lib.ref_mt19937.argtypes = [C.c_uint32, C.c_size_t, C.c_void_p]
        self.lib.ref_eigen33.argtypes = [C.c_void_p, C.c_void_p]
        self.lib.ref_ransac_hypotheses.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p]
        self.lib.ref_floor_detect.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.POINTER(_capi.FloorParams), C.POINTER(_capi.FloorResult),
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]

    def mt19937(self, seed, n):
        out = np.zeros(n, np.uint32)
        self.lib.ref_mt19937(seed, n, out.ctypes.data)
        return out

    def eigen33(self, A):
        A = np.ascontiguousarray(A, np.float32).reshape(9)
        v = np.zeros(3, np.float32)
        self.lib.ref_eigen33(A.ctypes.data, v.ctypes.data)
        return v

    def hypotheses(self, cloud, count):
        a = np.ascontiguousarray(cloud, np.float32)
        out = np.zeros(count, HYP)
        self.lib.ref_ransac_hypotheses(a.ctypes.data, a.shape[0], a.shape[1], count, out.ctypes.data)
        return out

    def detect(self, cloud, **kw):
        """the same dict as Registration.floor_detect, plus band_mask (per input point) and normal_keep (per band point)"""
        a = np.ascontiguousarray(cloud, np.float32)
        n, sf = a.shape
        p = params(**kw)
        r = _capi.FloorResult()
        filt = np.zeros((max(n, 1), sf), np.float32)
        inl = np.zeros((max(n, 1), sf), np.float32)
        band = np.zeros(max(n, 1), np.uint8)
        keep = np.zeros(max(n, 1), np.uint8)
        self.lib.ref_floor_detect(a.ctypes.data, n, sf, C.byref(p), C.byref(r), filt.ctypes.data, inl.ctypes.data, band.ctypes.data, keep.ctypes.data)
        nb = int(band[:n].sum())
        return {"detected": bool(r.detected), "reason": _capi.FLOOR_REASONS[r.reason], "coeffs": np.array(r.coeffs[:], np.float32),
                "n_filtered": r.n_filtered, "n_inliers": r.n_inliers, "ransac_iterations": r.ransac_iterations,
                "model_indices": tuple(r.model_indices[:]), "filtered": filt[: r.n_filtered], "inliers": inl[: r.n_inliers],
                "band_mask": band[:n].astype(bool), "normal_keep": keep[:nb].astype(bool)}


def bits(a):
    """float32 array -> uint32 bit patterns with every NaN folded into one pattern (payloads differ between x86 and the GPU)"""
    a = np.ascontiguousarray(a, np.float32)
    u = a.view(np.uint32).copy()
    u[np.isnan(a)] = 0x7FC00000
    return u


def same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


FIELDS = ("detected", "reason", "n_filtered", "n_inliers", "ransac_iterations", "model_indices")


def assert_same(got, want):
    """every output of the call bit for bit"""
    for k in FIELDS:
        assert got[k] == want[k], (k, got[k], want[k])
    assert same_bits(got["coeffs"], want["coeffs"]), (got["coeffs"], want["coeffs"])
    assert same_bits(got["filtered"], want["filtered"])
    assert same_bits(got["inliers"], want["inliers"])
