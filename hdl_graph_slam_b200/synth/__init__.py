"""ctypes wrapper of the synthetic LiDAR generator (synth/lidar_synth.c; SURVEY.md §8d).  Workload tooling only."""
import ctypes as C
import os
import numpy as np

_LIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "_lib", "libb2r_synth.so")
_lib = None

SENSORS = {"vlp16": (16, 4096), "vlp16_16k": (16, 1024), "hdl32e": (32, 4096), "kitti": (64, 1875)}


def _load():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB):
            raise RuntimeError(f"{_LIB} missing: run `python -m hdl_graph_slam_b200.build`")
        _lib = C.CDLL(_LIB)
        _lib.b2s_scan.restype = C.c_size_t
        _lib.b2s_scan.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_uint64, C.c_double,
                                  C.c_void_p, C.c_size_t]
        _lib.b2s_pose.restype = None
        _lib.b2s_pose.argtypes = [C.c_int, C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]
    return _lib


def pose(k, step=1.0):
    """(x, y, yaw) of trajectory frame k (closed circuit, radius 40 +- 2 m, ~`step` metres per frame, ~251.3 frames per lap)"""
    x, y, th = C.c_double(), C.c_double(), C.c_double()
    _load().b2s_pose(int(k), float(step), C.byref(x), C.byref(y), C.byref(th))
    return x.value, y.value, th.value


def pose_matrix(k, step=1.0):
    x, y, th = pose(k, step)
    T = np.eye(4)
    T[0, 0], T[0, 1], T[1, 0], T[1, 1] = np.cos(th), -np.sin(th), np.sin(th), np.cos(th)
    T[0, 3], T[1, 3], T[2, 3] = x, y, 1.8
    return T


def scan(sensor="vlp16", frame=0, step=1.0, sigma=0.02, stride=8, xyyaw=None, roll=0.0, pitch=0.0, seed=None, out=None):
    """One synthetic scan in the sensor frame: float32 (n, stride) array (stride 8 == pcl::PointXYZI record).  `sensor` is a name of
    SENSORS or a (rings, azimuth steps) pair with 2 to 64 rings; other shapes raise ValueError."""
    rings, n_az = SENSORS[sensor] if isinstance(sensor, str) else sensor
    x, y, th = pose(frame, step) if xyyaw is None else xyyaw
    n = rings * n_az
    if out is None:
        out = np.zeros((n, stride), np.float32)
    sd = (0xB2000000 + frame) if seed is None else seed
    if _load().b2s_scan(rings, n_az, x, y, th, roll, pitch, sd, sigma, out.ctypes.data_as(C.c_void_p), stride) != n:
        raise ValueError(f"scan shape ({rings}, {n_az}): the generator takes 2 to 64 rings and at least one azimuth step")
    return out
