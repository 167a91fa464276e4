"""Shared by the approximate voxel-grid tests: the sequential reference (tests/approx_voxelgrid_ref.cpp, compiled into a temporary
directory), a bitwise comparison of float records, and the adversarial clouds."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "approx_voxelgrid_ref.cpp")


class Reference:
    def __init__(self, tmpdir):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
        so = os.path.join(str(tmpdir), "libavg_ref.so")
        # -ffp-contract=off as for the oracle: the reference is built without FMA (/root/reference/CMakeLists.txt:10-11)
        subprocess.check_call([cxx, "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-Wall", "-o", so, SRC])
        self.lib = C.CDLL(so)
        self.lib.ref_approximate_voxelgrid.restype = C.c_size_t
        self.lib.ref_approximate_voxelgrid.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_float, C.c_void_p, C.c_void_p]
        self.lib.ref_x86_cvtt.restype = C.c_int
        self.lib.ref_x86_cvtt.argtypes = [C.c_float]
        self.lib.ref_static_cast_int.restype = C.c_int
        self.lib.ref_static_cast_int.argtypes = [C.c_float]

    def approximate_voxelgrid(self, cloud, leaf):
        """(outputs (m, stride) float32 in PCL's order, points per output (m,) int32)"""
        a = np.ascontiguousarray(cloud, np.float32)
        n, s = a.shape
        out = np.zeros((max(n, 1), s), np.float32)
        counts = np.zeros(max(n, 1), np.int32)
        m = self.lib.ref_approximate_voxelgrid(a.ctypes.data, n, s, C.c_float(leaf), out.ctypes.data, counts.ctypes.data)
        return out[:m], counts[:m]


def bits(a):
    """float32 array -> its uint32 bit patterns, every NaN folded into one pattern.  NaN payloads and signs are not part of the
    result: x86 propagates an operand's payload (and makes inf - inf a negative NaN), the GPU returns one canonical NaN."""
    a = np.ascontiguousarray(a, np.float32)
    u = a.view(np.uint32).copy()
    u[np.isnan(a)] = 0x7FC00000
    return u


def same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def records(xyz, stride, intensity=None):
    """(n, 3) coordinates -> (n, stride) float32 records: x y z 1 [intensity 0 0 0]"""
    xyz = np.asarray(xyz, np.float32)
    out = np.zeros((xyz.shape[0], stride), np.float32)
    out[:, :3] = xyz
    if stride >= 4:
        out[:, 3] = 1.0
    if stride >= 5:
        out[:, 4] = np.arange(xyz.shape[0]) % 97 * 0.5 if intensity is None else intensity
    return out


def decorate(cloud, seed):
    """a copy with exact lattice ties (every 97th point rounded to whole metres) and a few NaN / +-inf points"""
    c = np.array(cloud, np.float32, copy=True)
    c[::97, :3] = np.round(c[::97, :3])
    rng = np.random.default_rng(seed)
    bad = rng.choice(c.shape[0], 6, replace=False)
    c[bad[0], 0] = np.nan
    c[bad[1], 1] = np.nan
    c[bad[2], 2] = np.inf
    c[bad[3], 0] = -np.inf
    c[bad[4], :3] = np.nan
    c[bad[5], 1] = np.inf
    return c


def case(name, stride=8):
    """(cloud, leaf) of one named adversarial or boundary case"""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "negative":  # every coordinate negative: floor rounds away from zero
        xyz = rng.uniform(-40.0, -0.001, (6000, 3))
        return records(xyz, stride), 0.25
    if name == "boundaries":  # points exactly on cell faces (k * leaf in float32), +-0.0 and one ulp either side
        leaf = np.float32(0.1)
        k = rng.integers(-200, 200, (3000, 3)).astype(np.float32)
        xyz = k * leaf
        xyz[::3] = np.nextafter(xyz[::3], np.float32(np.inf))
        xyz[1::7] = np.nextafter(xyz[1::7], np.float32(-np.inf))
        xyz[2::11] = np.float32(-0.0)
        xyz[5::13, 0] = np.float32(0.0)
        return records(xyz, stride), float(leaf)
    if name == "nonfinite":  # NaN, +-inf and |x / leaf| >= 2^31 mixed into an ordinary cloud, all of which land in cell INT_MIN
        xyz = rng.uniform(-20.0, 20.0, (4000, 3)).astype(np.float32)
        specials = np.array([np.nan, np.inf, -np.inf, 3e9, -3e9, 2147483648.0, -2147483648.0, 2147483520.0, -2147483520.0, 1e30, -1e38],
                            np.float32)
        idx = rng.choice(xyz.shape[0], 600, replace=False)
        xyz[idx, rng.integers(0, 3, idx.size)] = specials[rng.integers(0, specials.size, idx.size)]
        xyz[idx[:40]] = np.nan
        return records(xyz, stride), 1.0
    if name == "same_bucket_alternating":  # cells (0,0,0) and (512,0,0) share bucket 0: every point flushes the other cell
        n = 3001
        xyz = np.zeros((n, 3), np.float32)
        xyz[:, 0] = np.where(np.arange(n) % 2 == 0, 0.25, 512.25)
        xyz[:, 1] = rng.uniform(0.0, 0.99, n)
        xyz[:, 2] = rng.uniform(0.0, 0.99, n)
        return records(xyz, stride), 1.0
    if name == "one_cell":  # every point in cell (3, -2, 7)
        xyz = np.array([3.0, -2.0, 7.0]) + rng.uniform(0.0, 0.999, (20000, 3))
        return records(xyz, stride), 1.0
    if name == "every_bucket":  # cells (i, 0, 0), i < 512, one point each: 7171 is odd, so they fill all 512 buckets; shuffled
        xyz = np.c_[rng.permutation(512) + 0.5, np.full(512, 0.5), np.full(512, 0.5)]
        return records(xyz, stride), 1.0
    raise KeyError(name)


CASES = ("negative", "boundaries", "nonfinite", "same_bucket_alternating", "one_cell", "every_bucket")
