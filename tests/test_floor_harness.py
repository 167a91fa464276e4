"""CPU: the floor-detection device source compiled for the host (tests/ransac_harness.cu) against the sequential reference
(tests/floor_ref.cpp), bit for bit: pcl_eigen33 on 1e5 random and degenerate covariances, and whole RANSAC sample streams."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from floor_ref import Reference, HYP, bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    r = Reference(tmp_path_factory.mktemp("floor_ref"))
    r.lib.ref_eigen33_many.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    return r


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = str(tmp_path_factory.mktemp("ransac_harness") / "libransac_harness.so")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-w", "-gencode", "arch=compute_90a,code=sm_90a", "-ccbin",
                           "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
                           "-o", so, os.path.join(ROOT, "tests", "ransac_harness.cu")])
    lib = C.CDLL(so)
    lib.h_eigen33.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    lib.h_ransac_hypotheses.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p]
    return lib


def covariances(n, seed):
    """n float32 3x3 covariances: random neighbourhoods at many scales and offsets, planes, lines, single points (zero matrix),
    near-FLT_MIN entries, and random symmetric (indefinite) matrices"""
    rng = np.random.default_rng(seed)
    out = np.empty((n, 9), f32)
    kinds = rng.integers(0, 7, n)
    for i, kind in enumerate(kinds):
        k = int(rng.integers(3, 11))
        if kind <= 2:
            P = rng.normal(size=(k, 3)) * rng.uniform(1e-3, 3, 3) + rng.uniform(-50, 50, 3)
            if kind == 1:
                P[:, 2] = P[0, 2] + rng.normal(0, 1e-4)  # planar
            elif kind == 2:
                P = P[0] + np.outer(rng.normal(size=k), rng.normal(size=3))  # collinear
            P = P.astype(f32)
            acc = np.zeros(9, f32)
            for p in P:  # PCL's float32 raw moments in neighbour order
                acc += np.array([p[0] * p[0], p[0] * p[1], p[0] * p[2], p[1] * p[1], p[1] * p[2], p[2] * p[2], p[0], p[1], p[2]], f32)
            acc = acc / f32(k)
            c = [acc[0] - acc[6] * acc[6], acc[1] - acc[6] * acc[7], acc[2] - acc[6] * acc[8], acc[3] - acc[7] * acc[7],
                 acc[4] - acc[7] * acc[8], acc[5] - acc[8] * acc[8]]
            M = np.array([[c[0], c[1], c[2]], [c[1], c[3], c[4]], [c[2], c[4], c[5]]], f32)
        elif kind == 3:
            M = np.zeros((3, 3), f32)
        elif kind == 4:
            M = (rng.normal(size=(3, 3)) * 1e-38).astype(f32)
            M = (M + M.T).astype(f32)
        elif kind == 5:
            M = np.diag(rng.uniform(0, 2, 3)).astype(f32)
            M[rng.integers(0, 3), :] *= 0
            M = np.minimum(M, M.T)
        else:
            M = rng.normal(size=(3, 3)).astype(f32)
            M = (M + M.T).astype(f32)
        out[i] = M.reshape(9)
    return out


@pytest.mark.parametrize("seed", [0, 1])
def test_eigen33_bitwise(ref, harness, seed):
    A = covariances(50000, seed)
    v_ref = np.zeros((len(A), 3), f32)
    v_dev = np.zeros((len(A), 3), f32)
    ref.lib.ref_eigen33_many(A.ctypes.data, len(A), v_ref.ctypes.data)
    harness.h_eigen33(A.ctypes.data, len(A), v_dev.ctypes.data)
    assert np.array_equal(bits(v_ref), bits(v_dev))


def _cloud(seed, n):
    rng = np.random.default_rng(seed)
    c = np.zeros((n, 8), f32)
    c[:, :3] = rng.uniform(-20, 20, (n, 3))
    c[: n // 3, 2] = -1.8
    c[n // 3: n // 2] = c[0]  # duplicates
    c[:, 3] = 1
    return c


@pytest.mark.parametrize("seed,n,count", [(0, 5, 200), (1, 200, 2000), (2, 5000, 10001), (3, 3, 50)])
def test_sample_stream_bitwise(ref, harness, seed, n, count):
    c = _cloud(seed, n)
    want = ref.hypotheses(c, count)
    got = np.zeros(count, HYP)
    harness.h_ransac_hypotheses(c.ctypes.data, n, 8, count, got.ctypes.data)
    assert np.array_equal(got["ok"], want["ok"])
    ok = want["ok"] == 1
    assert np.array_equal(got["idx"][ok], want["idx"][ok])
    assert np.array_equal(bits(got["c"][ok]), bits(want["c"][ok]))


def test_no_sample_stream_bitwise(ref, harness):
    t = (-0.25 - np.arange(1, 301) * 2.0 ** -10).astype(f32)
    c = np.zeros((300, 4), f32)
    c[:, 0], c[:, 1], c[:, 2], c[:, 3] = t, 2 * t, 4 * t, 1
    got = np.zeros(2, HYP)
    harness.h_ransac_hypotheses(c.ctypes.data, 300, 4, 2, got.ctypes.data)
    assert got["ok"][0] == 0 and ref.hypotheses(c, 1)["ok"][0] == 0
