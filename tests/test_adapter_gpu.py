"""GPU: the pcl::Registration adapter (adapter/b200_registration.hpp) EXECUTED, through tests/adapter_harness.cpp and the test-only
PCL stand-in adapter/pcl_shim.hpp, the way ScanMatchingOdometryNodelet::matching and its status publisher drive the handle
(apps/scan_matching_odometry_nodelet.cpp:172-246, :298-321).  For GICP and both NDT methods: poses and flags bitwise those of
b2r_align on a plain handle; getFitnessScore (through the base pointer) and the inlier count equal to a sequential numpy sum over
b2r_target_nearest's distances of the shim-transformed cloud; the `output` cloud of align bit-equal to that transform; ONE kernel
launch behind both sweeps (plus one per non-finite point, which the cache cannot serve); and the nearest-neighbour cache exact and
really used by consumers that restart, skip, go backwards, ask for foreign points, re-align, and switch keyframes."""
import os
import subprocess
import numpy as np
import pytest
import torch  # noqa: F401  before the engine library: it links the system NCCL, and torch's CUDA libraries must resolve against their own first
import hdl_graph_slam_b200 as pkg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
FLT_MAX = np.finfo(f32).max
NAN_AT, DUP_AT = (20, 300), (30, 700)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    from hdl_graph_slam_b200 import build
    build.build_engine()
    exe = str(tmp_path_factory.mktemp("adapter") / "adapter_harness")
    lib = os.path.join(ROOT, "hdl_graph_slam_b200", "_lib")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++14", "-O1", "-Wall", "-ffp-contract=off",
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "hdl_graph_slam_b200", "adapter"), "-o", exe,
                           os.path.join(ROOT, "tests", "adapter_harness.cpp"), "-L", lib, "-lb200reg", "-Wl,-rpath," + lib])
    return exe


@pytest.fixture(scope="module")
def frames(synth):
    fr = [synth.scan("vlp16_16k", frame=k, stride=8).copy() for k in range(5)]
    last = fr[-1]
    for i in NAN_AT:  # non-finite source points: same_point() is false for them, every query is a single exact one
        last[i, 0] = np.nan
    for i in DUP_AT:  # duplicate source points
        last[i + 1] = last[i]
    return fr


SWITCH = [0, 0, 1, 0, 0]  # the keyframe switches after frame 2


def shim_transform(T_col, cloud):
    """adapter/pcl_shim.hpp transformPointCloud: ((m0 x + m4 y) + m8 z) + m12 in float32, the record otherwise copied"""
    m = np.asarray(T_col, f32)
    x, y, z = cloud[:, 0], cloud[:, 1], cloud[:, 2]
    out = cloud.copy()
    with np.errstate(invalid="ignore"):
        for r in range(3):
            out[:, r] = ((m[r] * x + m[4 + r] * y) + m[8 + r] * z) + m[12 + r]
    return out


def nearest_ref(reg, q):
    """what DeviceSearch::nearestKSearch answers point by point: b2r_target_nearest, and (-1, FLT_MAX) when nothing is found"""
    idx, d2 = reg.nearestKSearch(q)
    return idx, np.where(idx < 0, FLT_MAX, d2).astype(f32)


def fitness_ref(d2):
    s, nr = 0.0, 0
    for d in d2.astype(np.float64):  # sequential, in index order, as the base class sums; `d <= max_range` drops a NaN
        if d <= np.finfo(np.float64).max:
            s += d
            nr += 1
    return s / nr if nr else np.finfo(np.float64).max


def same_xyz(a, b):
    a, b = np.ascontiguousarray(a, f32), np.ascontiguousarray(b, f32)
    nan = np.isnan(a) & np.isnan(b)
    return np.array_equal(a.view(np.uint32)[~nan], b.view(np.uint32)[~nan])


class Reader:
    def __init__(self, a):
        self.a, self.i = a, 0

    def take(self, n=None):
        if n is None:
            self.i += 1
            return self.a[self.i - 1]
        self.i += n
        return self.a[self.i - n:self.i]


@pytest.mark.parametrize("method", [pkg.B2R_METHOD_GICP, pkg.B2R_METHOD_NDT, pkg.B2R_METHOD_NDT_PCL], ids=["gicp", "ndt_omp", "ndt"])
def test_adapter_walk_and_cache(harness, frames, tmp_path, method):
    with open(tmp_path / "in.bin", "wb") as f:
        f.write(np.int32(len(frames)).tobytes())
        for c, s in zip(frames, SWITCH):
            f.write(np.array([c.shape[0], s], np.int32).tobytes())
            f.write(np.ascontiguousarray(c, f32).tobytes())
    out = subprocess.run([harness, str(method), str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    r = Reader(np.fromfile(tmp_path / "out.bin"))

    cfg = pkg.default_config(method)
    cfg.ndt_resolution = 1.0
    reg = pkg.Registration(cfg)
    reg.setInputTarget(frames[0])
    prev = np.eye(4, dtype=f32)
    for k in range(1, len(frames)):
        reg.setInputSource(frames[k])
        reg.align(prev)
        T = reg.getFinalTransformation()
        assert bool(r.take()) == reg.hasConverged(), k
        Tcol = r.take(16).astype(f32)
        assert np.array_equal(Tcol.view(np.uint32), np.ascontiguousarray(T.T).reshape(-1).view(np.uint32)), k  # bitwise b2r_align
        want_aligned = shim_transform(Tcol, frames[k])
        idx, d2 = nearest_ref(reg, want_aligned)
        assert r.take() == fitness_ref(d2), k
        assert r.take() == int((d2 < f32(0.25)).sum()), k
        n_nan = int(np.isnan(frames[k][:, :3]).any(axis=1).sum())
        assert r.take() == 1 + 2 * n_nan, k  # ONE launch serves getFitnessScore and the inlier sweep
        n = int(r.take())
        assert n == frames[k].shape[0]
        assert same_xyz(r.take(3 * n).reshape(n, 3), want_aligned[:, :3]), k  # align()'s output cloud
        if reg.hasConverged():
            prev = T
        if SWITCH[k]:
            reg.setInputTarget(frames[k])
            prev = np.eye(4, dtype=f32)
    assert n_nan == len(NAN_AT)
    aligned = want_aligned
    # ---- the awkward consumers: every answer is the uncached single query's
    single = lambda p: nearest_ref(reg, np.asarray(p, f32).reshape(1, -1))  # noqa: E731
    launches = {}
    for _ in range(int(r.take())):
        i = int(r.take())
        found, gi, gd, nl = r.take(4)
        wi, wd = single(aligned[i])
        assert (found, gi, f32(gd)) == (1, wi[0], wd[0]), i
        launches.setdefault(i, []).append(nl)
    for i in (1, 2, 10, 11, 11 + 64, 11 + 64 + 1):  # the restart at 0, the cursor, the look-ahead window up to its last slot
        assert launches[i] == [0], (i, launches)
    assert launches[0][0] == 0 and launches[400] == [1]  # beyond the window: one exact query
    assert all(v <= 1 for vs in launches.values() for v in vs)
    cnt, extra = r.take(2)
    assert cnt == 20 and extra == 0  # steps of 64 stay inside the window: served from the cache
    odd = r.take(3).astype(f32)
    found, gi, gd, nl = r.take(4)
    wi, wd = single(np.r_[odd, 1.0])
    assert (found, gi, f32(gd), nl) == (1, wi[0], wd[0], 1)  # a point that is not in the cloud: the miss path
    found, gi, gd, nl = r.take(4)
    wi, wd = single(aligned[6])
    assert (found, gi, f32(gd)) == (1, wi[0], wd[0]) and nl <= 1
    # ---- pointer early-outs
    up_src, up_other, up_same = r.take(3)
    assert up_src == 0 and up_other == frames[3].shape[0] * 32 and up_same == 0
    # ---- a second align on the same source (target now frame 3): a fresh cache, one launch again
    reg.setInputTarget(frames[3])
    far = np.eye(4, dtype=f32)
    far[0, 3] = 0.7
    reg.align(far)
    T = reg.getFinalTransformation()
    assert bool(r.take()) == reg.hasConverged()
    Tcol = r.take(16).astype(f32)
    assert np.array_equal(Tcol.view(np.uint32), np.ascontiguousarray(T.T).reshape(-1).view(np.uint32))
    want_aligned = shim_transform(Tcol, frames[4])
    idx, d2 = nearest_ref(reg, want_aligned)
    assert r.take() == fitness_ref(d2)
    assert r.take() == 1 + len(NAN_AT)
    n = int(r.take())
    assert same_xyz(r.take(3 * n).reshape(n, 3), want_aligned[:, :3])
    # ---- a third align straight after that sweep: another pose, so the second align's cache would answer for the wrong cloud
    other = np.eye(4, dtype=f32)
    other[1, 3] = -0.5
    reg.align(other)
    T3 = reg.getFinalTransformation()
    assert not np.array_equal(T3, T)
    assert bool(r.take()) == reg.hasConverged()
    Tcol = r.take(16).astype(f32)
    assert np.array_equal(Tcol.view(np.uint32), np.ascontiguousarray(T3.T).reshape(-1).view(np.uint32))
    idx, d2 = nearest_ref(reg, shim_transform(Tcol, frames[4]))
    assert r.take() == fitness_ref(d2)
    assert r.take() == 1 + len(NAN_AT)
    # ---- keyframe switch, then the same cloud as the next source: uploaded again, aligned onto itself
    assert r.take() == frames[4].shape[0] * 32
    reg.setInputTarget(frames[4])
    reg.setInputSource(frames[4])
    reg.align(np.eye(4, dtype=f32))
    assert bool(r.take()) == reg.hasConverged()
    idx, d2 = nearest_ref(reg, shim_transform(np.ascontiguousarray(reg.getFinalTransformation().T).reshape(-1), frames[4]))
    assert r.take() == fitness_ref(d2)
    # ---- an empty source
    assert list(r.take(3)) == [0, 0, 1]
    assert r.i == len(r.a)
    reg.close()
