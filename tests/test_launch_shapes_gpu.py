"""Every launch shape of the two cluster kernels against the oracle.

k_bvh_build_cluster<CL, PER, SINGLE> (csrc/bvh_build.cuh) and k_voxelgrid_cluster<CL, PER> (csrc/voxelgrid.cuh) are compiled in
nine (cluster size, pairs per thread) shapes, and build_shape_for(n, wide) picks one by cloud size: (1,1) (2,1) (4,1) (8,1) (8,2)
(8,4) (8,8), then (16,8) above 65 536 points, or (8,16) where a 16-CTA cluster is refused (cluster16_allowed(), B2R_NO_CLUSTER16).
Each test cloud sits at one end of a shape's size range, so some end exactly on a CTA boundary and others leave whole CTAs of the
cluster as padding.  Every cloud holds lattice ties, exact duplicates across a slice boundary and non-finite points at index 0,
at n - 1 and on both sides of every CTA slice boundary; a few sizes also take degenerate clouds (planar, all identical, one far
stray point, one finite point, none finite).

- structure build, through a GICP handle: 1-NN of foreign queries and of the cloud itself == oracle.knn (indices and float32
  distances bit for bit, no dropped point returned), covariances == oracle.gicp_covariances to 1e-8 at k = 20 (register kernel)
  and k = 7 (generic kernel);
- voxel grid: keys, counts, order, centroids and intensity == oracle.voxelgrid bit for bit at leaf 0.1, at 20 m (voxels whose
  runs continue through several CTAs' slices) and at a leaf that trips PCL's overflow rule (input passed through);
- the launch counters prove the one-kernel cluster path ran (one launch per build or filter; the fallback chains count 10 and 14);
- batched build: one RegistrationBatch holds clouds of every shape the process launches plus an empty cloud, built by one launch
  per shape; fitness == oracle, align == the single handle's bit for bit, map cloud == the host entry point row for row;
- the (8,16) shape, which an H100 never picks by itself: the same checks and a KITTI-size odometry with the voxel-grid downsample
  in a child process under B2R_NO_CLUSTER16=1, equal to the oracle and bit for bit to this process's (16,8) outputs;
- on the CPU: the size list reaches all nine shapes (tests/shape_harness.cu prints what build_shape_for picks)."""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch  # noqa: F401  before the engine library: it links the system NCCL, and torch's CUDA libraries must resolve against their own first
import hdl_graph_slam_b200 as pkg
from test_large_clouds_gpu import check_covariances

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# both ends of every shape's size range (the wide shapes, as an H100 picks them)
SIZES = (1, 1024, 1025, 2048, 2049, 4096, 4097, 8192, 8193, 16384, 16385, 32768, 32769, 65536, 65537, 131071, 131072)
NARROW_SIZES = (65537, 100000, 131071, 131072)   # run again with 16-CTA clusters refused: the (8,16) shape
DEGENERATE = ("planar", "identical", "stray", "one_finite", "none_finite")
DEGENERATE_SIZES = (2049, 32769, 131072)
LEAVES = (0.1, 20.0, 1e-4)                       # many short runs; runs across CTA slices; PCL's overflow rule
I4 = np.eye(4, dtype=np.float32)
GICP = {"registration_method": "FAST_GICP"}


def shape_of(n, wide):
    """(cluster size, pairs per thread) of an n-point cloud: build_shape_for restated (test_size_list_reaches_every_shape pins it)"""
    slices = max(1, -(-n // 1024))
    if slices > 128:
        return 0, 0
    if wide and slices > 64:
        return 16, 8
    per = 1
    while per * 8 < slices:
        per *= 2
    cl = 1
    while cl * per < slices:
        cl *= 2
    return cl, per


SHAPE_INDEX = {(1, 1): 0, (2, 1): 1, (4, 1): 2, (8, 1): 3, (8, 2): 4, (8, 4): 5, (8, 8): 6, (8, 16): 7, (16, 8): 8}


def slice_bounds(n):
    """the first index of every CTA slice after the first, under either shape the size can take"""
    out = set()
    for wide in (True, False):
        cl, per = shape_of(n, wide)
        out |= {k * per * 1024 for k in range(1, cl) if k * per * 1024 < n}
    return sorted(out)


def shaped_cloud(base, n, kind="decorated"):
    """the first n points of `base` (an hdl32e scan, 32-byte records) with lattice ties, exact duplicates across slice boundaries
    and non-finite points at 0, n - 1 and around every slice boundary; `kind` makes it degenerate on top of that"""
    c = np.array(base[:n], np.float32, copy=True)
    c[::97, :3] = np.round(c[::97, :3])                    # lattice ties
    if n >= 64:
        c[40:48, :3] = c[20:28, :3]                        # exact duplicates
    bounds = slice_bounds(n)
    for b in bounds:
        if b + 2 < n:
            c[b + 2, :3] = c[b - 3, :3]                    # a duplicate whose copies lie in two slices
    if n > 1:
        bad = sorted({0, n - 1} | {b - 1 for b in bounds} | set(bounds))
        pattern = ((0, np.nan), (1, np.inf), (2, -np.inf), (slice(0, 3), np.nan))
        for j, i in enumerate(bad):
            col, v = pattern[j % 4]
            c[i, col] = v
    fin = np.isfinite(c[:, :3]).all(axis=1)
    if kind == "planar":                                   # zero extent along z: one axis of the Hilbert box collapses
        c[fin, 2] = 1.5
    elif kind == "identical":                              # every finite point the same: the 1e-6 extent clamp
        c[fin, :3] = (1.25, -0.5, 2.0)
    elif kind == "stray":                                  # one point 1e6 m away squeezes the rest into a few Hilbert cells
        c[n // 3, :3] = (1.0e6, -3.0, 2.0)
    elif kind == "one_finite":
        c[:, :3] = np.nan
        c[n // 2, :3] = (3.0, -4.0, 0.5)
    elif kind == "none_finite":
        c[:, :3] = np.nan
        c[1::3, 1] = np.inf
        c[2::3, 2] = -np.inf
    return c


def finite_rows(c):
    return np.isfinite(c[:, :3]).all(axis=1)


def sha(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def launches(reg, cls):
    return reg.getStats()["launches"][cls]


def gicp(k=20):
    return pkg.select_registration_method({"registration_method": "FAST_GICP", "reg_correspondence_randomness": k})


def check_structure(oracle, cloud, queries):
    """1-NN and covariances of `cloud` as a GICP target == oracle; one cluster launch per build.  Returns output hashes."""
    fin = finite_rows(cloud)
    q = np.concatenate([queries, cloud[fin]])
    out = {}
    reg = gicp(20)
    b0 = launches(reg, "bvh_build")
    reg.setInputTarget(cloud)
    idx, d2 = reg.nearestKSearch(q)
    assert launches(reg, "bvh_build") - b0 == 1, "the structure build left the one-kernel cluster path"
    oi, od = oracle.knn(cloud, q, 1)
    assert np.array_equal(idx, oi[:, 0]) and np.array_equal(d2.view(np.uint32), od[:, 0].view(np.uint32))
    hit = idx >= 0
    assert np.all(fin[idx[hit]]), "a dropped point was returned as a neighbour"
    assert hit.all() == bool(fin.any())
    out["idx"], out["d2"] = sha(idx), sha(d2)
    for k, r in ((20, reg), (7, None)):
        if r is None:
            r = gicp(k)
            b0 = launches(r, "bvh_build")
            r.setInputTarget(cloud)
        got = r.getCovariances(1, cloud.shape[0])
        assert launches(r, "bvh_build") - b0 == 1
        if fin.sum() > k:
            check_covariances(oracle, got, cloud, k)
        else:  # fewer points than neighbours: every neighbourhood is the whole finite cloud
            want = oracle.gicp_covariances(cloud, k)
            assert np.max(np.abs(got[fin] - want[fin]), initial=0.0) < 1e-8
        assert np.all(np.isnan(got[~fin]))
        out[f"cov{k}"] = sha(np.nan_to_num(got, nan=-1.0))
        r.close()
    return out


def check_voxelgrid(reg, oracle, cloud, leaf):
    """voxelGridFilter == oracle.voxelgrid bit for bit, through one cluster launch.  Returns (rc, output hash)."""
    v0 = launches(reg, "voxelgrid_downsample")
    out, keys, counts, rc = reg.voxelGridFilter(cloud, leaf, with_keys=True)
    assert launches(reg, "voxelgrid_downsample") - v0 == 1, "the voxel grid left the one-kernel cluster path"
    oo, ok, oc, orc_ = oracle.voxelgrid(cloud, leaf)
    assert rc == orc_
    if rc == 1:  # PCL warns and passes the input through
        assert np.array_equal(out.view(np.uint32), cloud.view(np.uint32))
        return rc, sha(out)
    assert out.shape[0] == oo.shape[0] == keys.shape[0] == counts.shape[0]
    assert np.array_equal(keys, ok) and np.all(np.diff(keys) > 0)
    assert np.array_equal(counts, oc) and counts.sum() == finite_rows(cloud).sum()
    assert np.array_equal(out[:, :3].view(np.uint32), oo[:, :3].view(np.uint32))
    assert np.array_equal(out[:, 4].view(np.uint32), oo[:, 3].view(np.uint32))
    assert np.all(out[:, 3] == 1.0)
    return rc, sha(np.concatenate([out.reshape(-1).view(np.int32), keys, counts]))


def check_voxelgrids(oracle, cloud, overflow_expected):
    reg = gicp()
    res = {}
    for leaf in LEAVES:
        rc, h = check_voxelgrid(reg, oracle, cloud, leaf)
        res[f"vg{leaf:g}"] = h
        if leaf == 1e-4 and overflow_expected:
            assert rc == 1, "the overflow rule did not trip"
        if leaf == 20.0 and overflow_expected:
            assert rc == 0
    reg.close()
    return res


def foreign_queries(synth):
    return synth.scan("vlp16_16k", frame=4, stride=8)[:4096].copy()


def size_outputs(synth, oracle, n):
    base = synth.scan("hdl32e", frame=3, stride=8)
    cloud = shaped_cloud(base, n)
    out = check_structure(oracle, cloud, foreign_queries(synth))
    out.update(check_voxelgrids(oracle, cloud, overflow_expected=n > 1))
    return out


def batch_outputs(synth, oracle, sizes):
    """one batch, clouds of `sizes` plus an empty one, all built by the first call (one launch per shape): fitness == oracle,
    align == the single handle, map cloud == the host entry point.  Returns output hashes."""
    base = synth.scan("hdl32e", frame=3, stride=8)
    clouds = [shaped_cloud(base, n) for n in sizes] + [np.zeros((0, 8), np.float32)]
    q = foreign_queries(synth)
    rel = (np.linalg.inv(synth.pose_matrix(3)) @ synth.pose_matrix(4)).astype(np.float32)
    lb = pkg.RegistrationBatch(params=GICP)
    ids = [lb.addCloud(c) for c in clouds]
    qid = lb.addCloud(q)
    lb.calcFitnessScore([(qid, qid, I4)])  # the query cloud's own structure, so that the call below builds only the clouds under test
    b0 = launches(lb.engine, "bvh_build")
    scores = lb.calcFitnessScore([(cid, qid, rel) for cid in ids], 2.5)
    shapes = {shape_of(c.shape[0], True) for c in clouds if c.shape[0]}
    # one launch per shape when 16-CTA clusters are allowed; under B2R_NO_CLUSTER16 (16,8) sizes take (8,16): the count is the same
    assert launches(lb.engine, "bvh_build") - b0 == len(shapes)
    for c, s in zip(clouds, scores):
        fs, fn, _ = oracle.fitness(c, q, rel, 2.5)
        assert (s == fs) if fn == 0 else abs(s - fs) <= 1e-12 * fs, c.shape[0]
    out = {"fitness": sha(scores)}
    pairs = [(qid, cid, rel) for cid, c in zip(ids, clouds) if finite_rows(c).sum() >= 20]
    res = lb.align(pairs, True, 2.5)
    reg = gicp()
    reg.setInputSource(q)
    for (_, cid, g), r in zip(pairs, res):
        reg.setInputTarget(clouds[ids.index(cid)])
        reg.align(g)
        assert np.array_equal(reg.getFinalTransformation(), r["T"]), clouds[ids.index(cid)].shape[0]
        assert reg.hasConverged() == r["converged"] and reg.nr_iterations == r["iterations"]
    out["align"] = sha(np.stack([r["T"] for r in res]))
    poses = [synth.pose_matrix(k) for k in range(len(ids))]
    for res_ in (0.0, 0.25):
        got = lb.mapCloudGenerate(ids, poses, res_)
        want = lb.engine.mapCloudGenerate(list(zip(clouds, poses)), res_)
        assert got.shape == want.shape and got.shape[0] > 0
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        out[f"map{res_:g}"] = sha(got)
    reg.close()
    lb.close()
    return out


def odometry_outputs(synth, oracle):
    """GICP odometry with the nodelet's VOXELGRID downsample on raw 120 000-point KITTI-shape scans: the odometry's own filter
    slots pick their cluster shape separately from the handle's"""
    frames = [synth.scan("kitti", frame=k, stride=8) for k in range(4)]
    reg = gicp()
    out = {"vg_kitti": check_voxelgrid(reg, oracle, frames[0], 0.1)[1]}
    odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=1.5, keyframe_delta_angle=1.0, keyframe_delta_time=10000.0,
                                   downsample_method=pkg.B2R_DOWNSAMPLE_VOXELGRID, downsample_resolution=0.1)
    sts = []
    for k, c in enumerate(frames):
        st = odo.matching(0.1 * k, c)
        sts.append(np.concatenate([st["odom"].reshape(-1).view(np.uint32), [st["iterations"], st["converged"], st["keyframe_updated"]]]))
    assert all(s[-2] for s in sts[1:])
    odo.close()
    reg.close()
    out["odometry"] = sha(np.stack(sts).astype(np.uint32))
    return out


def narrow_outputs(synth, oracle):
    """every check of the (8,16) sizes; the same in the default process, where those sizes take (16,8)"""
    res = {str(n): size_outputs(synth, oracle, n) for n in NARROW_SIZES}
    res["batch"] = batch_outputs(synth, oracle, NARROW_SIZES)
    res.update(odometry_outputs(synth, oracle))
    return res


# ------------------------------------------------------------------------------------------------------------------- CPU
def test_size_list_reaches_every_shape(tmp_path):
    """build_shape_for, compiled from the engine's header, over this file's sizes: all nine shapes are reached, (8,16) through
    wide = false, and shape_of (which places the slice-boundary points) restates it exactly"""
    exe = tmp_path / "shape_harness"
    subprocess.check_call(["nvcc", "-O1", "-std=c++17", "-w", "-gencode", "arch=compute_90a,code=sm_90a", "-ccbin",
                           "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-o", str(exe), os.path.join(HERE, "shape_harness.cu")])
    sizes = sorted(set(SIZES) | set(NARROW_SIZES) | set(DEGENERATE_SIZES) | {131073})
    out = subprocess.run([str(exe)] + [str(n) for n in sizes], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stdout + out.stderr
    rows = [tuple(int(x) for x in line.split()) for line in out.stdout.split("\n") if line.strip()]
    assert len(rows) == 2 * len(sizes)
    for n, wide, index, cl, per in rows:
        assert shape_of(n, bool(wide)) == (cl, per), (n, wide)
        assert index == SHAPE_INDEX.get((cl, per), -1)
    wide_hits = {index for n, wide, index, _, _ in rows if wide and n in SIZES}
    narrow_hits = {index for n, wide, index, _, _ in rows if not wide and n in NARROW_SIZES}
    assert wide_hits == set(range(9)) - {7}
    assert narrow_hits == {7}
    assert wide_hits | narrow_hits == set(range(9))
    # both ends of every wide shape's range: the first and the last size of each shape are in the list
    index_of = {n: index for n, wide, index, _, _ in rows if wide}
    for n in SIZES:
        for m in (n - 1, n + 1):
            if 1 <= m <= 131072 and SHAPE_INDEX[shape_of(m, True)] != index_of[n]:
                assert m in SIZES, (n, m)


# ------------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_every_shape_matches_the_oracle(synth, oracle, n):
    size_outputs(synth, oracle, n)


@pytest.mark.gpu
@pytest.mark.parametrize("n", DEGENERATE_SIZES)
@pytest.mark.parametrize("kind", DEGENERATE)
def test_degenerate_clouds_match_the_oracle(synth, oracle, kind, n):
    cloud = shaped_cloud(synth.scan("hdl32e", frame=3, stride=8), n, kind)
    check_structure(oracle, cloud, foreign_queries(synth))
    check_voxelgrids(oracle, cloud, overflow_expected=kind in ("planar", "stray"))


@pytest.mark.gpu
def test_batched_build_of_every_shape(synth, oracle):
    """two clouds of each shape (the ends of its range) and an empty cloud in one batch"""
    sizes = (1, 1024, 1025, 2048, 2049, 4096, 4097, 8192, 8193, 16384, 16385, 32768, 32769, 65536, 65537, 131072)
    assert len({shape_of(n, True) for n in sizes}) == 8
    batch_outputs(synth, oracle, sizes)


@pytest.mark.gpu
def test_portable_cluster_shape_under_no_cluster16(synth, oracle):
    """B2R_NO_CLUSTER16=1 (what a device that refuses 16-CTA clusters gets): the (8,16) shape of both kernels, the batched build and
    the odometry's filter slots equal the oracle in the child, and this process's (16,8) outputs bit for bit"""
    want = narrow_outputs(synth, oracle)
    code = ("import sys, json\nsys.path[:0] = [%r, %r]\nimport test_launch_shapes_gpu as T\nfrom hdl_graph_slam_b200 import synth\n"
            "from oracle import oracle as orc\norc.lib()\nprint(json.dumps(T.narrow_outputs(synth, orc)))\n") % (ROOT, HERE)
    env = dict(os.environ)
    env["B2R_NO_CLUSTER16"] = "1"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert got.keys() == want.keys()
    for k in want:
        assert got[k] == want[k], k
