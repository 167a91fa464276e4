"""GPU: clouds beyond the one-cluster limit (131 072 points, csrc/bvh_build.cuh kBuildMaxPoints) against the oracle.

Above that size every structure build leaves the single-kernel cluster path for a chain of launches: the BVH (k_bbox /
k_morton_keys / cub radix sort / k_bvh_leaves, also on the prefetch stream and inside a batch), the voxel grid (k_vg_params /
k_vg_keys / cub sort / k_vg_heads / scan / k_vg_centroid).  Above 2^20 points the prefilter's stream compaction carries its
running offset over more than one group of 1024 block counts, and map-scale map clouds take every grid-stride loop of
map_cloud.cuh through several iterations per thread.  Tolerances are those of DESIGN.md §2: integers, NN indices, float32
distances, voxel-grid outputs and map clouds bit-exact; covariances <= 1e-8 absolute; H, b and cost <= 1e-9 relative; poses
<= 1e-6; the same iteration count and convergence flag.  Every input holds a few NaN / +-inf points and exact lattice ties."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi
from common import rot_err, trans_err, perturb, relrel

pytestmark = pytest.mark.gpu

LIMIT = 131072                 # the largest cloud one thread-block cluster builds
BIG = (64, 4096)               # 262 144 points: a 64-beam scan at 4096 azimuth steps
I4 = np.eye(4, dtype=np.float32)


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


def finite_rows(c):
    return np.isfinite(c[:, :3]).all(axis=1)


def to_world(cloud, T):
    """cloud (sensor frame) moved by the 4x4 pose T in float32, other fields kept"""
    out = np.array(cloud, np.float32, copy=True)
    Tf = np.asarray(T, np.float32)
    out[:, :3] = (cloud[:, :3] @ Tf[:3, :3].T + Tf[:3, 3]).astype(np.float32)
    return out


@pytest.fixture(scope="module")
def big(synth):
    """frame -> decorated 262 144-point scan (32-byte records)"""
    return {f: decorate(synth.scan(BIG, frame=f, stride=8), seed=f) for f in (0, 1)}


@pytest.fixture(scope="module")
def kitti_map(synth):
    """about 1.2 M points: ten KITTI-shape scans, each moved to its pose on the circuit"""
    parts = [to_world(synth.scan("kitti", frame=f, stride=8), synth.pose_matrix(f)) for f in range(10)]
    return decorate(np.concatenate(parts), seed=99)


def check_covariances(oracle, got, cloud, k):
    """engine covariances == oracle's to 1e-8 for every finite point whose k-neighbourhood is well posed.  A neighbourhood
    whose points lie on one line (lattice duplicates make some: 9 copies of a point and one other at k = 10) leaves the PLANE
    normal free in the plane orthogonal to the line, so there only the properties are pinned, as in test_edge_cases_gpu:
    eigenvalues {1e-3, 1, 1} with the 1e-3 direction orthogonal to the line."""
    want = oracle.gicp_covariances(cloud, k)
    ok = finite_rows(cloud)
    nb, _ = oracle.knn(cloud, cloud[ok], k)
    p = cloud[nb][:, :, :3].astype(np.float64)
    d = p - p.mean(axis=1, keepdims=True)
    w, V = np.linalg.eigh(np.einsum("nki,nkj->nij", d, d))
    line = w[:, 1] <= 1e-12 * np.maximum(w[:, 2], 1e-300)
    line &= w[:, 2] > 0  # k copies of one point: both follow JacobiSVD (diag(1, 1, 1e-3)) and are compared
    g, o = got[ok], want[ok]
    assert np.max(np.abs(g[~line] - o[~line])) < 1e-8
    for C in (g[line], o[line]):
        cw, cV = np.linalg.eigh(C)
        assert np.max(np.abs(cw - [1e-3, 1.0, 1.0]), initial=0.0) < 1e-12
        assert np.max(np.abs(np.einsum("ni,ni->n", cV[:, :, 0], V[line][:, :, 2])), initial=0.0) < 1e-6
    return want


def gicp(k=20):
    return pkg.select_registration_method({"registration_method": "FAST_GICP", "reg_correspondence_randomness": k})


# ---------------------------------------------------------------------------------------------------------- 1, 2: BVH chain
@pytest.mark.parametrize("stride", [8, 4])
def test_chain_bvh_exact_nearest_neighbour(synth, oracle, big, stride):
    """a 262 144-point target (chain build, 256 super-nodes): 1-NN indices and float32 d2 bit for bit, for queries inside the
    cloud, on its points (d2 = 0 ties with lattice duplicates), and far outside its bounding box"""
    tgt = np.ascontiguousarray(big[0][:, :stride])
    tgt[1000:1200, :3] = tgt[2000:2200, :3]  # exact duplicates: ties broken by the lowest index
    q = [np.ascontiguousarray(big[1][::16, :stride]), tgt[::4099].copy()]
    rng = np.random.default_rng(5)
    far = np.ones((64, stride), np.float32)  # 300 m to 24 km outside the scan (which ends ~125 m from the sensor)
    far[:, :3] = np.where(rng.uniform(size=(64, 3)) < 0.5, -1.0, 1.0) * (rng.uniform(0.0, 500.0, (64, 3)) + [300.0, 300.0, 300.0])
    far[:8, :3] *= 30.0
    q.append(far)
    q = np.concatenate(q)
    q = q[finite_rows(q)]
    reg = gicp()
    reg.setInputTarget(tgt)
    idx, d2 = reg.nearestKSearch(q)
    oi, od = oracle.knn(tgt, q, 1)
    reg.close()
    assert np.array_equal(idx, oi[:, 0]) and np.array_equal(d2, od[:, 0])
    assert np.all(d2[q.shape[0] - 64:] > 1e4) and np.any(d2 == 0)


@pytest.mark.parametrize("k", [20, 10])
def test_chain_bvh_covariances(oracle, big, k):
    """GICP covariances of a 262 144-point source and target: k = 20 takes the register-list kernel, k = 10 the shared-memory one"""
    src, tgt = big[1], big[0]
    reg = gicp(k)
    reg.setInputTarget(tgt)
    reg.setInputSource(src)
    for which, c in ((0, src), (1, tgt)):
        check_covariances(oracle, reg.getCovariances(which, c.shape[0]), c, k)
    reg.close()


# ------------------------------------------------------------------------------------------ 3, 4: linearise + align by size
def check_pair(oracle, src, tgt):
    reg = gicp()
    reg.setInputTarget(tgt)
    reg.setInputSource(src)
    scov = check_covariances(oracle, reg.getCovariances(0, src.shape[0]), src, 20)
    tcov = check_covariances(oracle, reg.getCovariances(1, tgt.shape[0]), tgt, 20)
    for T in (np.eye(4), perturb(11, 0.3, 2.0)):
        H, b, e = reg.gicpLinearizeAt(T)
        o = oracle.gicp_linearize(src, scov, tgt, tcov, T, 2.5)
        assert np.array_equal(reg.getCorrespondences(src.shape[0]), o["corr"])
        assert relrel(H, o["H"]) < 1e-9 and relrel(b, o["b"]) < 1e-9 and abs(e - o["err"]) <= 1e-9 * abs(o["err"])
    reg.align(I4)
    o = oracle.gicp_align(src, tgt, I4)
    assert reg.hasConverged() == o["converged"] and reg.nr_iterations == o["iterations"]
    assert np.array_equal(reg.getCorrespondences(src.shape[0]), o["corr"])
    T = reg.getFinalTransformation()
    assert trans_err(T, o["T"]) < 1e-6 and rot_err(T, o["T"]) < 1e-6
    for max_range in (np.finfo(np.float64).max, 1.0, 0.01):
        fs, fn, fi = oracle.fitness(tgt, src, o["T"], max_range)
        s, used, inl = reg.getFitnessScore(max_range, T=o["T"], full=True)
        assert used == fn and inl == fi
        assert (s == fs) if fn == 0 else abs(s - fs) <= 1e-12 * fs
    reg.close()


def test_linearize_align_and_fitness_above_the_limit(oracle, big):
    """a 262 144-point pair: covariances, two linearisations, one full align and fitness at three ranges"""
    check_pair(oracle, big[1], big[0])


@pytest.mark.parametrize("n", [LIMIT, LIMIT + 1])
def test_linearize_align_and_fitness_across_the_limit(oracle, big, n):
    """131 072 points take the cluster build (16-CTA or 8-CTA clusters), 131 073 the chain: both equal the oracle"""
    check_pair(oracle, np.ascontiguousarray(big[1][:n]), np.ascontiguousarray(big[0][:n]))


# ------------------------------------------------------------------------------------------------------- 5: voxel-grid chain
def check_voxelgrid(reg, oracle, cloud, leaf):
    out, keys, counts, rc = reg.voxelGridFilter(cloud, leaf, with_keys=True)
    oo, ok, oc, orc_ = oracle.voxelgrid(cloud, leaf)
    assert rc == orc_ == 0
    assert out.shape[0] == oo.shape[0] and 0 < out.shape[0] < cloud.shape[0]
    assert np.array_equal(keys, ok) and np.all(np.diff(keys) > 0)
    assert np.array_equal(counts, oc) and counts.sum() == finite_rows(cloud).sum()
    assert np.array_equal(out[:, :3], oo[:, :3])
    if cloud.shape[1] >= 5:
        assert np.array_equal(out[:, 4], oo[:, 3])
    if cloud.shape[1] >= 4:
        assert np.all(out[:, 3] == 1.0)


@pytest.mark.parametrize("case", ["131073", "262144_packed", "kitti_map"])
def test_voxelgrid_chain_equals_oracle(synth, oracle, big, kitti_map, case):
    reg = gicp()
    if case == "131073":
        check_voxelgrid(reg, oracle, np.ascontiguousarray(big[0][:LIMIT + 1]), 0.1)
    elif case == "262144_packed":
        check_voxelgrid(reg, oracle, np.ascontiguousarray(big[1][:, :4]), 0.1)   # 16-byte x y z 1 records
    else:
        assert kitti_map.shape[0] == 1200000
        check_voxelgrid(reg, oracle, kitti_map, 0.25)
    reg.close()


def test_voxelgrid_leaf_too_small_passes_through_above_the_limit(oracle, big):
    cloud = np.ascontiguousarray(big[0][:200000])
    cloud[17, :3] = [3000.0, 3000.0, 3000.0]
    reg = gicp()
    out, keys, counts, rc = reg.voxelGridFilter(cloud, 0.001, with_keys=True)
    reg.close()
    assert rc == oracle.voxelgrid(cloud, 0.001)[3] == 1
    assert np.array_equal(out, cloud, equal_nan=True) and np.all(keys == -1) and np.all(counts == 1)


# --------------------------------------------------------------------------------- 6: cluster build == chain on one input
_CLUSTER_VS_CHAIN = r'''
import sys, json, hashlib
import numpy as np
sys.path.insert(0, %r)
sys.path.insert(0, %r)
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import synth
from test_large_clouds_gpu import decorate
h = lambda a: hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()
full = decorate(synth.scan("hdl32e", frame=6, stride=8), seed=6)
q = synth.scan("vlp16_16k", frame=7, stride=8)[:4096]
reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
res = {}
for n in %r:
    c = np.ascontiguousarray(full[:n])
    out, keys, counts, rc = reg.voxelGridFilter(c, 0.1, with_keys=True)
    reg.setInputTarget(c)
    idx, d2 = reg.nearestKSearch(q)
    cov = reg.getCovariances(1, n)
    res[str(n)] = dict(m=int(out.shape[0]), rc=int(rc), out=h(np.nan_to_num(out, nan=-1.0)), keys=h(keys), counts=h(counts),
                       idx=h(idx), d2=h(d2), cov=h(np.nan_to_num(cov, nan=-1.0)))
reg.close()
print(json.dumps(res))
'''


def test_cluster_and_chain_builds_agree_on_the_same_input():
    """the same clouds through the one-kernel cluster paths and, with B2R_CUB_SORT=1, through the launch chains: every cluster
    shape's sizes (1, 2, 4, 8 and 16 CTAs) give identical voxel-grid outputs, 1-NN answers and covariances"""
    here = os.path.dirname(os.path.abspath(__file__))
    sizes = (1, 777, 16384, 40000, 65537, LIMIT)
    code = _CLUSTER_VS_CHAIN % (os.path.dirname(here), here, sizes)
    outs = []
    for extra in ({}, {"B2R_CUB_SORT": "1"}):
        env = dict(os.environ)
        env.pop("B2R_CUB_SORT", None)
        env.update(extra)
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        outs.append(json.loads(r.stdout.strip().splitlines()[-1]))
    for n in sizes:
        assert outs[0][str(n)] == outs[1][str(n)], n
    assert all(outs[0][str(n)]["m"] > 0 for n in sizes)


# --------------------------------------------------------------------------------------------- 7: prefilter above the limit
@pytest.mark.parametrize("chain", ["voxelgrid", "radius"])
def test_prefilter_above_the_limit_equals_stagewise_oracle(synth, oracle, chain):
    raw = decorate(synth.scan(BIG, frame=9, stride=8), seed=9)
    reg = gicp()
    if chain == "voxelgrid":
        w = (0.01, -0.02, 0.3)
        out, dptr, m = reg.prefilter(raw, deskewing=1, scan_period=0.1, angular_velocity=w, distance_near_thresh=1.0, distance_far_thresh=60.0,
                                     downsample_method=1, downsample_resolution=0.1, outlier_removal_method=0)
        c = oracle.deskew(raw, 0.1, w)
        c = c[oracle.distance_filter(c, 1.0, 60.0)]
        assert c.shape[0] > LIMIT  # the voxel grid gets a cloud above the limit
        xyzi, _, _, rc = oracle.voxelgrid(c, 0.1)
        want = np.zeros((xyzi.shape[0], 8), np.float32)
        want[:, :3], want[:, 3], want[:, 4] = xyzi[:, :3], 1.0, xyzi[:, 3]
    else:
        out, dptr, m = reg.prefilter(raw, distance_near_thresh=1.0, distance_far_thresh=60.0, downsample_method=0, outlier_removal_method=2,
                                     radius_radius=0.3, radius_min_neighbors=3)
        c = raw[oracle.distance_filter(raw, 1.0, 60.0)]
        assert c.shape[0] > LIMIT  # the radius filter's k-NN runs on a chain-built BVH
        keep = oracle.radius_outlier(c, 0.3, 3)
        want = c[keep]
        assert 0 < want.shape[0] < c.shape[0]
    reg.close()
    assert m == want.shape[0] and dptr
    assert np.array_equal(out, want)


# ------------------------------------------------------------------------------------------- 8: compaction above 2^20 points
def test_distance_filter_above_two_to_the_twenty(oracle, kitti_map):
    for cloud in (kitti_map, np.ascontiguousarray(kitti_map[:(1 << 20) + 1])):
        reg = gicp()
        out = reg.distanceFilter(cloud, 2.0, 45.0)
        reg.close()
        keep = oracle.distance_filter(cloud, 2.0, 45.0)
        assert 0 < keep.sum() < cloud.shape[0]
        assert np.array_equal(out, cloud[keep])  # records whole, input order kept


def test_outlier_removal_above_two_to_the_twenty(oracle, kitti_map):
    reg = gicp()
    out = reg.radiusOutlierRemoval(kitti_map, 0.3, 3)
    keep = oracle.radius_outlier(kitti_map, 0.3, 3)
    assert 0 < keep.sum() < kitti_map.shape[0]
    assert np.array_equal(out, kitti_map[keep])
    out = reg.statisticalOutlierRemoval(kitti_map, 20, 1.0)
    keep, _ = oracle.statistical_outlier(kitti_map, 20, 1.0)
    assert 0 < keep.sum() < kitti_map.shape[0]
    assert np.array_equal(out, kitti_map[keep], equal_nan=True)  # non-finite points are kept, as PCL does
    reg.close()


# -------------------------------------------------------------------------------------- 9: batch and prefetch with big clouds
def test_batch_with_a_big_cloud_equals_each_pair_alone(synth, big):
    """one 262 144-point cloud among 16k clouds: the batch builds it with the chain, the small ones with clusters"""
    clouds = {"big": big[0], "a": synth.scan("vlp16_16k", frame=1, stride=8), "b": synth.scan("vlp16_16k", frame=2, stride=8)}
    g = perturb(7, 0.2, 1.0).astype(np.float32)
    pairs = [("a", "big", I4), ("big", "a", g), ("b", "a", I4), ("b", "big", g)]
    lb = pkg.RegistrationBatch(params={"registration_method": "FAST_GICP"})
    ids = {k: lb.addCloud(c) for k, c in clouds.items()}
    res = lb.align([(ids[s], ids[t], gg) for s, t, gg in pairs], True, 2.5)
    lb.close()
    reg = gicp()
    for (s, t, gg), q in zip(pairs, res):
        reg.setInputTarget(clouds[t])
        reg.setInputSource(clouds[s])
        reg.align(gg)
        assert np.array_equal(reg.getFinalTransformation(), q["T"]), (s, t)
        assert reg.hasConverged() == q["converged"] and reg.nr_iterations == q["iterations"]
    reg.close()


def test_prefetched_big_scans_give_identical_odometry(synth):
    """prefetch builds the next scan's BVH (chain) and covariances on the second stream with its own scratch"""
    frames = [decorate(synth.scan(BIG, frame=k, stride=8), seed=20 + k) for k in range(4)]
    outs = []
    for use_prefetch in (False, True):
        reg = gicp()
        odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=1.5, keyframe_delta_angle=1.0, keyframe_delta_time=10000.0)
        res = []
        for k, cloud in enumerate(frames):
            if use_prefetch and k + 1 < len(frames):
                nxt = frames[k + 1]
                odo.prefetch_raw(nxt.ctypes.data, nxt.shape[0], nxt.shape[1] * 4)
            st = odo.matching(0.1 * k, cloud)
            res.append((st["odom"].copy(), st["iterations"], st["converged"], st["keyframe_updated"]))
        outs.append(res)
        odo.close()
        reg.close()
    for a, b in zip(*outs):
        assert np.array_equal(a[0], b[0]) and a[1:] == b[1:]
    assert any(r[3] for r in outs[0][1:]) and all(r[2] for r in outs[0][1:])


# ---------------------------------------------------------------------------------------------------- 10, 11: map clouds
@pytest.fixture(scope="module")
def map_keyframes(synth):
    """250 keyframes of 16 384 points around the circuit (about 4.1 M points), empty keyframes first, in between and last"""
    empty = np.zeros((0, 8), np.float32)
    kfs = [(empty, synth.pose_matrix(0))]
    for f in range(250):
        c = synth.scan("vlp16_16k", frame=f, stride=8)
        if f % 50 == 7:
            c = decorate(c, seed=f)
        kfs.append((c, synth.pose_matrix(f) @ perturb(f, 0.05, 0.5)))
        if f % 61 == 3:
            kfs.append((empty, synth.pose_matrix(f)))
    kfs.append((empty, synth.pose_matrix(3)))
    return kfs


def test_map_cloud_at_map_scale_unfiltered(oracle, map_keyframes):
    reg = gicp()
    got = reg.mapCloudGenerate(map_keyframes, 0.0)
    reg.close()
    want = oracle.map_cloud_generate(map_keyframes, 0.0)
    assert got.shape[0] == want.shape[0] == sum(c.shape[0] for c, _ in map_keyframes) > 4000000
    assert np.array_equal(got[:, :3], want[:, :3], equal_nan=True)
    assert np.all(got[:, 3] == 1.0) and np.array_equal(got[:, 4], want[:, 4])


@pytest.mark.parametrize("res", [0.05, 0.25])
def test_map_cloud_at_map_scale_voxel_centres(oracle, map_keyframes, res):
    reg = gicp()
    got = reg.mapCloudGenerate(map_keyframes, res)
    reg.close()
    want = oracle.map_cloud_generate(map_keyframes, res)
    assert got.shape[0] == want.shape[0] > 0
    g = got[:, :3]
    g = g[np.lexsort((g[:, 0], g[:, 1], g[:, 2]))]
    assert np.array_equal(g, want)
    assert np.all(got[:, 3] == 1.0) and np.all(got[:, 4] == 0.0)


def test_map_too_deep_for_the_octree_keys_is_an_error(synth, oracle):
    """at 1 mm resolution two keyframes 3 km apart need more than 21 octree levels: an error, not an empty map"""
    c = synth.scan("vlp16_16k", frame=0, stride=8)[:200].copy()
    far = np.eye(4)
    far[0, 3] = 3000.0
    kfs = [(c, np.eye(4)), (c, far)]
    assert oracle.map_cloud_generate(kfs, 0.001).shape[0] > 0
    reg = gicp()
    with pytest.raises(pkg.B2RError) as e:
        reg.mapCloudGenerate(kfs, 0.001)
    assert e.value.code == _capi.B2R_EUNSUPPORTED and "21 octree levels" in str(e.value)
    # the handle stays usable, and a map that fits still comes out
    assert reg.mapCloudGenerate(kfs[:1], 0.001).shape[0] > 0
    reg.close()
