"""GPU: the pcl NDT pass (B2R_METHOD_NDT_PCL, csrc/ndt_pcl.cuh) on the inputs where it branches, rounds or indexes differently
from the scans of tests/test_ndt_pcl_gpu.py, against the sequential reference tests/ndt_pcl_ref.cpp:
- source sizes around the 128-point chunks, the 4096-point groups and the 32-row unrolled sum of the group rows, after a larger
  source has left non-zero rows in the handle's workspace;
- degenerate leaves: 5 / 6 / 7 points (a centroid iff >= 6, counted before invalidation), planes, lines, identical points, at
  the origin and far from it; an invalidated leaf stays searchable and adds exactly -d1 per point;
- the radius test at its boundary: queries at d2 == (float)(r*r) and one float32 ulp either side, at resolutions where
  (float)(r*r) rounds differently, exact d2 ties, centroids on bucket faces, queries beyond every face of the map (incl. a
  centroid that rounds into the padding ring of buckets);
- a map of more than 10^5 leaves; ndt_search_method (not read by this method); pass counts with the line search active;
- the batch on mixed sizes, degenerate pairs and co-scheduled pairs, bitwise equal to the single handle;
- the search's second and later selection rounds (more than 32 neighbours), which only a radius larger than the leaf reaches:
  tests/ndt_pcl_rounds_harness.cu launches the engine's neighbour kernel at such a radius on a map built through the ABI.

Tolerances: centroids, keys, neighbour lists and pair counts bit for bit; score / g / H rel <= 1e-9; poses <= 1e-4 with the same
iteration count and flag.  Cases marked (indep.) also check the neighbour lists against a numpy / scipy restatement that shares no
code with the reference: float32 centroids of the leaves of >= 6 points summed in index order, cKDTree candidates at a slightly
larger radius, the exact float32 filter ((dx*dx + dy*dy) + dz*dz) < np.float32(r*r), order (d2, leaf key)."""
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree

import hdl_graph_slam_b200 as pkg
from common import voxel_points, perturb, rot_err, trans_err
from ndt_pcl_ref import Reference, records, room, outside_cell_voxel
from test_ndt_edges_gpu import degenerate_cloud, NEAR_POSES, SHIFT
from test_ndt_pcl_oracle import np_centroids, np_leaf_keys, np_pose, np_transform, np_gauss

HERE = os.path.dirname(os.path.abspath(__file__))
F = np.float32
MAXR = 2.5
POSES = [np.zeros(6), np.array([0.1, -0.05, 0.02, 0.01, -0.02, 0.03]), np.array([-0.2, 0.1, 0.05, 0.05, 0.02, -0.04])]
K_PCL_NB = 32  # kPclNb: neighbours held per selection round


@pytest.fixture(scope="module")
def ref(oracle, tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("ndt_pcl_ref"))


def pcl_cfg(res=1.0, flag=0, fixed=0, max_iterations=64, search=7):
    c = pkg.default_config(pkg.B2R_METHOD_NDT_PCL)
    c.ndt_resolution = res
    c.ndt_mt_interval_flag = flag
    c.ndt_fixed_iterations = fixed
    c.max_iterations = max_iterations
    c.ndt_search_method = search
    return c


def handle(cfg, tgt, src=None):
    r = pkg.Registration(cfg)
    r.setInputTarget(tgt)
    if src is not None:
        r.setInputSource(src)
    return r


def rel(a, b):
    return np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(np.asarray(b))), 1e-300)


# ------------------------------------------------------------------------------------------------- independent restatement
def indep_neighbours(keys, cent, q, r):
    """per query the leaf keys of every centroid with float32 ((dx*dx + dy*dy) + dz*dz) < np.float32(r*r), d = q - c:
    (counts, keys in (query, d2, key) order, keys in (query, key) order, d2 in (query, d2, key) order)"""
    r2 = F(r * r)
    q = np.asarray(q, F).reshape(-1, 3)
    n = q.shape[0]
    ok = np.isfinite(q).all(axis=1)
    if len(cent) == 0 or not ok.any():
        z = np.zeros(0, np.int64)
        return np.zeros(n, np.int64), z, z, np.zeros(0, F)
    tree = cKDTree(np.asarray(cent, np.float64))
    cand = tree.query_ball_point(np.where(ok[:, None], q, 0).astype(np.float64), r * 1.001)  # a superset: d2 < r2 => |d| < r (1 + 3u)
    lens = np.array([len(c) if o else 0 for c, o in zip(cand, ok)], np.int64)
    qi = np.repeat(np.arange(n), lens)
    ci = np.fromiter((j for c, o in zip(cand, ok) if o for j in c), np.int64, int(lens.sum()))
    d = q[qi] - cent[ci]
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    keep = d2 < r2
    qi, ci, d2 = qi[keep], ci[keep], d2[keep]
    k = keys[ci]
    by_d2 = np.lexsort((k, d2, qi))
    by_key = np.lexsort((k, qi))
    return np.bincount(qi, minlength=n), k[by_d2], k[by_key], d2[by_d2]


def transformed(src, p):
    with np.errstate(invalid="ignore", over="ignore"):
        return np_transform(np_pose(np.asarray(p, np.float64)), src)


def check_neighbours(r, M, src, p, indep=False):
    """the engine's radius neighbours of every source point at p == the reference's, bit for bit (and == numpy when indep)"""
    cnt, keys = r.ndtNeighborsAt(p, src.shape[0])
    rcnt, rkeys = M.neighbors(src, p)
    assert np.array_equal(cnt, rcnt), f"counts at {p}: {int(np.sum(cnt != rcnt))} differ"
    assert np.array_equal(keys, rkeys), f"neighbour keys at {p}"
    if indep:
        ck, cc = np_centroids(M.tgt, M.resolution)
        icnt, _, ikeys, _ = indep_neighbours(ck, cc, transformed(src, p), M.resolution)
        assert np.array_equal(cnt, icnt), f"counts at {p} differ from numpy: {int(np.sum(cnt != icnt))}"
        assert np.array_equal(keys, ikeys), f"neighbour keys at {p} differ from numpy"
    return cnt, keys


def check_passes(r, M, src, p, min_pairs=0):
    """derivative pass and Hessian-only pass == the reference (rel 1e-9, pair count exact), and bitwise repeatable"""
    s, g, H, npairs = r.ndtDerivativesAt(p)
    o = M.derivatives(src, p)
    assert npairs == o["n_pairs"] and npairs >= min_pairs, (npairs, o["n_pairs"])
    if npairs:
        assert abs(s - o["score"]) <= 1e-9 * abs(o["score"])
        assert rel(g, o["g"]) <= 1e-9 and rel(H, o["H"]) <= 1e-9
    else:
        assert s == 0.0 and not g.any() and not H.any()
    assert np.array_equal(r.ndtHessianAt(p), H)  # computeHessian's term is updateDerivatives' Hessian term
    again = r.ndtDerivativesAt(p)
    assert again[0] == s and np.array_equal(again[1], g) and np.array_equal(again[2], H) and again[3] == npairs
    return s, g, H, npairs


def check_centroids(r, M, indep=True):
    k, c = r.ndtGetCentroids()
    rk, rc = M.centroids()
    assert np.array_equal(k, rk) and np.array_equal(c.view(np.uint32), rc.view(np.uint32))
    if indep:
        nk, nc = np_centroids(M.tgt, M.resolution)
        assert np.array_equal(k, nk) and np.array_equal(c.view(np.uint32), nc.view(np.uint32))
    return k, c


# ------------------------------------------------------------------------------------------------------------ source sizes
@pytest.fixture(scope="module")
def vlp_map(ref, synth):
    tgt = synth.scan("vlp16", frame=0, stride=8)
    return tgt, ref.map(tgt, 1.0)


@pytest.fixture(scope="module")
def big_source(synth):
    return np.concatenate([synth.scan("vlp16", frame=f, stride=8) for f in (1, 2, 3, 4)])


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 127, 128, 129, 4095, 4096, 4097, 131073, 200000])
def test_source_sizes(vlp_map, big_source, n):
    """one point, a chunk -1 / +0 / +1, a group -1 / +0 / +1, 33 groups (one full round of the unrolled 32-row sum of the group
    rows plus a remainder of one) and 49 groups (remainder 17).

    The handle first runs a 200 000-point source (1568 chunks) of points within a few centimetres of the map's centroids, so every
    one of its chunk rows holds a non-zero score: the rows of a group that a later, smaller source does not own (24 of 32 at 1 -
    129, 4097 and 131 073 points) hold values, and a group sum that read them would be wrong.  (A scan would not do: the
    Hilbert-sorted scan's first 4096 points may lie where the map has no leaf, and their rows are then zero, like fresh ones.)"""
    tgt, M = vlp_map
    src = big_source[np.random.default_rng(n).permutation(big_source.shape[0])[:n]].copy() if n < 4096 else big_source[:n].copy()
    r = handle(pcl_cfg(1.0), tgt)
    _, cent = r.ndtGetCentroids()
    rng = np.random.default_rng(17)
    prime = np.repeat(cent, -(-200000 // cent.shape[0]), axis=0)[:200000].astype(np.float64)
    r.setInputSource(records(prime + rng.normal(0.0, 0.05, prime.shape)))
    assert r.ndtDerivativesAt(np.zeros(6))[3] >= 200000  # every point has a neighbour: every chunk row is non-zero
    r.setInputSource(src)
    for p in POSES[1:]:
        check_passes(r, M, src, p, min_pairs=1 if n < 4096 else n // 2)
    r.close()


# -------------------------------------------------------------------------------------------------------- degenerate leaves
@pytest.mark.gpu
@pytest.mark.parametrize("res", [1.0, 0.5])
@pytest.mark.parametrize("shifted", [False, True])
def test_degenerate_leaves(ref, res, shifted):
    """(indep.) every VOXEL_KIND with 5, 6 and 7 points: a centroid exactly for the leaves of >= 6 points, invalidated leaves
    included; neighbour lists, derivative and Hessian passes at the poses the NDT_OMP test uses"""
    off = SHIFT if shifted else (0.0, 0.0, 0.0)
    tgt = degenerate_cloud(res, off, seed=1)
    M = ref.map(tgt, res)
    r = handle(pcl_cfg(res), tgt)
    k, c = check_centroids(r, M)
    _, lk = np_leaf_keys(tgt, res)
    ks, cnt = np.unique(lk, return_counts=True)
    assert np.array_equal(k, ks[cnt >= 6])  # presence decided by the count alone: 5 -> none, 6 and 7 -> a centroid
    for m in (5, 6, 7):
        assert np.sum(cnt == m) >= 10, m
    invalid = M.voxels["keys"][M.voxels["npts"] == -1]
    assert invalid.size >= 10 and np.isin(invalid, k).all()  # invalidated after counting: still emitted
    rng = np.random.default_rng(2)
    src = np.repeat(tgt, 3, axis=0).copy()
    src[:, :3] += rng.normal(0.0, 0.3 * res, (src.shape[0], 3)).astype(F)
    src = np.concatenate([src, records(c)])  # a query exactly at every centroid: every emitted leaf, invalidated ones too, is found
    r.setInputSource(src)
    poses = [np.r_[np.asarray(p[:3]) * res, p[3:]] for p in (NEAR_POSES if shifted else POSES)]
    for p in poses:
        check_neighbours(r, M, src, p, indep=True)
        check_passes(r, M, src, p, min_pairs=100)
    _, keys = r.ndtNeighborsAt(np.zeros(6), src.shape[0])
    assert np.isin(invalid, keys).all()
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("res", [1.0, 0.5])
@pytest.mark.parametrize("shifted", [False, True])
def test_invalidated_leaf_adds_minus_d1_per_point(ref, res, shifted):
    """leaves of 6, 7 and 9 identical points (zero covariance: invalidated, zero inverse) three cells apart, and queries within r
    of exactly one of them: every pair adds -d1 to the score and nothing to g or H"""
    off = SHIFT if shifted else (0.0, 0.0, 0.0)
    rng = np.random.default_rng(3)
    cells = [(3 * i, 3 * j, 3 * (i + j) % 2) for i in range(-3, 4) for j in range(-3, 4)]
    tgt = np.concatenate([voxel_points("identical", (6, 7, 9)[t % 3], cl, res, rng, off) for t, cl in enumerate(cells)])
    M = ref.map(tgt, res)
    assert (M.voxels["npts"] == -1).all() and not M.voxels["icov"].any()
    r = handle(pcl_cfg(res), tgt)
    k, c = check_centroids(r, M)
    assert k.size == len(cells)
    q = np.repeat(c, 20, axis=0).astype(np.float64) + rng.uniform(-0.5 * res, 0.5 * res, (20 * len(cells), 3))  # |d| < 0.87 r
    src = records(q)
    r.setInputSource(src)
    cnt, _ = check_neighbours(r, M, src, np.zeros(6), indep=True)
    assert (cnt == 1).all()
    s, g, H, npairs = check_passes(r, M, src, np.zeros(6))
    d1, _ = np_gauss(res)
    assert npairs == src.shape[0] and abs(s - (-d1 * npairs)) <= 1e-12 * abs(d1 * npairs)
    assert not g.any() and not H.any()
    r.close()


# ----------------------------------------------------------------------------------------------------------- radius boundary
RESOLUTIONS = [0.1, 0.3, 0.5, 0.7, 1.0, 1.1, 2.0, 5.0]


def dy(x):
    """x rounded to a multiple of 2^-10: small sums of such values are exact in float32"""
    return np.round(np.asarray(x, np.float64) * 1024.0) / 1024.0


def sym_leaf(c, a):
    """6 points c -+ a along each axis: a valid leaf whose float32 centroid is exactly c (c, a multiples of 2^-10)"""
    c = np.asarray(c, np.float64)
    pts = [c + s * a * np.eye(3)[d] for d in range(3) for s in (1.0, -1.0)]
    return records(pts)


def boundary_queries(c, r, axis, sign, lateral):
    """three float32 queries moving from centroid c along `axis` (direction `sign`), the other two coordinates offset by
    `lateral`: the last one inside the radius, the first one not (at d2 == r2 when such a float32 exists), and the next one out.
    Returns (queries, d2 == r2 exactly at the middle one)."""
    r2 = F(r * r)
    c = np.asarray(c, F)
    base = c.copy()
    o = [d for d in range(3) if d != axis]
    base[o[0]] = F(c[o[0]] + F(lateral[0]))
    base[o[1]] = F(c[o[1]] + F(lateral[1]))

    def d2(x):
        q = base.copy()
        q[axis] = x
        d = q - c
        return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
    away, toward = F(sign * np.inf), c[axis]
    lat2 = float(base[o[0]] - c[o[0]]) ** 2 + float(base[o[1]] - c[o[1]]) ** 2
    x = F(float(c[axis]) + sign * np.sqrt(r * r - lat2))  # within a few ulps of the boundary
    while d2(x) < r2:
        x = np.nextafter(x, away)
    while d2(np.nextafter(x, toward)) >= r2:
        x = np.nextafter(x, toward)
    qs = []
    for v in (np.nextafter(x, toward), x, np.nextafter(x, away)):
        q = base.copy()
        q[axis] = v
        qs.append(q)
    return np.array(qs, F), bool(d2(x) == r2)


def test_resolutions_cover_both_roundings_of_r2():
    """(float)(r*r) of the float64 radius, as KdTreeFLANN receives it, differs from the float32 square of (float)r at some of
    RESOLUTIONS and equals it at others: a kernel squaring the float32 radius fails test_radius_boundary"""
    diff = [F(r * r) != F(F(r) * F(r)) for r in RESOLUTIONS]
    assert any(diff) and not all(diff)


@pytest.mark.gpu
@pytest.mark.parametrize("res", RESOLUTIONS)
def test_radius_boundary(ref, res):
    """(indep.) clusters of six valid leaves at -+ s (s < r) along each axis around an empty cell, centroids exactly on
    multiples of 2^-10: the cluster's centre has six neighbours at one d2 (a tie broken by leaf); from every centroid, queries
    one ulp inside the radius, at it and one ulp outside, along each axis and three skew directions"""
    s, a = dy(0.75 * res), dy(res / 8)
    centres = [dy((np.array(cl) + 0.5) * res) for cl in ((0, 0, 0), (-5, 3, 2), (7, -4, -3), (12, 9, -8))]
    anchors = [q + sg * s * np.eye(3)[d] for q in centres for d in range(3) for sg in (1.0, -1.0)]
    tgt = np.concatenate([sym_leaf(x, a) for x in anchors])
    M = ref.map(tgt, res)
    r = handle(pcl_cfg(res), tgt)
    k, c = check_centroids(r, M)
    assert k.size == len(anchors) and np.array_equal(np.sort(c.view(np.uint32), axis=0), np.sort(np.array(anchors, F).view(np.uint32), axis=0))
    qs, want, exact = [np.array(centres, F)], [], 0
    for ci, cc in enumerate(c):
        for axis in range(3):
            for sign in (1.0, -1.0):
                for lat in ((0.0, 0.0), (0.25 * res, 0.5 * res), (-0.6 * res, 0.1 * res), (0.3 * res, -0.3 * res)):
                    b, ex = boundary_queries(cc, res, axis, sign, lat)
                    qs.append(b)
                    want.append((k[ci], [True, False, False]))
                    exact += ex
    src = records(np.concatenate(qs))
    r.setInputSource(src)
    cnt, keys = check_neighbours(r, M, src, np.zeros(6), indep=True)
    assert (cnt[:len(centres)] == 6).all()  # the six tied leaves around every centre
    off = np.r_[0, np.cumsum(cnt)]
    for t, (key, inside) in enumerate(want):
        for j in range(3):
            i = len(centres) + 3 * t + j
            assert (key in keys[off[i]:off[i + 1]]) == inside[j], (t, j)
    assert exact >= 1, "no query sits at d2 == r2 exactly"
    check_passes(r, M, src, np.zeros(6), min_pairs=len(want))
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("res", [0.1, 0.5, 0.7, 1.0])
def test_lattice_planes(ref, res):
    """(indep.) leaves whose points all lie on one lattice plane x = k res (float32), so their centroids lie on a bucket face or
    an ulp from it, in a map of random fill; queries on the lattice points"""
    r32 = F(res)
    xs = np.float32(np.arange(-10, 11, dtype=F) * r32)
    ys = np.float32(np.arange(-3, 4, dtype=F) * r32)
    g = np.stack(np.meshgrid(xs, ys, ys, indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    e = res / 8
    offs = np.array([[0, 0, 0], [0, e, 0], [0, -e, 0], [0, 0, e], [0, 0, -e], [0, e, e], [0, -e, -e]])
    leaves = (g[:, None, :] + offs[None, :, :]).reshape(-1, 3)
    rng = np.random.default_rng(8)
    fill = np.repeat(g, 3, axis=0) + rng.uniform(-1.5 * res, 1.5 * res, (3 * g.shape[0], 3)) + [0, 0, 9 * res]  # above the block
    tgt = records(np.r_[leaves, fill])
    M = ref.map(tgt, res)
    r = handle(pcl_cfg(res), tgt)
    k, c = check_centroids(r, M)
    on_face = np.isin(c[:, 0], xs)
    assert on_face.sum() >= 50
    src = records(np.r_[g, g + [res / 2, 0, 0]])
    r.setInputSource(src)
    for p in POSES[:2]:
        check_neighbours(r, M, src, p, indep=True)
        check_passes(r, M, src, p, min_pairs=200)
    r.close()


def edge_scene(leaf=0.1, seed=0):
    """a blob of random points below x, y, z = (k - 1) leaf, and on each axis a leaf at the top of cell k - 1 whose float32
    centroid rounds into cell k: the padding ring of buckets beyond the map's last cell holds a centroid on three faces"""
    x, n, k = outside_cell_voxel(leaf)
    rng = np.random.default_rng(seed)
    hi = (k - 1) * leaf - 0.05 * leaf
    blob = rng.uniform(-0.5, hi, (6000, 3))
    parts = [blob]
    for axis in range(3):
        p = rng.uniform(0.01, 0.09, (n, 3))
        p[:, axis] = x
        parts.append(p.astype(F).astype(np.float64))
        parts[-1][:, axis] = x
    return records(np.concatenate(parts)), (x, n, k)


@pytest.mark.gpu
def test_queries_beyond_every_face(ref):
    """(indep.) from the outermost centroids of each of the six faces, queries straight out and skew at 0.5 ... 100 r: just
    inside and just beyond r of an edge centroid, and far out where every bucket coordinate clamps onto the outer ring"""
    leaf = 0.1
    tgt, (x, n, kk) = edge_scene(leaf)
    M = ref.map(tgt, leaf)
    r = handle(pcl_cfg(leaf), tgt)
    k, c = check_centroids(r, M)
    inv = F(1) / F(leaf)
    assert all((np.floor(c[:, a] * inv) == kk).any() for a in range(3))  # a centroid in the padding ring on each max face
    qs = []
    for axis in range(3):
        for sign in (1.0, -1.0):
            order = np.argsort(sign * c[:, axis])[::-1][:6]  # the outermost centroids on this face
            for j, ci in enumerate(order):
                for t in (0.3, 0.5, 0.9, 0.999, 0.9999, 1.0, 1.0001, 1.001, 1.2, 1.5, 2.5, 100.0):
                    q = c[ci].astype(np.float64)
                    q[axis] += sign * t * leaf
                    qs.append(q)
                    lat = q.copy()
                    lat[(axis + 1) % 3] += 0.3 * leaf * (1 - 2 * (j % 2))
                    qs.append(lat)
                b, _ = boundary_queries(c[ci], leaf, axis, sign, (0.0, 0.0))
                qs.extend(b.astype(np.float64))
    far = np.array([[1e6, 0, 0], [-1e6, 0, 0], [0, 3e7, 0], [0, 0, -3e7], [1e30, 1e30, 1e30], [-3e38, 0.05, 0.05]])
    src = records(np.r_[np.array(qs), far])
    r.setInputSource(src)
    cnt, _ = check_neighbours(r, M, src, np.zeros(6), indep=True)
    assert cnt.sum() > len(qs) // 4 and not cnt[-len(far):].any()
    check_passes(r, M, src, np.zeros(6), min_pairs=100)
    r.close()


# ---------------------------------------------------------------------------------------------------------------- large map
@pytest.mark.gpu
def test_large_map(ref):
    """(indep.) 1.2 M points at 0.2 m: more than 10^5 leaves with a centroid and bucket keys spread over a 360 x 360-cell floor
    and two walls; the neighbour lists of 100 000 query points at two poses, and both passes.  (The bucket table has at least
    twice as many slots as the map has points and a bucket needs 6 points, so it is never more than 1/12 full: this case is
    about the size of the map, not about long probe chains.)"""
    rng = np.random.default_rng(11)
    nf, nw = 1_100_000, 50_000
    floor = np.c_[rng.uniform(-36, 36, (nf, 2)), rng.uniform(0.05, 0.15, nf)]
    walls = [np.c_[rng.uniform(-36, 36, nw), np.full(nw, 30.1) + rng.normal(0, 0.02, nw), rng.uniform(0, 6, nw)],
             np.c_[np.full(nw, -30.1) + rng.normal(0, 0.02, nw), rng.uniform(-36, 36, nw), rng.uniform(0, 6, nw)]]
    tgt = records(np.concatenate([floor] + walls))
    res = 0.2
    M = ref.map(tgt, res)
    r = handle(pcl_cfg(res), tgt)
    k, _ = check_centroids(r, M)
    assert k.size >= 100_000, k.size
    src = tgt[rng.choice(tgt.shape[0], 100_000, replace=False)].copy()
    src[:, :3] += rng.normal(0, 0.1, (src.shape[0], 3)).astype(F)
    r.setInputSource(src)
    for p in POSES[:2]:
        cnt, _ = check_neighbours(r, M, src, p, indep=True)
        assert cnt.sum() > 30_000 and cnt.max() < K_PCL_NB
        check_passes(r, M, src, p, min_pairs=30_000)
    r.close()


# ------------------------------------------------------------------------------------------------------ ndt_search_method
@pytest.mark.gpu
def test_search_method_changes_nothing(synth):
    """pcl::NormalDistributionsTransform has no search-method choice: DIRECT1 / DIRECT7 / KDTREE (through the factory, which
    accepts it for this branch) give bitwise the same neighbours, passes and aligns"""
    tgt, src = synth.scan("vlp16_16k", frame=0, stride=8), synth.scan("vlp16_16k", frame=1, stride=8)
    G = perturb(3, 0.2, 1.0).astype(np.float32)

    def outputs(r):
        o = []
        for p in POSES[1:]:
            o += list(r.ndtNeighborsAt(p, src.shape[0]))
            s, g, H, npairs = r.ndtDerivativesAt(p)
            o += [np.array([s, npairs]), g, H, r.ndtHessianAt(p)]
        for guess in (np.eye(4, dtype=np.float32), G):
            r.align(guess)
            o += [r.getFinalTransformation(), np.array([r.nr_iterations, r.hasConverged()]), np.array([r.getFitnessScore(MAXR)])]
        return [np.asarray(x).tobytes() for x in o]
    want = None
    for make in [lambda: pkg.Registration(pcl_cfg(1.0, search=7)), lambda: pkg.Registration(pcl_cfg(1.0, search=1)),
                 lambda: pkg.Registration(pcl_cfg(1.0, search=0)),
                 lambda: pkg.select_registration_method({"registration_method": "NDT", "reg_resolution": 1.0, "reg_nn_search_method": "KDTREE"}),
                 lambda: pkg.select_registration_method({"registration_method": "NDT", "reg_resolution": 1.0, "reg_nn_search_method": "DIRECT1"})]:
        r = make()
        r.setInputTarget(tgt)
        r.setInputSource(src)
        got = outputs(r)
        r.close()
        if want is None:
            want = got
        assert got == want


# ------------------------------------------------------------------------------------------------------------- line search
@pytest.mark.gpu
def test_line_search_runs_the_hessian_pass(ref, synth):
    """mt_interval_flag = 1 with a guess for which the reference's line search iterates: the engine launches the Hessian-only
    pass as often as the reference runs computeHessian, and the derivative pass as often as its other passes"""
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)
    src = synth.scan("vlp16_16k", frame=1, stride=8)
    M = ref.map(tgt, 1.0)
    for seed in range(20, 60):
        G = perturb(seed, 0.5, 3.0).astype(np.float32)
        o = M.align(src, G, mt_interval_flag=1)
        if o["hessian_passes"] >= 1:
            break
    assert o["hessian_passes"] >= 1, "no guess made the reference's line search iterate"
    r = handle(pcl_cfg(1.0, flag=1), tgt, src)
    r.ndtGetCentroids()  # the map build is not part of the counted launches
    r.getStats(reset=True)
    r.align(G)
    launches = r.getStats()["launches"]
    assert launches["ndt_hessian"] == o["hessian_passes"]
    assert launches["ndt_derivatives"] == o["derivative_passes"] - o["hessian_passes"]
    assert r.nr_iterations == o["iterations"] and r.hasConverged() == o["converged"]
    T = r.getFinalTransformation()
    assert trans_err(T, o["T"]) < 1e-4 and rot_err(T, o["T"]) < 1e-4
    r.close()


# ------------------------------------------------------------------------------------------------------------------- batch
def run_batch(cfg, clouds, pairs, want_fitness=True):
    lb = pkg.RegistrationBatch(cfg=cfg)
    ids = {k: lb.addCloud(c) for k, c in clouds.items()}
    res = lb.align([(ids[s], ids[t], g) for s, t, g in pairs], want_fitness, MAXR)
    lb.close()
    return res


def run_single(cfg, clouds, pairs):
    r = pkg.Registration(cfg)
    out = []
    for s, t, g in pairs:
        r.setInputTarget(clouds[t])
        r.setInputSource(clouds[s])
        r.align(g)
        out.append({"T": r.getFinalTransformation(), "converged": r.hasConverged(), "iterations": r.nr_iterations,
                    "fitness": r.getFitnessScore(MAXR)})
    r.close()
    return out


def same(a, b, fitness=True):
    ok = np.array_equal(np.asarray(a["T"]).view(np.uint32), np.asarray(b["T"]).view(np.uint32))
    ok = ok and bool(a["converged"]) == bool(b["converged"]) and a["iterations"] == b["iterations"]
    if fitness:
        ok = ok and np.float64(a["fitness"]).tobytes() == np.float64(b["fitness"]).tobytes()
    return ok


@pytest.mark.gpu
def test_batch_mixed_sizes(synth):
    """sources of 1, 129, 4097, 16 384, 65 536 and 131 073 points against two targets, a source that is its target, and an
    iteration cap some pairs stop at while others converge: every pair == the single handle, bitwise, for both polarities"""
    big = synth.scan("hdl32e", frame=41, stride=8)
    clouds = {"t0": synth.scan("vlp16_16k", frame=0, stride=8), "t1": synth.scan("hdl32e", frame=40, stride=8),
              "n1": big[5000:5001].copy(), "n129": big[::1000][:129].copy(), "n4097": big[:4097].copy(),
              "n16k": synth.scan("vlp16_16k", frame=1, stride=8), "n64k": synth.scan("vlp16", frame=2, stride=8), "n131073": np.r_[big, big[:1]]}
    frame = {"t0": 0, "t1": 40, "n1": 41, "n129": 41, "n4097": 41, "n16k": 1, "n64k": 2, "n131073": 41}
    pairs = []
    for j, (s, t) in enumerate([("n1", "t1"), ("n129", "t1"), ("n4097", "t1"), ("n16k", "t0"), ("n64k", "t0"), ("n131073", "t1"),
                                ("t0", "t0"), ("n4097", "t0"), ("n131073", "t0")]):
        rel_ = np.linalg.inv(synth.pose_matrix(frame[t])) @ synth.pose_matrix(frame[s])
        pairs.append((s, t, (rel_ @ perturb(90 + j, 0.3, 2.0)).astype(np.float32) if s != t else np.eye(4, dtype=np.float32)))
    for flag in (0, 1):
        cfg = pcl_cfg(1.0, flag, max_iterations=4)
        got = run_batch(cfg, clouds, pairs)
        want = run_single(cfg, clouds, pairs)
        for i, (a, b) in enumerate(zip(got, want)):
            assert same(a, b), f"flag {flag} pair {i}"
        its = [q["iterations"] for q in got]
        assert min(its) < max(its)


@pytest.mark.gpu
def test_batch_degenerate_pairs(synth):
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)
    src = synth.scan("vlp16_16k", frame=1, stride=8)
    nan_src = src.copy()
    nan_src[::7, :3] = np.nan
    nan_src[3::11, 1] = np.inf
    nan_src[5::13, 2] = -1e12
    clouds = {"t": tgt, "s": src, "nan": nan_src, "sparse": tgt[:5].copy(), "allnan": np.full((64, 8), np.nan, np.float32),
              "empty": np.zeros((0, 8), np.float32), "one": src[100:101].copy()}
    G = perturb(5, 0.2, 1.0).astype(np.float32)
    pairs = [("s", "t", G), ("empty", "t", G), ("s", "empty", G), ("s", "sparse", G), ("s", "allnan", G), ("nan", "t", G),
             ("one", "t", G), ("s", "t", np.eye(4, dtype=np.float32))]
    cfg = pcl_cfg(1.0)
    got = run_batch(cfg, clouds, pairs)
    want = run_single(cfg, clouds, pairs)
    for i, (a, b) in enumerate(zip(got, want)):
        assert same(a, b), f"pair {i}"
    assert got[1]["fitness"] == np.finfo(np.float64).max and not got[1]["converged"]


@pytest.mark.gpu
def test_batch_co_scheduled_pairs_do_not_matter(synth):
    clouds, pairs = {}, []
    for gi, tf in enumerate(range(0, 60, 10)):
        clouds.setdefault(tf, synth.scan("vlp16_16k", frame=tf, stride=8))
        for j, off in enumerate((1, 2, 3, 251, 252, 253, 4, 254)):
            sf = tf + off
            clouds.setdefault(sf, synth.scan("vlp16_16k", frame=sf, stride=8))
            g = (np.linalg.inv(synth.pose_matrix(tf)) @ synth.pose_matrix(sf) @ perturb(60 + 7 * gi + j, 0.3, 2.0)).astype(np.float32)
            g[2, 3] = 0.0
            pairs.append((sf, tf, g))
    cfg = pcl_cfg(1.0)
    lb = pkg.RegistrationBatch(cfg=cfg)
    ids = {k: lb.addCloud(c) for k, c in clouds.items()}
    pl = [(ids[s], ids[t], g) for s, t, g in pairs]
    full = lb.align(pl, True, MAXR)
    again = lb.align(pl, True, MAXR)
    rev = lb.align(pl[::-1], True, MAXR)[::-1]
    for i in range(len(pl)):
        assert same(full[i], again[i]) and same(full[i], rev[i]), f"pair {i}"
    for i in (0, 21, len(pl) - 1):
        assert same(lb.align([pl[i]], True, MAXR)[0], full[i])
    lb.close()
    pick = (0, 20, len(pairs) - 1)
    for i, w in zip(pick, run_single(cfg, clouds, [pairs[i] for i in pick])):
        assert same(full[i], w)


# ----------------------------------------------------------------------------------------------- selection rounds (> 32)
def test_abi_neighbour_count_stays_below_one_round_of_selection():
    """Documents why the search's second round is unreachable through the ABI: the radius equals the leaf, so an open ball of
    radius r meets at most 27 cells (3 per axis), each holding one centroid.  27 centroids placed 0.515625 r per axis from a
    query all qualify; the (indep.) restatement is enough here, the GPU counterpart is in test_abi_neighbour_count_gpu."""
    tgt, q = twenty_seven()
    keys, cent = np_centroids(tgt, 1.0)
    cnt, _, _, _ = indep_neighbours(keys, cent, q, 1.0)
    assert cnt.tolist() == [27] and 27 < K_PCL_NB


def twenty_seven():
    cs = (-1.0 / 64, 0.5, 1.0 + 1.0 / 64)
    tgt = np.concatenate([sym_leaf((x, y, z), 1.0 / 128) for x in cs for y in cs for z in cs])
    return tgt, np.array([[0.5, 0.5, 0.5]], F)


@pytest.mark.gpu
def test_abi_neighbour_count_gpu(ref, synth):
    """the largest neighbour count the product reaches: 27 (the bound above), in a constructed map and never more in a dense room
    at two resolutions, a degenerate map and a scan; all of them below kPclNb = 32, so the pass never runs a second round"""
    tgt, q = twenty_seven()
    r = handle(pcl_cfg(1.0), tgt, records(q))
    cnt, _ = check_neighbours(r, ref.map(tgt, 1.0), records(q), np.zeros(6), indep=True)
    r.close()
    most = int(cnt.max())
    assert most == 27
    for t, s, res in ((room(200000, 5), room(50000, 6), 0.5), (room(200000, 5), room(50000, 6), 0.2),
                      (degenerate_cloud(0.5, seed=1), degenerate_cloud(0.5, seed=4), 0.5),
                      (synth.scan("hdl32e", frame=0, stride=8), synth.scan("hdl32e", frame=1, stride=8), 1.0)):
        r = handle(pcl_cfg(res), t, s)
        for p in POSES:
            c, _ = r.ndtNeighborsAt(p, s.shape[0])
            most = max(most, int(c.max()))
        r.close()
    assert most == 27 < K_PCL_NB


@pytest.fixture(scope="module")
def rounds_harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("rounds") / "ndt_pcl_rounds_harness")
    subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-w", "--compiler-options=-ffp-contract=off",
                           "-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-o", exe,
                           os.path.join(HERE, "ndt_pcl_rounds_harness.cu"), "-lnccl"])
    return exe


def test_rounds_harness_compiles(rounds_harness):
    assert os.path.exists(rounds_harness)


def lattice_scene():
    """a 12^3 block of valid leaves at res 1 whose centroids are exactly the cell centres: queries at cell centres have their
    neighbours in shells of equal d2 (1 at 0, 6 at 1, 12 at 2, 8 at 3, 6 at 4, 24 at 5, 24 at 6, 12 at 8, ...): at radius 2.5 the
    shell d2 = 4 holds positions 28 ... 33, a tie across the 32nd / 33rd neighbour"""
    cells = np.stack(np.meshgrid(*[np.arange(-6, 6)] * 3, indexing="ij"), -1).reshape(-1, 3)
    tgt = np.concatenate([sym_leaf(cl + 0.5, 0.125) for cl in cells])
    inner = cells[(np.abs(cells + 0.5) < 4).all(axis=1)] + 0.5
    rng = np.random.default_rng(12)
    q = np.r_[inner, inner[::5] + 0.5, rng.uniform(-7.5, 7.5, (1500, 3)), dy(rng.uniform(-6, 6, (500, 3)))]
    return tgt, q.astype(F)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["lattice_2.5", "lattice_3", "random_2.5", "random_3"])
def test_selection_rounds(rounds_harness, tmp_path, case):
    """(indep.) radius 2.5 or 3 leaves: 40 - 200 neighbours per query, taken in up to seven rounds of 32; every list, in the
    kernel's (d2, leaf) order, == numpy brute force bit for bit"""
    kind, leaves = case.split("_")
    if kind == "lattice":
        tgt, q = lattice_scene()
        res = 1.0
    else:  # 200 000 random points in a 10 m cube at 0.5 m: about 25 per leaf, every leaf with a centroid somewhere inside it
        rng = np.random.default_rng(13)
        tgt = records(rng.uniform(-5, 5, (200000, 3)))
        q = rng.uniform(-6, 6, (3000, 3)).astype(F)
        res = 0.5
    radius = float(leaves) * res
    tf, qf, out = tmp_path / "t.f32", tmp_path / "q.f32", tmp_path / "out.bin"
    np.ascontiguousarray(tgt[:, :4], F).tofile(tf)
    np.ascontiguousarray(q, F).tofile(qf)
    p = subprocess.run([rounds_harness, str(tf), str(qf), repr(res), repr(radius), str(out)], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    stats = dict(kv.split("=") for kv in p.stdout.split())
    raw = np.fromfile(out, np.uint8)
    m = q.shape[0]
    cnt = raw[:4 * m].view(np.uint32)
    keys = raw[4 * m:].view(np.int64)
    ck, cc = np_centroids(tgt, res)
    icnt, ikeys, _, id2 = indep_neighbours(ck, cc, q, radius)
    assert np.array_equal(cnt, icnt), f"{int(np.sum(cnt != icnt))} counts differ"
    assert np.array_equal(keys, ikeys)
    assert int(stats["max_count"]) == cnt.max() and int(stats["rounds"]) == int(np.sum(cnt > K_PCL_NB)) > m // 4
    assert 40 <= cnt.max() <= 200
    off = np.r_[0, np.cumsum(icnt)]
    ties = [i for i in range(m) if icnt[i] > K_PCL_NB and id2[off[i] + K_PCL_NB - 1] == id2[off[i] + K_PCL_NB]]
    if kind == "lattice":
        assert len(ties) >= 100  # equal d2 at the 32nd and 33rd neighbour: the next round starts inside a tie
        assert cnt.max() > 2 * K_PCL_NB  # three rounds or more
