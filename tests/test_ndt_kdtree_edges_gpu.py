"""GPU: NDT_OMP's KDTREE search (B2R_METHOD_NDT_KDTREE) on the inputs where it branches, rounds or indexes differently from scans,
against the sequential reference tests/ndt_kdtree_ref.cpp:
- empty and tiny clouds;
- the radius test at d2 == (float)(r*r) and one float32 ulp either side;
- queries beyond every face of the map, and source points beyond 1e9 cells (no cell index is formed, so they are not dropped: they
  simply have no neighbour);
- zero-inverse and non-finite-inverse leaves (no nr_points check: they take part with the inverse they hold), degenerate leaves of
  5 / 6 / 7 points, lattice-plane leaves;
- non-finite source points;
- sources of 1 ... 200 000 points, across the 128-point chunks and the 4096-point groups.

Tolerances: centroids, keys, neighbour lists and pair counts bit for bit; score / g / H of both passes rel <= 1e-9.  Cases marked
(indep.) also check neighbour lists against test_ndt_pcl_edges_gpu's numpy / scipy restatement."""
import numpy as np
import pytest

import hdl_graph_slam_b200 as pkg
from common import voxel_points
from ndt_kdtree_ref import Reference
from ndt_pcl_ref import records
from test_ndt_edges_gpu import degenerate_cloud, NEAR_POSES, SHIFT
from test_ndt_pcl_edges_gpu import boundary_queries, check_centroids, check_neighbours, dy, edge_scene, sym_leaf
from test_ndt_pcl_oracle import np_gauss, np_leaf_keys

pytestmark = pytest.mark.gpu
F = np.float32
POSES = [np.zeros(6), np.array([0.1, -0.05, 0.02, 0.01, -0.02, 0.03]), np.array([-0.2, 0.1, 0.05, 0.05, 0.02, -0.04])]


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("ndt_kdtree_ref"))


def kd_cfg(res=1.0, flag=0):
    c = pkg.default_config(pkg.B2R_METHOD_NDT_KDTREE)
    c.ndt_resolution = res
    c.ndt_mt_interval_flag = flag
    return c


def handle(cfg, tgt, src=None):
    r = pkg.Registration(cfg)
    r.setInputTarget(tgt)
    if src is not None:
        r.setInputSource(src)
    return r


def rel(a, b):
    return np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(np.asarray(b))), 1e-300)


def check_passes(r, M, src, p, min_pairs=0):
    """derivative pass and Hessian-only pass == the reference (rel 1e-9, pair count exact), and bitwise repeatable"""
    s, g, H, npairs = r.ndtDerivativesAt(p)
    o = M.derivatives(src, p)
    assert npairs == o["n_pairs"] and npairs >= min_pairs, (npairs, o["n_pairs"])
    Hh = r.ndtHessianAt(p)
    Hr = M.hessian_at(src, p)
    if npairs:
        if o["score"] != 0.0:
            assert abs(s - o["score"]) <= 1e-9 * abs(o["score"])
        assert rel(g, o["g"]) <= 1e-9 if o["g"].any() else not g.any()
        assert rel(H, o["H"]) <= 1e-9 if o["H"].any() else not H.any()
        assert rel(Hh, Hr) <= 1e-9 if Hr.any() else not Hh.any()
    else:
        assert s == 0.0 and not g.any() and not H.any() and not Hh.any()
    again = r.ndtDerivativesAt(p)
    assert again[0] == s and np.array_equal(again[1], g) and np.array_equal(again[2], H) and again[3] == npairs
    return s, g, H, npairs


def test_empty_and_tiny_clouds(ref, synth):
    src = synth.scan("vlp16_16k", frame=1, stride=8)
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)
    for name, t in {"empty": np.zeros((0, 8), F), "all_nan": np.full((64, 8), np.nan, F), "five": tgt[:5].copy()}.items():
        r = pkg.Registration(kd_cfg(1.0))
        r.setInputSource(src)
        r.setInputTarget(t)
        r.align(np.eye(4, dtype=F))
        assert not r.hasConverged() or name == "five", name
        if name != "empty":
            k, _ = r.ndtGetCentroids()
            assert k.size == 0, name
            cnt, keys = r.ndtNeighborsAt(POSES[1], src.shape[0])
            assert cnt.sum() == 0 and keys.size == 0
            assert r.ndtDerivativesAt(POSES[1])[3] == 0
        r.close()
    M = ref.map(tgt, 1.0)
    for n in (0, 1, 2):
        r = handle(kd_cfg(1.0), tgt, src[:n].copy()) if n else handle(kd_cfg(1.0), tgt)
        if n:
            check_passes(r, M, src[:n], POSES[1])
        r.align(np.eye(4, dtype=F))
        o = M.align(src[:n])
        assert r.hasConverged() == o["converged"] and r.nr_iterations == o["iterations"]
        r.close()


@pytest.mark.parametrize("res", [0.5, 0.7, 1.0])
def test_radius_boundary(ref, res):
    """(indep.) six valid leaves around an empty cell, centroids on multiples of 2^-10: from every centroid, queries one ulp inside
    the radius, at it (d2 == (float)(r*r)) and one ulp outside"""
    s, a = dy(0.75 * res), dy(res / 8)
    centres = [dy((np.array(cl) + 0.5) * res) for cl in ((0, 0, 0), (-5, 3, 2))]
    anchors = [q + sg * s * np.eye(3)[d] for q in centres for d in range(3) for sg in (1.0, -1.0)]
    tgt = np.concatenate([sym_leaf(x, a) for x in anchors])
    M = ref.map(tgt, res)
    r = handle(kd_cfg(res), tgt)
    k, c = check_centroids(r, M)
    qs, want, exact = [], [], 0
    for ci, cc in enumerate(c):
        for axis in range(3):
            for sign in (1.0, -1.0):
                for lat in ((0.0, 0.0), (0.25 * res, 0.5 * res)):
                    b, ex = boundary_queries(cc, res, axis, sign, lat)
                    qs.append(b)
                    want.append(k[ci])
                    exact += ex
    src = records(np.concatenate(qs))
    r.setInputSource(src)
    cnt, keys = check_neighbours(r, M, src, np.zeros(6), indep=True)
    off = np.r_[0, np.cumsum(cnt)]
    for t, key in enumerate(want):
        for j, inside in enumerate((True, False, False)):
            i = 3 * t + j
            assert (key in keys[off[i]:off[i + 1]]) == inside, (t, j)
    assert exact >= 1
    check_passes(r, M, src, np.zeros(6), min_pairs=len(want))
    r.close()


def test_queries_beyond_every_face_and_beyond_1e9_cells(ref):
    """(indep.) queries out of each of the six faces at 0.3 ... 100 r, centroids in the padding ring of buckets, and far points:
    beyond 1e9 cells and at the float32 limit (no neighbour, not an error)"""
    leaf = 0.1
    tgt, _ = edge_scene(leaf)
    M = ref.map(tgt, leaf)
    r = handle(kd_cfg(leaf), tgt)
    k, c = check_centroids(r, M)
    qs = []
    for axis in range(3):
        for sign in (1.0, -1.0):
            for ci in np.argsort(sign * c[:, axis])[::-1][:4]:
                for t in (0.3, 0.9, 0.9999, 1.0, 1.0001, 1.5, 100.0):
                    q = c[ci].astype(np.float64)
                    q[axis] += sign * t * leaf
                    qs.append(q)
    far = np.array([[1e6, 0, 0], [-1e6, 0, 0], [0, 3e8, 0], [0, 0, -3e8], [1e12, 0.05, 0.05], [1e30, 1e30, 1e30], [-3e38, 0.05, 0.05]])
    src = records(np.r_[np.array(qs), far])
    r.setInputSource(src)
    for p in POSES[:2]:
        cnt, _ = check_neighbours(r, M, src, p, indep=True)
        assert not cnt[-len(far):].any()
        check_passes(r, M, src, p, min_pairs=20)
    r.close()


@pytest.mark.parametrize("res", [1.0, 0.5])
@pytest.mark.parametrize("shifted", [False, True])
def test_degenerate_and_invalidated_leaves(ref, res, shifted):
    """(indep.) every degenerate leaf kind with 5, 6 and 7 points: a centroid exactly for the leaves of >= 6 points, invalidated ones
    included, and those take part in the passes with the inverse they hold (no nr_points check)"""
    off = SHIFT if shifted else (0.0, 0.0, 0.0)
    tgt = degenerate_cloud(res, off, seed=1)
    M = ref.map(tgt, res)
    r = handle(kd_cfg(res), tgt)
    k, c = check_centroids(r, M)
    _, lk = np_leaf_keys(tgt, res)
    ks, cnt = np.unique(lk, return_counts=True)
    assert np.array_equal(k, ks[cnt >= 6])
    v = M.voxels()
    invalid = v["keys"][v["npts"] == -1]
    assert invalid.size >= 10 and np.isin(invalid, k).all()
    rng = np.random.default_rng(2)
    src = np.repeat(tgt, 3, axis=0).copy()
    src[:, :3] += rng.normal(0.0, 0.3 * res, (src.shape[0], 3)).astype(F)
    src = np.concatenate([src, records(c)])
    r.setInputSource(src)
    for p in [np.r_[np.asarray(p[:3]) * res, p[3:]] for p in (NEAR_POSES if shifted else POSES)]:
        check_neighbours(r, M, src, p, indep=True)
        check_passes(r, M, src, p, min_pairs=100)
    r.close()


@pytest.mark.parametrize("res", [1.0, 0.5])
def test_zero_inverse_leaf_adds_minus_d1_per_point(ref, res):
    """leaves of identical points (zero covariance: invalidated, zero inverse) three cells apart; queries within r of exactly one:
    every pair adds the float32 -d1 to the score and nothing to g or H (DIRECT7 skips these leaves)"""
    rng = np.random.default_rng(3)
    cells = [(3 * i, 3 * j, 3 * (i + j) % 2) for i in range(-2, 3) for j in range(-2, 3)]
    tgt = np.concatenate([voxel_points("identical", (6, 7, 9)[t % 3], cl, res, rng, (0.0, 0.0, 0.0)) for t, cl in enumerate(cells)])
    M = ref.map(tgt, res)
    r = handle(kd_cfg(res), tgt)
    k, c = check_centroids(r, M)
    q = np.repeat(c, 20, axis=0).astype(np.float64) + rng.uniform(-0.5 * res, 0.5 * res, (20 * len(cells), 3))
    src = records(q)
    r.setInputSource(src)
    cnt, _ = check_neighbours(r, M, src, np.zeros(6), indep=True)
    assert (cnt == 1).all()
    s, g, H, npairs = check_passes(r, M, src, np.zeros(6))
    d1, _ = np_gauss(res)
    assert npairs == src.shape[0] and abs(s - float(F(-d1)) * npairs) <= 1e-12 * abs(d1 * npairs)
    assert not g.any() and not H.any() and not r.ndtHessianAt(np.zeros(6)).any()
    r.close()


def test_non_finite_inverse_leaf_adds_nothing(ref):
    """a leaf whose covariance passes the eigenvalue check but whose inverse overflows (invalidated with a non-finite inverse): its
    centroid is found, and every term with it fails the range check and adds nothing, not even its score"""
    base = np.array([0.25, 0.25, 0.25])
    tiny = 1e-20  # second moments ~1e-40 survive the eigenvalue check; their inverse ~1e40 ... is not finite in the determinant form
    pts = [base + tiny * np.array(v) for v in ([1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [0, 0, 0])]
    tgt = records(np.array(pts))
    M = ref.map(tgt, 1.0)
    v = M.voxels()
    r = handle(kd_cfg(1.0), tgt)
    check_centroids(r, M)
    src = records(base + np.random.default_rng(4).uniform(-0.4, 0.4, (64, 3)))
    r.setInputSource(src)
    cnt, _ = check_neighbours(r, M, src, np.zeros(6), indep=True)
    assert (cnt == 1).all()
    s, g, H, npairs = check_passes(r, M, src, np.zeros(6))
    assert npairs == 64
    if v["npts"][0] == -1 and not np.isfinite(v["icov"]).all():
        assert s == 0.0 and not g.any() and not H.any()


@pytest.mark.parametrize("res", [0.5, 1.0])
def test_lattice_planes(ref, res):
    """(indep.) leaves on lattice planes x = k res, so their centroids lie on a bucket face or an ulp from it"""
    r32 = F(res)
    xs = np.float32(np.arange(-6, 7, dtype=F) * r32)
    ys = np.float32(np.arange(-3, 4, dtype=F) * r32)
    g = np.stack(np.meshgrid(xs, ys, ys, indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    e = res / 8
    offs = np.array([[0, 0, 0], [0, e, 0], [0, -e, 0], [0, 0, e], [0, 0, -e], [0, e, e], [0, -e, -e]])
    tgt = records((g[:, None, :] + offs[None, :, :]).reshape(-1, 3))
    M = ref.map(tgt, res)
    r = handle(kd_cfg(res), tgt)
    check_centroids(r, M)
    src = records(np.r_[g, g + [res / 2, 0, 0]])
    r.setInputSource(src)
    for p in POSES[:2]:
        check_neighbours(r, M, src, p, indep=True)
        check_passes(r, M, src, p, min_pairs=200)
    r.close()


def test_non_finite_source_points(ref, synth):
    tgt, src = synth.scan("vlp16_16k", frame=0, stride=8), synth.scan("vlp16_16k", frame=1, stride=8)
    odd = src.copy()
    odd[::7, :3] = np.nan
    odd[3::11, 0] = np.inf
    odd[5::13, 2] = -1e12
    M = ref.map(tgt, 1.0)
    r = handle(kd_cfg(1.0), tgt, odd)
    for p in POSES:
        cnt, _ = check_neighbours(r, M, odd, p)
        assert cnt[::7].sum() == 0 and cnt[3::11].sum() == 0
        check_passes(r, M, odd, p, min_pairs=1000)
    r.align(np.eye(4, dtype=F))
    o = M.align(odd)
    assert r.nr_iterations == o["iterations"] and r.hasConverged() == o["converged"]
    assert np.max(np.abs(r.getFinalTransformation() - o["T"])) < 1e-4
    r.close()


@pytest.fixture(scope="module")
def vlp_map(ref, synth):
    tgt = synth.scan("vlp16", frame=0, stride=8)
    return tgt, ref.map(tgt, 1.0)


@pytest.fixture(scope="module")
def big_source(synth):
    return np.concatenate([synth.scan("vlp16", frame=f, stride=8) for f in (1, 2, 3, 4)])


@pytest.mark.parametrize("n", [1, 127, 128, 129, 4095, 4096, 4097, 131073, 200000])
def test_source_sizes(vlp_map, big_source, n):
    """one point, a chunk -1 / +0 / +1, a group -1 / +0 / +1, 33 and 49 groups; after a 200 000-point source has left non-zero
    rows in the handle's workspace"""
    tgt, M = vlp_map
    src = big_source[np.random.default_rng(n).permutation(big_source.shape[0])[:n]].copy() if n < 4096 else big_source[:n].copy()
    r = handle(kd_cfg(1.0), tgt)
    _, cent = r.ndtGetCentroids()
    rng = np.random.default_rng(17)
    prime = np.repeat(cent, -(-200000 // cent.shape[0]), axis=0)[:200000].astype(np.float64)
    r.setInputSource(records(prime + rng.normal(0.0, 0.05, prime.shape)))
    assert r.ndtDerivativesAt(np.zeros(6))[3] >= 200000
    r.ndtHessianAt(np.zeros(6))
    r.setInputSource(src)
    for p in POSES[1:]:
        check_passes(r, M, src, p, min_pairs=1 if n < 4096 else n // 2)
    r.close()
