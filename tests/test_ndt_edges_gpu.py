"""GPU parity of the NDT path on the inputs where its kernels branch, against the CPU oracle (and, where the answer is well-posed,
against numpy): degenerate voxels (5-7 points, exact planes and lines, identical points, eigenvalues at the 1 % clamp, both sides of
0, far from the origin), the staged and the unstaged voxel reads of the derivative pass, source sizes around every chunk / group
boundary of its two-level sum, points outside the map, on its border and exactly on the voxel lattice, non-finite points, a map
without a usable voxel, and the float64 Hessian pass.

Tolerances: voxel keys, point counts, means and inverse covariances bit-exact (the finalisation is the oracle's unfused float64
sequence); score, gradient, Hessian rel <= 1e-9; number of (point, cell) pairs exact."""
import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg
from common import VOXEL_KINDS, voxel_points, perturb, relrel, rot_err, trans_err

pytestmark = pytest.mark.gpu

POSES = ([0, 0, 0, 0, 0, 0], [0.09, 0.05, -0.02, 0.01, -0.015, 0.03], [-0.2, 0.1, 0.05, 0.05, 0.02, -0.04])
# far from the origin a rotation of 0.01 rad moves a point by hundreds of metres: there only translations and micro-rotations
NEAR_POSES = ([0, 0, 0, 0, 0, 0], [0.09, 0.05, -0.02, 0, 0, 0], [-0.2, 0.1, 0.05, 3e-6, -2e-6, 1e-6])
SHIFT = (20000.0, -30000.0, 50.0)


def make(res, search="DIRECT7", **kw):
    params = {"registration_method": "NDT_OMP", "reg_resolution": res, "reg_nn_search_method": search}
    params.update(kw)
    return pkg.select_registration_method(params)


def degenerate_cloud(res, offset=(0.0, 0.0, 0.0), seed=0):
    """every kind of VOXEL_KINDS with 5, 6 and 7 points, in cells on both sides of 0 (every other cell, so voxels also have empty
    face neighbours), plus generic 12-point voxels between them as face neighbours of some"""
    rng = np.random.default_rng(seed)
    parts, cell = [], 0
    for kind in VOXEL_KINDS:
        for n in (5, 6, 7):
            for sgn in (1, -1):
                c = (sgn * (2 * (cell % 6) + 1), sgn * (2 * ((cell // 6) % 6)), (cell // 36) * 2 - 1)
                parts.append(voxel_points(kind, n, c, res, rng, offset))
                parts.append(voxel_points("generic", 12, (c[0] + 1, c[1], c[2]), res, rng, offset))
                cell += 1
    return np.concatenate(parts)


def source_near(tgt, rng, n_jitter=3, sigma=0.3):
    """points around the target's: every target point moved by a few random offsets"""
    src = np.repeat(tgt, n_jitter, axis=0).copy()
    src[:, :3] += rng.normal(0.0, sigma, (src.shape[0], 3)).astype(np.float32)
    return src


def check_voxels(r, om):
    got, want = r.ndtGetVoxels(), om.dump()
    assert np.array_equal(got["min_b"], want["min_b"]) and np.array_equal(got["div_b"], want["div_b"])
    assert np.array_equal(got["keys"], want["keys"])
    bad = int(np.sum(got["npts"] != want["npts"]))
    assert bad == 0, f"{bad} voxels differ in point count / validity"
    assert np.array_equal(got["mean"], want["mean"])
    assert np.array_equal(got["icov"], want["icov"])  # bit-exact, invalidated voxels included
    return want


def check_derivatives(r, om, src, search, poses=POSES, min_pairs=1):
    sm = 7 if search == "DIRECT7" else 1
    for p in poses:
        score, g, H, npairs = r.ndtDerivativesAt(p)
        o = om.derivatives(src, p, search_method=sm)
        assert npairs == o["n_pairs"] and npairs >= min_pairs, (p, npairs, o["n_pairs"])
        assert abs(score - o["score"]) <= 1e-9 * abs(o["score"])
        assert relrel(g, o["g"]) < 1e-9 and relrel(H, o["H"]) < 1e-9
        Hh = r.ndtHessianAt(p)
        oh = om.hessian_at(src, p, search_method=sm)
        assert relrel(Hh, oh) < 1e-9, p


def independent_voxel_check(cloud, res, dump):
    """float64 numpy restatement of VoxelGridCovariance for voxels whose validity / clamp decision is well-posed (margin above 1e-9
    relative): np.linalg.eigh of the (n-1)/n-scaled population covariance, ndt_omp's 1 % clamp, inverse.  Catches the oracle and
    the engine being wrong together."""
    xyz = cloud[:, :3]
    inv = np.float32(1.0) / np.float32(res)
    ijk = np.floor(xyz * inv).astype(np.int64)  # float32 product, as the map build
    ijk -= dump["min_b"].astype(np.int64)
    div = dump["div_b"].astype(np.int64)
    keys = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1]
    checked = 0
    for v, k in enumerate(dump["keys"]):
        pts = xyz[keys == k].astype(np.float64)
        n = pts.shape[0]
        assert n == abs(dump["npts"][v]) or dump["npts"][v] == -1
        if n < 6:
            assert dump["npts"][v] == n
            continue
        cov = np.cov(pts.T, ddof=0) * (n - 1) / n
        w, V = np.linalg.eigh(cov)
        scale = max(w[2], 1e-300)
        # ndt_omp's moment formula S2/n - mean mean^T cancels: far from the origin its covariance carries an absolute error of
        # ~eps |mean|^2, which bounds how well-posed the decisions are and how close its inverse can come to this one
        noise = 16 * np.finfo(np.float64).eps * (float(np.dot(pts[0], pts[0])) + scale)
        margins = [w[0], abs(w[0] - 0.01 * scale), abs(w[1] - 0.01 * scale)]
        if w[2] <= 1e-9 * res * res or min(margins) < 1e-9 * scale + noise:
            continue  # rounding decides: ill-posed for any solver
        checked += 1
        assert dump["npts"][v] == n
        wc = w.copy()
        if wc[0] < 0.01 * wc[2]:
            wc[0] = 0.01 * wc[2]
            wc[1] = max(wc[1], 0.01 * wc[2])
        icov = V @ np.diag(1.0 / wc) @ V.T
        tol = 1e-6 + 100 * noise / wc[0]
        assert np.max(np.abs(dump["icov"][v] - icov)) <= tol * np.max(np.abs(icov)), (v, tol)
    return checked


@pytest.mark.parametrize("res", [1.0, 0.5])
@pytest.mark.parametrize("shifted", [False, True])
def test_degenerate_voxels(oracle, res, shifted):
    off = SHIFT if shifted else (0.0, 0.0, 0.0)
    tgt = degenerate_cloud(res, off, seed=1)
    r = make(res)
    r.setInputTarget(tgt)
    om = oracle.NdtMap(tgt, res)
    want = check_voxels(r, om)
    assert np.sum(want["npts"] == -1) >= 10 and np.sum(want["npts"] >= 6) >= 40 and np.sum((want["npts"] > 0) & (want["npts"] < 6)) >= 10
    assert independent_voxel_check(tgt, res, want) >= 40
    src = source_near(tgt, np.random.default_rng(2), sigma=0.3 * res)
    r.setInputSource(src)
    poses = [np.r_[np.asarray(p[:3]) * res, p[3:]] for p in (NEAR_POSES if shifted else POSES)]
    for search in ("DIRECT7", "DIRECT1"):
        r2 = make(res, search)
        r2.setInputTarget(tgt)
        r2.setInputSource(src)
        check_derivatives(r2, om, src, search, poses, min_pairs=100)
        r2.close()
    r.close()


def test_staged_voxel_reads(oracle):
    """a source confined to a 4x4x4-cell cube: a block's box of base cells +-1 is at most 6^3 = 216 <= 320 cells, so every chunk
    stages its voxel records in shared memory"""
    rng = np.random.default_rng(3)
    tgt = np.c_[rng.uniform(-3, 7, (20000, 3)), np.ones(20000)].astype(np.float32)
    src = np.c_[rng.uniform(0.05, 3.95, (6000, 3)), np.ones(6000)].astype(np.float32)
    poses = ([0, 0, 0, 0, 0, 0], [0.01, -0.01, 0.01, 0.002, -0.002, 0.002])  # moves no point by more than 0.03: all stay in the cube
    r = make(1.0)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    om = oracle.NdtMap(tgt, 1.0)
    check_voxels(r, om)
    check_derivatives(r, om, src, "DIRECT7", poses, min_pairs=6000 * 5)
    r.close()


def test_unstaged_voxel_reads(oracle):
    """a source on a line along x with consecutive points 400 cells apart: any 128 of them span more than 320 cells, so every
    chunk reads its voxels from the hash table directly"""
    rng = np.random.default_rng(4)
    k = np.arange(-512, 512)
    centres = np.c_[400.0 * k + 0.5, np.full(k.size, 0.5), np.full(k.size, 0.5)]
    tgt = np.concatenate([np.c_[c + rng.integers(-12, 13, (10, 3)) / 32.0, np.ones(10)] for c in centres]).astype(np.float32)
    src = np.c_[centres + rng.integers(-14, 15, (k.size, 3)) / 32.0, np.ones(k.size)].astype(np.float32)
    cells = np.unique(np.floor(src[:, 0]))
    assert cells.size == src.shape[0] and np.min(np.diff(cells)) > 320
    for search in ("DIRECT7", "DIRECT1"):
        r = make(1.0, search)
        r.setInputTarget(tgt)
        r.setInputSource(src)
        om = oracle.NdtMap(tgt, 1.0)
        check_voxels(r, om)
        check_derivatives(r, om, src, search, poses=NEAR_POSES, min_pairs=500)
        r.close()


@pytest.fixture(scope="module")
def big_source(synth):
    return np.concatenate([synth.scan("vlp16", frame=f, stride=8) for f in (1, 2, 3, 4)])


@pytest.mark.parametrize("n", [1, 127, 128, 129, 4095, 4096, 4097, 131073, 200000])
def test_source_sizes(oracle, synth, big_source, n):
    """128-point chunks, 32-chunk (4096-point) groups: one point, a chunk -1 / +0 / +1, a group -1 / +0 / +1, 33 groups (one full
    round of the unrolled 32-row sum of the group rows plus a remainder of one) and 49 groups (remainder 17)"""
    tgt = synth.scan("vlp16", frame=0, stride=8)
    src = big_source[np.random.default_rng(n).permutation(big_source.shape[0])[:n]].copy() if n < 4096 else big_source[:n].copy()
    r = make(1.0)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    om = oracle.NdtMap(tgt, 1.0)
    check_derivatives(r, om, src, "DIRECT7", poses=POSES[1:2], min_pairs=1 if n < 4096 else n)
    r.close()


@pytest.mark.parametrize("search", ["DIRECT7", "DIRECT1"])
def test_points_outside_and_on_the_border_of_the_map(oracle, synth, search):
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)
    lo, hi = tgt[:, :3].min(axis=0), tgt[:, :3].max(axis=0)
    rng = np.random.default_rng(6)
    base = synth.scan("vlp16_16k", frame=1, stride=8)[::4].copy()
    out = base[:600].copy()
    out[:300, 0] = hi[0] + rng.uniform(0.0, 3.0, 300)      # beyond the max border (incl. the face-neighbour cell just outside)
    out[300:, 1] = lo[1] - rng.uniform(0.0, 3.0, 300)      # beyond the min border
    border = tgt[rng.choice(tgt.shape[0], 400, replace=False)].copy()
    border[:100, 0] = hi[0]; border[100:200, 0] = lo[0]; border[200:300, 2] = hi[2]; border[300:, 2] = lo[2]  # exactly on the extremes
    src = np.concatenate([base, out, border])
    r = make(1.0, search)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    check_derivatives(r, oracle.NdtMap(tgt, 1.0), src, search, min_pairs=1000)
    r.close()


def test_map_without_a_usable_voxel(oracle):
    """every voxel holds fewer than 6 points: no pair, score exactly 0, and the align returns what the oracle's does"""
    rng = np.random.default_rng(7)
    tgt = np.concatenate([voxel_points("generic", 5, (i, j, 0), 1.0, rng) for i in range(-10, 10) for j in range(-10, 10)])
    src = source_near(tgt, rng, 2, 0.2)
    r = make(1.0)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    om = oracle.NdtMap(tgt, 1.0)
    assert np.all(check_voxels(r, om)["npts"] < 6)
    score, g, H, npairs = r.ndtDerivativesAt(POSES[1])
    assert npairs == 0 and score == 0.0 and not np.any(g) and not np.any(H)
    G = perturb(3, 0.2, 1.0).astype(np.float32)
    r.align(G)
    o = om.align(src, G)
    assert r.hasConverged() == o["converged"] and r.nr_iterations == o["iterations"]
    assert np.array_equal(r.getFinalTransformation(), o["T"])
    r.close()


@pytest.mark.parametrize("res", [0.1, 0.5, 0.7, 1.0])
def test_points_on_lattice_planes(oracle, res):
    """coordinates exactly k * res in float32 (negative k and -0.0 included): the map is built with floor(x * (1 / res)), lookups use
    floor(x / res); the lattice values where the two disagree (at res 0.7 from |k| ~ 2000 on) are included, and the engine must
    reproduce both roundings"""
    r32 = np.float32(res)
    k = np.arange(-3000, 3001, dtype=np.float32)
    lat = np.float32(k * r32)
    split = lat[np.floor(lat * (np.float32(1) / r32)) != np.floor(lat / r32)][::6][:24]
    xs = np.r_[np.float32(np.arange(-12, 13, dtype=np.float32) * r32), np.float32(-0.0), split].astype(np.float32)
    ys = np.r_[np.float32(np.arange(-4, 5, dtype=np.float32) * r32), np.float32(-0.0)].astype(np.float32)
    g = np.stack(np.meshgrid(xs, ys, ys[::2], indexing="ij"), -1).reshape(-1, 3)
    rng = np.random.default_rng(8)
    fill = np.repeat(g, 4, axis=0) + rng.uniform(-1.5 * res, 1.5 * res, (4 * g.shape[0], 3))
    tgt = np.c_[np.r_[g, fill], np.ones(5 * g.shape[0])].astype(np.float32)
    src = np.c_[g, np.ones(g.shape[0])].astype(np.float32)
    r = make(res)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    om = oracle.NdtMap(tgt, res)
    check_voxels(r, om)
    check_derivatives(r, om, src, "DIRECT7", poses=POSES[:1], min_pairs=500)
    r.close()


def test_non_finite_source_points(oracle, synth):
    """NaN / inf coordinates and points whose cell index leaves int range contribute nothing, in the engine and in the oracle"""
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)
    src = synth.scan("vlp16_16k", frame=1, stride=8)[::2].copy()
    src[3, 0] = np.nan; src[10, 1] = np.inf; src[11, 2] = -np.inf; src[500, :3] = np.nan
    src[700, 0] = 3.0e12; src[701, 1] = -3.0e12
    keep = np.isfinite(src[:, :3]).all(axis=1) & (np.abs(src[:, :3]) < 1e9).all(axis=1)
    r = make(1.0)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    om = oracle.NdtMap(tgt, 1.0)
    check_derivatives(r, om, src, "DIRECT7", min_pairs=1000)
    clean = om.derivatives(src[keep], POSES[1])
    assert om.derivatives(src, POSES[1])["n_pairs"] == clean["n_pairs"]
    r.close()


@pytest.mark.parametrize("search", ["DIRECT7", "DIRECT1"])
def test_hessian_pass_on_a_scan(oracle, synth, search):
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)
    src = synth.scan("vlp16_16k", frame=1, stride=8)
    r = make(1.0, search)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    om = oracle.NdtMap(tgt, 1.0)
    sm = 7 if search == "DIRECT7" else 1
    for p in ([0, 0, 0, 0, 0, 0], [0.9, 0.05, -0.02, 0.01, -0.015, 0.03], [1.0, 0.0, 0.0, 3.1, 3.13, -3.1]):
        H = r.ndtHessianAt(p)
        o = om.hessian_at(src, p, search_method=sm)
        assert np.any(o) and relrel(H, o) < 1e-9
        # the float64 pass and the float32 derivative pass compute the same Hessian to float32 accuracy
        assert relrel(H, om.derivatives(src, p, search_method=sm)["H"]) < 1e-3
    r.close()


def test_line_search_runs_the_hessian_pass(oracle, synth):
    """mt_interval_flag = 1 (More-Thuente loop active) with a guess for which the oracle's line search iterates: the engine launches
    the float64 Hessian pass as often as the oracle runs it, and the derivative pass as often as the oracle's other passes"""
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)
    src = synth.scan("vlp16_16k", frame=1, stride=8)
    om = oracle.NdtMap(tgt, 1.0)
    for seed in range(20, 40):
        G = perturb(seed, 0.5, 3.0).astype(np.float32)
        o = om.align(src, G, mt_interval_flag=1)
        if o["hessian_passes"] >= 1:
            break
    assert o["hessian_passes"] >= 1, "no guess made the oracle's line search iterate"
    cfg = pkg.default_config(pkg.B2R_METHOD_NDT)
    cfg.ndt_resolution = 1.0
    cfg.ndt_mt_interval_flag = 1
    r = pkg.Registration(cfg)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    r.ndtGetVoxels()  # the map build is not part of the counted launches
    r.getStats(reset=True)
    r.align(G)
    launches = r.getStats()["launches"]
    assert launches["ndt_hessian"] == o["hessian_passes"]
    assert launches["ndt_derivatives"] == o["derivative_passes"] - o["hessian_passes"]
    assert r.nr_iterations == o["iterations"] and r.hasConverged() == o["converged"]
    T = r.getFinalTransformation()
    assert trans_err(T, o["T"]) < 1e-4 and rot_err(T, o["T"]) < 1e-4
    r.close()
