"""GPU: the neighbour searches at every accepted k and their float32 distance decisions placed exactly on their thresholds.

Every discrete output of the engine comes from a float32 squared distance compared with a threshold, or from the k nearest
points.  On random scans no distance ever lands on a threshold, so these tests build clouds where it does, and compare each
decision at the threshold and one step either side with the oracle and with a numpy brute force written here:
  d2 = ((dx^2 + dy^2) + dz^2) in float32 (numpy does not contract to FMA), the k smallest (d2, index) pairs, ties to the lowest index;
  covariances: fast_gicp's mean and covariance in float64 over the min(k, n) neighbours, divided by the count, then I - 0.999 n n^T.
Covered: k_correspondences 1..64 (register-list kernel at 20, the shared-memory list below and above 48 KB), the batch and the
prefetch stream at k != 20; both outlier filters over min_neighbors / mean_k 0..63 at several record strides and through
b2r_prefilter; correspondence, fitness, radius and distance thresholds; the statistical filter's threshold against PCL's sums."""
import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200._capi import B2RError, B2R_EINVAL
from common import rot_err, trans_err

pytestmark = pytest.mark.gpu

SHIFT = np.array([2e4, -3e4, 50.0])
F32MAX = float(np.finfo(np.float32).max)


# ------------------------------------------------------------------------------------------------------ numpy brute force
def bf_d2(pts, q):
    """(nq, n) float32 squared distances in the documented association ((dx^2 + dy^2) + dz^2)"""
    p = np.asarray(pts, np.float32)[:, :3]
    q = np.asarray(q, np.float32)[:, :3]
    d = q[:, None, :] - p[None, :, :]
    s = d * d
    return (s[..., 0] + s[..., 1]) + s[..., 2]


def bf_knn(pts, q, k):
    """k nearest finite points of each query: (idx, d2), ascending by (d2, index); -1 / inf beyond the finite count"""
    d2 = bf_d2(pts, q)
    fin = np.isfinite(np.asarray(pts, np.float32)[:, :3]).all(axis=1)
    d2 = np.where(fin[None, :], d2, np.inf)
    order = np.argsort(d2, axis=1, kind="stable")[:, :k]  # stable: equal d2 stay in index order
    dd = np.take_along_axis(d2, order, axis=1)
    if order.shape[1] < k:
        pad = k - order.shape[1]
        order, dd = np.pad(order, ((0, 0), (0, pad))), np.pad(dd, ((0, 0), (0, pad)), constant_values=np.inf)
    cnt = min(k, int(fin.sum()))
    order[:, cnt:] = -1
    return order.astype(np.int32), dd


def bf_covariances(pts, k, order=None, full=False):
    """fast_gicp calculate_covariances with the PLANE regularisation; also returns, per point, whether the normal is unique (and,
    with full, the unregularised covariances and their eigen-decomposition)"""
    p = np.asarray(pts, np.float32)[:, :3].astype(np.float64)
    n = p.shape[0]
    if order is None:
        order = bf_knn(pts, pts, k)[0]
    kk = min(k, n)
    nb = p[order[:, :kk]]                                     # (n, kk, 3)
    mean = nb.sum(axis=1) / kk
    v = nb - mean[:, None, :]
    C = np.einsum("nki,nkj->nij", v, v) / kk
    w, V = np.linalg.eigh(C)
    normal = V[:, :, 0]
    cov = np.eye(3)[None] - 0.999 * np.einsum("ni,nj->nij", normal, normal)
    unique = (w[:, 1] - w[:, 0]) > 1e-5 * np.maximum(w[:, 2], 1e-300)
    return (cov, unique, C, w, V) if full else (cov, unique)


def plane_properties_hold(C):
    """a regularised covariance: symmetric, eigenvalues {1e-3, 1, 1}"""
    w = np.linalg.eigvalsh(C)
    return np.max(np.abs(C - np.transpose(C, (0, 2, 1)))) < 1e-12 and np.max(np.abs(w - [1e-3, 1.0, 1.0])) < 1e-9


def xyz1(x):
    x = np.asarray(x, np.float64)
    return np.c_[x, np.ones(x.shape[0])].astype(np.float32)


# ------------------------------------------------------------------------------------------------------ clouds
def random_cloud(seed, n=1500, shift=False):
    """uniform points on a 1/128 grid (exact after the shift), with 10 % duplicated points: exact ties at every slot"""
    rng = np.random.default_rng(seed)
    x = np.round(rng.uniform(-4, 4, (n, 3)) * 128) / 128
    x = np.concatenate([x, x[rng.choice(n, n // 10, replace=False)]])
    x = x[rng.permutation(x.shape[0])]
    return xyz1(x + SHIFT if shift else x)


def lattice_cloud(shift=True):
    """anisotropic lattice (spacings 0.5, 0.75, 1.25): every neighbour shell is an exact tie of 2, 4 or 8 points"""
    g = np.stack(np.meshgrid(np.arange(11) * 0.5, np.arange(9) * 0.75, np.arange(7) * 1.25, indexing="ij"), -1).reshape(-1, 3)
    g = np.concatenate([g, g[::13]])
    return xyz1(g + SHIFT if shift else g)


def cov_clouds():
    return {"random": random_cloud(1), "random_shifted": random_cloud(2, shift=True), "lattice_shifted": lattice_cloud()}


def gicp(k=20, **extra):
    p = {"registration_method": "FAST_GICP", "reg_correspondence_randomness": k}
    p.update(extra)
    return pkg.select_registration_method(p)


def smallest_direction(C):
    """unit eigenvector of each matrix's smallest eigenvalue (the normal a regularised covariance carries)"""
    return np.linalg.eigh(C)[1][:, :, 0]


def check_covariances(got, cloud, k, oracle, what, order=None):
    """unique normal: engine == oracle == numpy to 1e-8.  One-point neighbourhood (zero covariance, every direction a normal): engine
    == oracle == diag(1, 1, 1e-3) to 1e-8 (DESIGN.md §2).  Any other degenerate neighbourhood (a line, or a plane with two equal
    spreads) leaves the normal free inside the degenerate eigenspace, and each solver picks its own vector there; both must then be
    regularised covariances whose normal is orthogonal to every direction in which the brute force's neighbour set does spread,
    which pins the set of neighbours chosen (a line through the wrong second neighbour has another direction)."""
    want = oracle.gicp_covariances(cloud, k)
    ref, unique, C, w, V = bf_covariances(cloud, k, None if order is None else order[:, :k], full=True)
    bad = []
    if np.any(unique):
        e_o = np.max(np.abs(got[unique] - want[unique]))
        e_n = np.max(np.abs(got[unique] - ref[unique]))
        if not (e_o < 1e-8 and e_n < 1e-8):
            bad.append(f"{what} k={k}: |engine-oracle| {e_o:.3g} |engine-numpy| {e_n:.3g}")
    iso = ~unique & (C[:, 0, 1] == 0) & (C[:, 0, 2] == 0) & (C[:, 1, 2] == 0) & (C[:, 0, 0] == C[:, 1, 1]) & (C[:, 1, 1] == C[:, 2, 2])
    if np.any(iso):
        e_o = np.max(np.abs(got[iso] - want[iso]))
        e_d = np.max(np.abs(got[iso] - np.diag([1.0, 1.0, 1e-3])))
        if not (e_o < 1e-8 and e_d < 1e-8):
            bad.append(f"{what} k={k}: one-point neighbourhoods |engine-oracle| {e_o:.3g} |engine-diag(1,1,1e-3)| {e_d:.3g}")
    free = ~unique & ~iso
    if np.any(free):
        if not (plane_properties_hold(got[free]) and plane_properties_hold(want[free])):
            bad.append(f"{what} k={k}: degenerate neighbourhoods are not regularised covariances")
        spread = (w[free] - w[free][:, :1]) > 1e-5 * np.maximum(w[free][:, 2:], 1e-300)   # eigenvalues outside the degenerate space
        for name, n in (("engine", smallest_direction(got[free])), ("oracle", smallest_direction(want[free]))):
            dots = np.abs(np.einsum("ni,nij->nj", n, V[free]))
            worst = np.max(np.where(spread, dots, 0.0))
            if not worst < 1e-9:
                bad.append(f"{what} k={k}: {name} normal of a degenerate neighbourhood leans {worst:.3g} into its spread")
    return bad


# ------------------------------------------------------------------------------------------------------ 1. every k
def test_covariances_at_every_k(oracle):
    """k = 1..64 through getCovariances on source and target: the register-list kernel at 20, the shared-memory list up to 48 KB
    below 49 and the opted-in larger list from 49; the target is a full cloud, the source has n = k - 1, k or k + 1 points"""
    clouds = cov_clouds()
    orders = {name: bf_knn(c, c, 64)[0] for name, c in clouds.items()}
    pool = random_cloud(7, n=80, shift=True)
    bad = []
    for k in range(1, 65):
        r = gicp(k)
        for name, tgt in clouds.items():
            r.setInputTarget(tgt)
            bad += check_covariances(r.getCovariances(1, tgt.shape[0]), tgt, k, oracle, name, orders[name])
        for n in (k - 1, k, k + 1):
            if n < 1:
                continue
            src = pool[:n].copy()
            r.setInputSource(src)
            bad += check_covariances(r.getCovariances(0, n), src, k, oracle, f"source n={n}")
        r.close()
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("k", [0, 65, -1])
def test_k_correspondences_out_of_range_is_einval(k):
    with pytest.raises(B2RError) as e:
        gicp(k)
    assert e.value.code == B2R_EINVAL
    cfg = pkg.default_config(pkg.B2R_METHOD_GICP)
    cfg.k_correspondences = k
    with pytest.raises(B2RError) as e:
        pkg.Registration(cfg)
    assert e.value.code == B2R_EINVAL


@pytest.mark.parametrize("k", [1, 19, 21, 48, 49, 64])
def test_batch_align_at_k_equals_single_handle_and_oracle(synth, oracle, k):
    """the batch's k != 20 covariance path: bitwise the single-handle align, and the oracle's align at the same k"""
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)[::4].copy()
    srcs = [synth.scan("vlp16_16k", frame=f, stride=8)[::4].copy() for f in (1, 2)]
    guess = np.eye(4, dtype=np.float32)
    lb = pkg.RegistrationBatch(params={"registration_method": "FAST_GICP", "reg_correspondence_randomness": k})
    ti = lb.addCloud(tgt)
    ids = [lb.addCloud(s) for s in srcs]
    res = lb.align([(i, ti, guess) for i in ids], True, 2.5)
    lb.close()
    r = gicp(k)
    r.setInputTarget(tgt)
    for s, q in zip(srcs, res):
        r.setInputSource(s)
        r.align(guess)
        T = r.getFinalTransformation()
        assert np.array_equal(T, q["T"]) and r.hasConverged() == q["converged"] and r.nr_iterations == q["iterations"]
        f = r.getFitnessScore(2.5)
        assert abs(f - q["fitness"]) <= 1e-12 * abs(f)
        o = oracle.gicp_align(s, tgt, guess, k=k)
        assert o["converged"] == q["converged"] and o["iterations"] == q["iterations"]
        assert trans_err(T, o["T"]) < 1e-6 and rot_err(T, o["T"]) < 1e-6
    r.close()


@pytest.mark.parametrize("k", [49, 64])
def test_prefetched_odometry_at_large_k_is_identical(synth, k):
    """the prefetch stream builds the next scan's covariances with the opted-in shared-memory list"""
    frames = [synth.scan("vlp16_16k", frame=f, stride=8)[::2].copy() for f in range(4)]
    outs = []
    for use_prefetch in (False, True):
        r = gicp(k)
        odo = pkg.ScanMatchingOdometry(r, keyframe_delta_trans=0.5, keyframe_delta_angle=1.0, keyframe_delta_time=10000.0)
        res = []
        for i, c in enumerate(frames):
            if use_prefetch and i + 1 < len(frames):
                odo.prefetch_raw(frames[i + 1].ctypes.data, frames[i + 1].shape[0], frames[i + 1].shape[1] * 4)
            st = odo.matching(0.1 * i, c)
            res.append((st["odom"].copy(), st["iterations"], st["converged"], st["keyframe_updated"]))
        odo.close()
        r.close()
        outs.append(res)
    for a, b in zip(*outs):
        assert np.array_equal(a[0], b[0]) and a[1:] == b[1:]


# ------------------------------------------------------------------------------------------------------ 2. outlier filters
def filter_clouds():
    """a scan-like cloud with duplicates and non-finite points, a tiny one (n <= k for most k) and one with no finite point but
    one; the extra record fields carry distinct values so a partial copy shows"""
    rng = np.random.default_rng(11)
    a = random_cloud(12, n=700, shift=True)[:, :3]
    a[5] = np.nan
    a[17, 2] = np.inf
    a[40, 0] = -np.inf
    tiny = random_cloud(13, n=24)[:, :3]
    tiny[3, 1] = np.nan
    return {"cloud": a, "tiny": tiny, "one_finite": np.array([[1.0, 2.0, 3.0], [np.nan, 0, 0]], np.float32)}, rng


def with_stride(xyz, stride_f, rng):
    out = rng.standard_normal((xyz.shape[0], stride_f)).astype(np.float32)
    out[:, :3] = xyz
    return out


def same_records(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.fixture(scope="module")
def reg():
    r = gicp()
    yield r
    r.close()


def median_radius(xyz, k):
    """radius at the median (k+1)-th neighbour distance over the finite points (None if no point has k + 1 neighbours): about
    half the points are kept and half removed at every min_neighbors = k"""
    fin = np.isfinite(xyz).all(axis=1)
    d2 = bf_knn(xyz, xyz[fin], k + 1)[1][:, k]
    d2 = d2[np.isfinite(d2)]
    return float(np.sqrt(np.median(d2.astype(np.float64)))) if d2.size else None


@pytest.mark.parametrize("which", ["radius", "statistical"])
def test_outlier_filters_over_their_whole_range(reg, oracle, which):
    """min_neighbors / mean_k 0..63 at record strides 16, 20, 32 and 48 bytes: keep masks equal to the oracle's, records copied
    whole; b2r_prefilter with only that stage gives the same records.  The radius filter runs at a fixed radius and at the
    median (k+1)-th neighbour distance of the cloud, so that every k keeps some points and removes others."""
    clouds, rng = filter_clouds()
    bad = []
    for name, xyz in clouds.items():
        for k in range(64):
            params = [0.5]
            if which == "radius":
                r_med = median_radius(xyz, k)
                params = [0.6] + ([r_med] if r_med is not None else [])
            for prm in params:
                for sf in (4, 5, 8, 12):
                    c = with_stride(xyz, sf, rng)
                    if which == "radius":
                        keep = oracle.radius_outlier(c, prm, k)
                        out = reg.radiusOutlierRemoval(c, prm, k)
                    else:
                        keep, _ = oracle.statistical_outlier(c, k, prm)
                        out = reg.statisticalOutlierRemoval(c, k, prm)
                    if not same_records(out, c[keep]):
                        bad.append(f"{which} {name} k={k} param={prm!r} stride={sf * 4}: kept {out.shape[0]}, oracle {int(keep.sum())}")
                pre = dict(use_distance_filter=0, downsample_method=0, outlier_removal_method=1 if which == "statistical" else 2,
                           statistical_mean_k=k, statistical_stddev=prm, radius_radius=prm, radius_min_neighbors=k)
                c = with_stride(xyz, 8, rng)
                keep = oracle.statistical_outlier(c, k, prm)[0] if which == "statistical" else oracle.radius_outlier(c, prm, k)
                out = reg.prefilter(c, **pre)[0]
                if not same_records(out, c[keep]):
                    bad.append(f"b2r_prefilter {which} {name} k={k} param={prm!r}: kept {out.shape[0]}, oracle {int(keep.sum())}")
                # the big cloud discriminates at every k > 0: some points kept, some removed (min_neighbors = 0 keeps every finite
                # point, its own distance being 0; mean_k = 0 keeps every point)
                if name == "cloud" and prm != 0.6 and k > 0:
                    n_fin = int(np.isfinite(xyz).all(axis=1).sum())
                    assert 0 < int(keep.sum()) < n_fin, (which, k, prm, int(keep.sum()))
    assert not bad, "\n".join(bad)


def test_statistical_mean_k_zero_keeps_every_point(reg, oracle):
    """mean_k = 0: every mean distance is 0/0 = NaN, so is the threshold, and !(d > NaN) keeps every point (PCL, the oracle)"""
    c = with_stride(random_cloud(3, n=500)[:, :3], 8, np.random.default_rng(3))
    c[7, 0] = np.nan
    keep, _ = oracle.statistical_outlier(c, 0, 1.0)
    assert keep.all()
    assert same_records(reg.statisticalOutlierRemoval(c, 0, 1.0), c)


@pytest.mark.parametrize("k", [64, 65, -1, -2])
def test_outlier_filter_counts_out_of_range_are_einval(reg, k):
    c = random_cloud(4, n=100)
    for call in (lambda: reg.radiusOutlierRemoval(c, 0.5, k), lambda: reg.statisticalOutlierRemoval(c, k, 1.0),
                 lambda: reg.prefilter(c, use_distance_filter=0, downsample_method=0, outlier_removal_method=2, radius_min_neighbors=k),
                 lambda: reg.prefilter(c, use_distance_filter=0, downsample_method=0, outlier_removal_method=1, statistical_mean_k=k)):
        with pytest.raises(B2RError) as e:
            call()
        assert e.value.code == B2R_EINVAL


# ------------------------------------------------------------------------------------------------------ 3. thresholds on the data
def f32_prev(v):
    return float(np.nextafter(np.float32(v), np.float32(-np.inf)))


def f32_next(v):
    return float(np.nextafter(np.float32(v), np.float32(np.inf)))


def place(v):
    """(dx, dy) in float32 with fl(fl(dx*dx) + fl(dy*dy)) == v exactly (dz = 0): a source point at that offset from a target point
    at the origin has squared distance v"""
    v = np.float32(v)
    x0 = np.float32(np.sqrt(np.float64(v)))
    for i in range(-8, 9):
        dx = np.float32(x0 + np.float32(i) * np.spacing(x0))
        rest = np.float64(v) - np.float64(dx * dx)
        if rest < 0:
            continue
        y0 = np.float32(np.sqrt(rest))
        for j in range(-8, 9):
            dy = np.float32(y0 + np.float32(j) * np.spacing(max(y0, np.float32(1e-30))))
            if dy >= 0 and (dx * dx) + (dy * dy) == v:
                return float(dx), float(dy)
    raise AssertionError(f"no float32 offset has squared distance {float(v)!r}")


def placed_pair(values):
    """target point i at (0, 0, 40 i) and the source point i at (dx, dy, 40 i) with squared distance values[i]; far-apart pairs
    make each source point's nearest target its own.  The target also gets 24 filler points around each target point at
    distance >= 9 so that its covariances are proper ones."""
    tgt, src = [], []
    rng = np.random.default_rng(5)
    for i, v in enumerate(values):
        dx, dy = place(v)
        z = 40.0 * i
        tgt.append([0.0, 0.0, z])
        src.append([dx, dy, z])
        d = rng.standard_normal((24, 3))
        tgt.extend((np.array([0.0, 0.0, z]) + 9.5 * d / np.linalg.norm(d, axis=1)[:, None] * rng.uniform(1.0, 1.5, (24, 1))).tolist())
    tgt, src = xyz1(tgt), xyz1(src)
    d2 = bf_knn(tgt, src, 1)[1][:, 0]
    assert np.array_equal(d2, np.asarray(values, np.float32))
    return src, tgt


@pytest.mark.parametrize("dist", [2.5, 0.1, 0.3])
def test_correspondence_threshold(oracle, dist):
    """a correspondence needs float64(d2) < max_correspondence_distance^2: 2.5^2 = 6.25 is a float, 0.1^2 and 0.3^2 are not"""
    thr2 = dist * dist
    lo = np.float32(thr2)
    below = float(lo) if float(lo) < thr2 else f32_prev(lo)
    above = float(lo) if float(lo) > thr2 else f32_next(lo)
    values = [f32_prev(below), below, above, f32_next(above)]
    if float(lo) == thr2:
        values.insert(2, float(lo))
    src, tgt = placed_pair(values)
    want = np.array([25 * i if v < thr2 else -1 for i, v in enumerate(values)], np.int32)  # target point i is record 25 i
    r = gicp(20, reg_max_correspondence_distance=dist)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    r.gicpLinearizeAt(np.eye(4))
    got = r.getCorrespondences(src.shape[0])
    r.close()
    o = oracle.gicp_linearize(src, oracle.gicp_covariances(src, 20), tgt, oracle.gicp_covariances(tgt, 20), np.eye(4), dist)
    assert np.array_equal(o["corr"], want)
    assert np.array_equal(got, want)


def fitness_ranges(d2):
    v = float(d2)
    return [v, float(np.nextafter(v, -np.inf)), 0.1, 0.0, -1.0, F32MAX, float(np.nextafter(F32MAX, np.inf)), np.inf, np.nan]


def assert_score(got, want):
    assert (got == want) or abs(got - want) <= 1e-12 * abs(want), (got, want)


def test_fitness_thresholds_on_all_four_paths(synth, oracle):
    """the score and its count take d2 <= max_range, the inliers d2 < inlier_thresh_sq: b2r_fitness, align + getFitnessScore,
    b2r_batch_align with want_fitness, b2r_batch_calc_fitness_score.  max_range sits on a point's d2, one double below it, and on
    0.1, 0, a negative value, FLT_MAX, the next double above FLT_MAX, +inf and NaN."""
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)[::8].copy()
    src = synth.scan("vlp16_16k", frame=1, stride=8)[::8].copy()
    r = gicp()
    r.setInputTarget(tgt)
    r.setInputSource(src)
    r.align(np.eye(4, dtype=np.float32))
    T = r.getFinalTransformation()
    _, _, _, _, nd2 = oracle.fitness(tgt, src, T, want_nn=True)
    srt = np.sort(nd2)
    probes = [srt[len(srt) // 2], srt[len(srt) // 5], srt[-1]]
    lb = pkg.RegistrationBatch(params={"registration_method": "FAST_GICP"})
    ti, si = lb.addCloud(tgt), lb.addCloud(src)
    bad = []
    for p in probes:
        for mr in fitness_ranges(p):
            w_score, w_nr, w_inl = oracle.fitness(tgt, src, T, max_range=mr, inlier_thresh_sq=float(p))
            assert w_nr == int(np.sum(nd2.astype(np.float64) <= mr)) and w_inl == int(np.sum(nd2 < p))
            # 1: b2r_fitness at T;  2: after align (the handle's own final pose, which is T)
            for tag, got in (("b2r_fitness", r.getFitnessScore(mr, T=T, inlier_thresh_sq=float(p), full=True)),
                             ("align+getFitnessScore", r.getFitnessScore(mr, inlier_thresh_sq=float(p), full=True))):
                if got[1:] != (w_nr, w_inl) or not ((got[0] == w_score) or abs(got[0] - w_score) <= 1e-12 * abs(w_score)):
                    bad.append(f"{tag} max_range={mr!r}: {got} vs oracle {(w_score, w_nr, w_inl)}")
            # 3: the batch's fitness after its own align (bitwise the same pose)
            q = lb.align([(si, ti, np.eye(4, dtype=np.float32))], True, mr)[0]
            assert np.array_equal(q["T"], T)
            # 4: calc_fitness_score of the edge (target, source, T)
            f4 = lb.calcFitnessScore([(ti, si, T)], max_range=mr)[0]
            for tag, got in (("batch_align", q["fitness"]), ("batch_calc_fitness_score", f4)):
                if not ((got == w_score) or abs(got - w_score) <= 1e-12 * abs(w_score)):
                    bad.append(f"{tag} max_range={mr!r}: {got!r} vs oracle {w_score!r}")
    lb.close()
    r.close()
    assert not bad, "\n".join(bad)


def test_radius_on_the_kth_distance(reg, oracle):
    """a radius whose square is exactly the k-th squared distance keeps the point; the next double below removes it"""
    rng = np.random.default_rng(9)
    line = np.c_[np.arange(40) * 0.75, np.zeros(40), np.zeros(40)]           # neighbours at exactly 0.75, 1.5, ...: d2 0.5625, 2.25
    far = rng.uniform(100, 200, (60, 3))
    c = with_stride(np.r_[line, far].astype(np.float32), 8, rng)
    for radius, min_nb in ((0.75, 2), (1.5, 4), (1.5, 3)):
        for rr, inner_kept in ((radius, True), (float(np.nextafter(radius, 0)), False)):
            keep = oracle.radius_outlier(c, rr, min_nb)
            assert keep[5] == inner_kept and not keep[40:].any()
            assert same_records(reg.radiusOutlierRemoval(c, rr, min_nb), c[keep])


def test_distance_filter_on_near_and_far(reg, oracle):
    """PrefilteringNodelet::distance_filter keeps near < |p| < far: a float norm equal to either bound is excluded"""
    pts = np.array([[3, 4, 0], [0, 3, 4], [6, 8, 0], [0, 0, 10], [f32_next(3.0), 4, 0], [f32_prev(6.0), 8, 0], [1, 2, 2]], np.float32)
    norms = np.sqrt((pts[:, 0] * pts[:, 0] + pts[:, 1] * pts[:, 1]) + pts[:, 2] * pts[:, 2])
    assert norms[0] == norms[1] == 5 and norms[2] == norms[3] == 10
    c = with_stride(pts, 5, np.random.default_rng(1))
    for near, far in ((5.0, 10.0), (f32_prev(5.0), f32_next(10.0)), (float(np.nextafter(5.0, 6)), float(np.nextafter(10.0, 0))), (3.0, 5.0)):
        keep = oracle.distance_filter(c, near, far)
        want = (norms.astype(np.float64) > near) & (norms.astype(np.float64) < far)
        assert np.array_equal(keep, want)
        assert same_records(reg.distanceFilter(c, near, far), c[keep])


# ------------------------------------------------------------------------------------------------------ 4. statistical threshold
def wide_range_cloud():
    """a voxelised VLP-16 scan, 300 points spread over a 4 km cube and a 1 mm cluster: mean distances over many binades, so the
    float64 sums of the statistical filter depend on their order"""
    from hdl_graph_slam_b200 import synth
    from oracle import oracle
    synth_scan = synth.scan("vlp16", frame=3, stride=8)
    v = oracle.voxelgrid(synth_scan, 0.1)[0]
    rng = np.random.default_rng(17)
    spread = rng.uniform(-2000, 2000, (300, 3))
    cluster = np.array([5.0, -7.0, 1.0]) + rng.uniform(0, 1e-3, (200, 3))
    xyz = np.r_[v[:, :3].astype(np.float64), spread, cluster]
    return with_stride(xyz.astype(np.float32), 8, rng)


def sequential_stats(dist):
    """PCL's sums: index order, float64, squares formed in float32"""
    s = sq = 0.0
    for d in dist:
        s += float(d)
        sq += float(np.float32(d) * np.float32(d))
    n = len(dist)
    return s / n, (sq - s * s / n) / (n - 1)


def threshold(mean, var, mul):
    return mean + mul * np.sqrt(var)


def statistical_probes(dist, mean_var, count=6):
    """(point index, mul) such that mean + mul * sqrt(var) equals that point's mean distance exactly, found by nextafter steps from
    the real-valued solution; with the next mul below, the threshold is below the point"""
    mean, var = mean_var
    sd = np.sqrt(var)
    order = np.argsort(dist)[::-1]
    out = []
    for i in order:
        d = float(dist[i])
        if not d > mean:
            break
        mul = (d - mean) / sd
        for _ in range(64):
            t = threshold(mean, var, mul)
            if t == d:
                break
            mul = float(np.nextafter(mul, np.inf if t < d else -np.inf))
        if threshold(mean, var, mul) == d and threshold(mean, var, float(np.nextafter(mul, -np.inf))) < d:
            out.append((int(i), mul))
        if len(out) == count:
            break
    return out


def test_statistical_threshold_probes(reg, oracle):
    """the threshold is mean + mul * stddev of PCL's sequential sums: at a mul that puts it exactly on a point's mean distance the
    point is kept, one step lower it is removed — exactly as the oracle decides, for every point of the cloud"""
    c = wide_range_cloud()
    _, dist = oracle.statistical_outlier(c, 20, 1.0)
    probes = statistical_probes(dist, sequential_stats(dist))
    assert len(probes) >= 3
    for i, mul in probes:
        for m, kept in ((mul, True), (float(np.nextafter(mul, -np.inf)), False)):
            keep, _ = oracle.statistical_outlier(c, 20, m)
            assert keep[i] == kept
            assert same_records(reg.statisticalOutlierRemoval(c, 20, m), c[keep]), (i, m)
            out = reg.prefilter(c, use_distance_filter=0, downsample_method=0, outlier_removal_method=1, statistical_mean_k=20, statistical_stddev=m)[0]
            assert same_records(out, c[keep]), (i, m)
