"""GPU: b2r_floor_detect on edge inputs against tests/floor_ref.cpp bit for bit, argument errors, and isolation from the registration
and prefilter buffers of the same handle."""
import numpy as np
import pytest
import torch  # noqa: F401  (before the engine library, see test_floor_gpu.py)
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi

from floor_ref import Reference, LAUNCH, assert_same, params

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("floor_ref"))


@pytest.fixture(scope="module")
def reg():
    r = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    yield r
    r.close()


def ground(n, seed=0, noise=0.02, extent=10.0, z=-1.8):
    rng = np.random.default_rng(seed)
    c = np.zeros((n, 8), f32)
    c[:, 0] = rng.uniform(-extent, extent, n)
    c[:, 1] = rng.uniform(-extent, extent, n)
    c[:, 2] = z + rng.normal(0, noise, n)
    c[:, 3] = 1
    c[:, 4] = np.arange(n) % 101
    return c


def both(reg, ref, c, **kw):
    got = reg.floor_detect(c, **kw)
    want = ref.detect(c, **kw)
    assert_same(got, want)
    return got


def test_empty(reg, ref):
    r = both(reg, ref, np.zeros((0, 8), f32))
    assert r["reason"] == "EMPTY_INPUT" and not r["detected"]


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_band_size_around_threshold(reg, ref, delta):
    c = ground(600)
    r = both(reg, ref, c, use_normal_filtering=0, floor_pts_thresh=600 + delta)
    assert (r["reason"] == "TOO_FEW_FILTERED") == (delta > 0)


def test_negative_threshold_always_rejects(reg, ref):
    r = both(reg, ref, ground(2000), floor_pts_thresh=-1)
    assert r["reason"] == "TOO_FEW_FILTERED" and r["n_filtered"] > 0


@pytest.mark.parametrize("n", [1, 2, 3, 5, 9, 10, 11])
def test_tiny_bands(reg, ref, n):
    for normals in (0, 1):
        r = both(reg, ref, ground(n, seed=n), use_normal_filtering=normals, floor_pts_thresh=0)
        if normals and n < 3:
            assert r["n_filtered"] == 0
        if r["n_filtered"] < 3:  # getSamples' "one of these will make it stop"
            assert r["ransac_iterations"] == 2 ** 31 - 2


def test_points_on_both_planes_and_non_finite(reg, ref):
    c = ground(3000, seed=3)
    c[:40, 2] = f32(-3.0)
    c[40:80, 2] = f32(-1.0)
    c[80, 2] = np.nan
    c[81, 0] = np.inf
    c[82, 1] = -np.inf
    c[83, 2] = np.inf
    c[84, 2] = -np.inf
    c[85, :3] = np.nan
    for normals in (0, 1):
        both(reg, ref, c, use_normal_filtering=normals, floor_pts_thresh=100)


def test_collinear_cloud_has_no_model(reg, ref):
    t = (-0.25 - np.arange(1, 801) * 2.0 ** -10).astype(f32)
    c = np.zeros((800, 4), f32)
    c[:, 0], c[:, 1], c[:, 2], c[:, 3] = t, 2 * t, 4 * t, 1
    r = both(reg, ref, c, use_normal_filtering=0, floor_pts_thresh=100)
    assert r["reason"] == "NO_MODEL" and r["model_indices"] == (-1, -1, -1)


def test_duplicate_points_zero_model(reg, ref):
    c = np.tile(np.array([[1.0, 2.0, -1.8, 1.0]], f32), (700, 1))
    r = both(reg, ref, c, use_normal_filtering=0, floor_pts_thresh=100)
    assert r["n_inliers"] == 700 and np.all(r["coeffs"][:3] == 0)


def test_wall_only_band_is_not_vertical(reg, ref):
    rng = np.random.default_rng(4)
    c = np.zeros((3000, 4), f32)
    c[:, 0] = 5.0 + rng.normal(0, 0.01, 3000)
    c[:, 1] = rng.uniform(-5, 5, 3000)
    c[:, 2] = rng.uniform(-2.9, -1.1, 3000)
    c[:, 3] = 1
    r = both(reg, ref, c, use_normal_filtering=0)
    assert r["reason"] == "NOT_VERTICAL"


def test_normal_flipped_upward(reg, ref):
    """the published plane is RANSAC's model, negated when its normal points down: both cases occur and both are checked against
    the model hypothesis itself (the filtered cloud is the input here, so the reference's stream indexes it)"""
    down = up = 0
    for seed in range(12):
        c = ground(3000, seed=10 + seed)
        r = both(reg, ref, c, use_normal_filtering=0)
        assert r["detected"] and r["coeffs"][2] > 0
        hyps = ref.hypotheses(c, r["ransac_iterations"])
        model = next(h for h in hyps if tuple(h["idx"]) == r["model_indices"])
        if model["c"][2] < 0:
            down += 1
            assert np.array_equal(r["coeffs"].view(np.uint32), (-model["c"]).view(np.uint32))
        else:
            up += 1
            assert np.array_equal(r["coeffs"].view(np.uint32), model["c"].view(np.uint32))
    assert down > 0 and up > 0


def test_best_model_on_the_last_capped_hypothesis(reg, ref):
    """the 10 001st hypothesis (the last one before the 10 000-iteration cap stops the loop) is made the strict best: 60 points are
    moved onto its plane.  computeModel saves it before it increments and breaks, so it must be the published model"""
    rng = np.random.default_rng(21)
    c = np.zeros((3000, 4), f32)
    c[:, :3] = rng.uniform(-30, 30, (3000, 3))
    c[:, 3] = 1
    last = ref.hypotheses(c, 10001)[10000]
    assert last["ok"]
    k = np.asarray(last["c"], np.float64)
    a = int(np.argmax(np.abs(k[:3])))
    moved = [i for i in range(3000) if i not in set(last["idx"].tolist())][:60]
    for i in moved:
        rest = sum(k[j] * c[i, j] for j in range(3) if j != a) + k[3]
        c[i, a] = f32(-rest / k[a])
    assert tuple(ref.hypotheses(c, 10001)[10000]["idx"]) == tuple(last["idx"])
    r = both(reg, ref, c, use_normal_filtering=0, floor_pts_thresh=0, height_clip_range=100.0)
    assert r["ransac_iterations"] == 10001
    assert r["model_indices"] == tuple(last["idx"].tolist())
    assert r["n_inliers"] >= 60


def test_noise_band_runs_to_the_iteration_cap(reg, ref):
    """uniform noise in a 60 m band: no plane holds more than a few per cent of it, so k stays above 10 000"""
    rng = np.random.default_rng(5)
    c = np.zeros((5000, 4), f32)
    c[:, :3] = rng.uniform([-30, -30, -30], [30, 30, 30], (5000, 3))
    c[:, 3] = 1
    r = both(reg, ref, c, use_normal_filtering=0, floor_pts_thresh=0, height_clip_range=50.0)
    assert r["ransac_iterations"] == 10001
    assert r["ransac_batches"] > 1


@pytest.mark.parametrize("n", [262144, 1200000])
def test_large_clouds(reg, ref, synth, n):
    parts, total, f = [], 0, 0
    while total < n:
        c = synth.scan("kitti", frame=f, stride=8)
        c[:, 0] += f32(0.37 * f)
        parts.append(c)
        total += c.shape[0]
        f += 1
    c = np.concatenate(parts)[:n]
    for normals in (0, 1):
        both(reg, ref, c, **dict(LAUNCH["hdl"], use_normal_filtering=normals))


def test_argument_errors(reg):
    c = ground(100)
    r = _capi.FloorResult()
    p = params()
    lib = reg._lib
    import ctypes as C
    ptr = c.ctypes.data_as(C.c_void_p)
    for stride in (8, 13, 52):
        assert lib.b2r_floor_detect(reg._h, ptr, 100, stride, 0, C.byref(p), C.byref(r), None, None, None, None) == _capi.B2R_EINVAL
    assert lib.b2r_floor_detect(reg._h, ptr, 100, 32, 0, None, C.byref(r), None, None, None, None) == _capi.B2R_EINVAL
    assert lib.b2r_floor_detect(reg._h, ptr, 100, 32, 0, C.byref(p), None, None, None, None, None) == _capi.B2R_EINVAL
    assert lib.b2r_floor_detect(reg._h, None, 100, 32, 0, C.byref(p), C.byref(r), None, None, None, None) == _capi.B2R_EINVAL


def _read_device(reg, dptr, n):
    """n 32-byte records at a device pointer, read back through a prefilter call with every stage off (it reads its input in place)"""
    import ctypes as C
    out = np.zeros((n, 8), f32)
    p = _capi.PrefilterParams()
    _capi.check(reg._lib.b2r_prefilter_params_default(C.byref(p)))
    p.use_distance_filter, p.downsample_method, p.outlier_removal_method = 0, 0, 0
    m = C.c_size_t()
    _capi.check(reg._lib.b2r_prefilter(reg._h, C.c_void_p(dptr), n, 32, 1, C.byref(p), out.ctypes.data_as(C.c_void_p), None, C.byref(m)))
    return out


def test_isolation_from_the_odometry_chain(synth):
    """b2r_prefilter -> b2r_odometry_matching_device(d_out) -> b2r_floor_detect(d_out): the same poses, flags and aligned cloud as
    without the floor calls, and the prefilter's output bytes are not changed by them"""
    def run(with_floor):
        reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
        odo = pkg.ScanMatchingOdometry(reg)
        out = []
        try:
            for f in range(8):
                c = synth.scan("vlp16", frame=f, stride=8)
                host, dptr, m = reg.prefilter(c, want_host=True)
                st = odo.matching_raw(0.1 * f, dptr, m, 32, device=True)
                if with_floor:
                    assert reg.floor_detect(ptr=dptr, n=m, stride_bytes=32, device=True)["detected"]
                after = _read_device(reg, dptr, m)
                assert np.array_equal(after.view(np.uint32), host.view(np.uint32))
                out.append((st["odom"], st["trans"], st["converged"], st["iterations"], st["keyframe_updated"], st["frame_rejected"]))
        finally:
            odo.close()
            reg.close()
        return out
    a, b = run(False), run(True)
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            if isinstance(u, np.ndarray):
                assert np.array_equal(np.asarray(u).view(np.uint8), np.asarray(v).view(np.uint8))
            else:
                assert u == v


def test_isolation_from_an_aligned_pair(synth):
    """a floor call on the source cloud between align and b2r_get_aligned leaves the aligned cloud, the pose and a following align
    bitwise as without it"""
    tgt, src, nxt = (synth.scan("vlp16", frame=f, stride=8) for f in (0, 1, 2))

    def run(with_floor):
        reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
        try:
            reg.setInputTarget(tgt)
            reg.setInputSource(src)
            reg.align(np.eye(4, dtype=f32))
            if with_floor:
                assert reg.floor_detect(src)["detected"]
            out = [reg.getFinalTransformation(), reg.getAligned()]
            reg.setInputSource(nxt)
            reg.align(np.eye(4, dtype=f32))
            if with_floor:
                reg.floor_detect(nxt, use_normal_filtering=0)
            out += [reg.getFinalTransformation(), reg.getAligned()]
        finally:
            reg.close()
        return out
    for u, v in zip(run(False), run(True)):
        assert np.array_equal(np.asarray(u).view(np.uint8), np.asarray(v).view(np.uint8))
