"""GPU: b2r_get_aligned, the `aligned` output cloud of align() (pcl::transformPointCloud with final_transformation_), bit for bit
against the documented float32 transform ((m0 x + m1 y) + m2 z) + m3 (DESIGN.md §2) computed in numpy with every product and sum a
separate float32 operation: record strides and untouched bytes, sizes around the 256-thread block, non-finite and denormal
coordinates, every way a source can be set, GICP / NDT_OMP / NDT handles, the pose used before any align and after a refused one,
argument errors, the odometry mirror's filtered cloud, and the contract after b2r_promote_source_to_target: no source, B2R_ESTATE."""
import ctypes as C
import numpy as np
import pytest
import torch  # before the engine library: it links the system NCCL, and torch's CUDA libraries must resolve against their own first
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi

pytestmark = pytest.mark.gpu
f32 = np.float32
METHODS = {"gicp": {"registration_method": "FAST_GICP"}, "ndt_omp": {"registration_method": "NDT_OMP", "reg_resolution": 1.0},
           "ndt": {"registration_method": "NDT", "reg_resolution": 1.0}}
SENTINEL = 0xA5


def transform_ref(T, xyz):
    """row r: ((m_r0 x + m_r1 y) + m_r2 z) + m_r3, each operation rounded to float32"""
    T, xyz = np.asarray(T, f32), np.asarray(xyz, f32)
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    with np.errstate(all="ignore"):
        return np.stack([((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3] for r in range(3)], axis=1)


def same_values(a, b):
    """bit-equal, except that any NaN equals any NaN (the GPU returns one canonical NaN, x86 propagates a payload)"""
    a, b = np.ascontiguousarray(a, f32), np.ascontiguousarray(b, f32)
    nan = np.isnan(a) & np.isnan(b)
    return np.array_equal(a.view(np.uint32)[~nan], b.view(np.uint32)[~nan])


def get_aligned(reg, n, stride):
    """-> (rc, the output buffer as bytes (n, stride), pre-filled with a sentinel)"""
    buf = np.full((max(n, 1), stride), SENTINEL, np.uint8)
    rc = reg._lib.b2r_get_aligned(reg._h, buf.ctypes.data_as(C.c_void_p), n, stride)
    return rc, buf[:n]


def check_records(buf, want_xyz, stride):
    n = buf.shape[0]
    got = np.ascontiguousarray(buf[:, :12]).view(f32).reshape(n, 3)
    assert same_values(got, want_xyz)
    if stride >= 16:
        assert np.array_equal(np.ascontiguousarray(buf[:, 12:16]).view(f32).reshape(n), np.ones(n, f32))
    assert np.all(buf[:, 16 if stride >= 16 else 12:] == SENTINEL)  # every other byte untouched


def cloud_of(rng, n, stride):
    a = np.zeros((n, stride // 4), f32)
    a[:, :3] = rng.uniform(-40, 40, (n, 3)).astype(f32)
    a[:, 2] *= 0.1
    if stride >= 16:
        a[:, 3:] = rng.uniform(0, 255, (n, stride // 4 - 3))
    return a


@pytest.fixture(scope="module")
def pair(synth):
    return synth.scan("vlp16_16k", frame=1, stride=8), synth.scan("vlp16_16k", frame=0, stride=8)


@pytest.fixture(params=list(METHODS))
def aligned_reg(request, pair):
    """a handle that has aligned the pair once: final_T is a real, non-trivial pose"""
    src, tgt = pair
    reg = pkg.select_registration_method(dict(METHODS[request.param]))
    reg.setInputTarget(tgt)
    reg.setInputSource(src)
    reg.align(np.eye(4, dtype=f32))
    T = reg.getFinalTransformation()
    assert not np.array_equal(T, np.eye(4, dtype=f32))
    yield reg, T, request.param
    reg.close()


def test_identity_before_any_align(pair):
    src, tgt = pair
    for params in METHODS.values():
        reg = pkg.select_registration_method(dict(params))
        reg.setInputTarget(tgt)
        reg.setInputSource(src)
        rc, buf = get_aligned(reg, src.shape[0], 32)
        assert rc == 0
        check_records(buf, transform_ref(np.eye(4), src[:, :3]), 32)
        reg.close()


@pytest.mark.parametrize("stride", [12, 16, 32, 48])
def test_strides_and_untouched_bytes(aligned_reg, pair, stride):
    reg, T, _ = aligned_reg
    src = pair[0]
    # the source stays the 32-byte cloud of the align; the OUTPUT records may have any stride
    rc, buf = get_aligned(reg, src.shape[0], stride)
    assert rc == 0
    check_records(buf, transform_ref(T, src[:, :3]), stride)
    # and a source of that stride
    a = cloud_of(np.random.default_rng(stride), 3000, stride)
    reg.setInputSourceRaw(a.ctypes.data, a.shape[0], stride)
    rc, buf = get_aligned(reg, a.shape[0], stride)
    assert rc == 0
    check_records(buf, transform_ref(T, a[:, :3]), stride)


@pytest.mark.parametrize("n", [1, 255, 256, 257, 65536, 262144])
def test_sizes_and_special_values(aligned_reg, n):
    reg, T, _ = aligned_reg
    rng = np.random.default_rng(n)
    a = cloud_of(rng, n, 16)
    tiny = np.finfo(f32).tiny
    special = [np.nan, np.inf, -np.inf, f32(tiny) / f32(4), -f32(tiny) / f32(1024), np.finfo(f32).max, 0.0, -0.0]
    for k, v in enumerate(special):  # one special coordinate per record, at the first, the last and block-boundary records
        for i in {0, n - 1, min(255, n - 1), min(256, n - 1)}:
            if n > 8 or k == 0:
                a[(i + k * 7) % n, k % 3] = v
    reg.setInputSource(a)
    rc, buf = get_aligned(reg, n, 16)
    assert rc == 0
    want = transform_ref(T, a[:, :3])
    check_records(buf, want, 16)
    if n > 8:
        assert np.isnan(want).any() and np.isinf(want).any()


@pytest.mark.parametrize("how", ["pageable", "pinned", "device", "prefetch_host", "prefetch_device"])
def test_every_way_to_set_the_source(aligned_reg, how):
    reg, T, _ = aligned_reg
    a = cloud_of(np.random.default_rng(5), 20000, 32)
    n, s = a.shape[0], 32
    keep = None
    if how == "pageable":
        reg.setInputSource(a)
    elif how == "pinned":
        keep = torch.from_numpy(a).pin_memory()
        reg.setInputSourceRaw(keep.data_ptr(), n, s)
    elif how == "device":
        keep = torch.from_numpy(a).cuda()
        torch.cuda.synchronize()
        reg.setInputSourceDevice(keep.data_ptr(), n, s)
    elif how == "prefetch_host":
        h2d = reg.getStats()["h2d_bytes"]
        reg.prefetchSource(a)
        reg.setInputSourceRaw(a.ctypes.data, n, s)
        assert reg.getStats()["h2d_bytes"] - h2d == n * s  # adopted: uploaded once, by the prefetch
    else:
        keep = torch.from_numpy(a).cuda()
        torch.cuda.synchronize()
        reg.prefetchSourceRaw(keep.data_ptr(), n, s, device=True)
        reg.setInputSourceDevice(keep.data_ptr(), n, s)
    rc, buf = get_aligned(reg, n, s)
    assert rc == 0
    check_records(buf, transform_ref(T, a[:, :3]), s)
    del keep


def test_argument_errors(aligned_reg, pair):
    reg, T, _ = aligned_reg
    n = pair[0].shape[0]
    for bad_n in (n - 1, n + 1, 0):
        rc, buf = get_aligned(reg, bad_n, 32)
        assert rc == _capi.B2R_EINVAL and np.all(buf == SENTINEL)
    for bad_stride in (0, 4, 8, 11, 13, 14, 18, 30):
        buf = np.full((n, 64), SENTINEL, np.uint8)
        assert reg._lib.b2r_get_aligned(reg._h, buf.ctypes.data_as(C.c_void_p), n, bad_stride) == _capi.B2R_EINVAL
        assert np.all(buf == SENTINEL)
    assert reg._lib.b2r_get_aligned(reg._h, None, n, 32) == _capi.B2R_EINVAL
    assert reg._lib.b2r_get_aligned(None, None, 0, 32) == _capi.B2R_EINVAL
    reg.setInputSource(np.zeros((0, 8), f32))  # an empty source: nothing to write
    assert reg._lib.b2r_get_aligned(reg._h, None, 0, 32) == 0


@pytest.mark.parametrize("device_clouds", [False, True], ids=["host", "device"])
def test_no_source_after_promote(aligned_reg, pair, device_clouds):
    """b2r_promote_source_to_target takes the source away: align, fitness and the aligned cloud answer B2R_ESTATE until a new source
    is set, instead of reading the slot the old target was left in (whose records may be the caller's released device memory).
    A refused align leaves the final transformation as it was."""
    reg, T, method = aligned_reg
    src, tgt = pair
    lib, h = reg._lib, reg._h
    keep = []
    if device_clouds:  # the target that the promotion displaces was registered from device memory
        keep = [torch.from_numpy(tgt).cuda(), torch.from_numpy(src).cuda()]
        torch.cuda.synchronize()
        reg.setInputTargetDevice(keep[0].data_ptr(), tgt.shape[0], 32)
        reg.setInputSourceDevice(keep[1].data_ptr(), src.shape[0], 32)
        reg.align(np.eye(4, dtype=f32))
        assert np.array_equal(reg.getFinalTransformation(), T)
    reg.promoteSourceToTarget()
    res = _capi.Result()
    g = np.eye(4, dtype=f32).reshape(-1)
    score = C.c_double(-1.0)
    for n in (src.shape[0], tgt.shape[0]):
        rc, buf = get_aligned(reg, n, 32)
        assert rc == _capi.B2R_ESTATE and np.all(buf == SENTINEL)
    assert b"source" in lib.b2r_last_error()
    assert lib.b2r_align(h, g.ctypes.data_as(C.POINTER(C.c_float)), C.byref(res)) == _capi.B2R_ESTATE
    assert res.converged == 0 and res.iterations == 0 and list(res.T) == list(g)  # the failure signal of every refused align
    assert lib.b2r_fitness(h, None, 1e300, 0.25, C.byref(score), None, None) == _capi.B2R_ESTATE and score.value == -1.0
    assert lib.b2r_promote_source_to_target(h) == _capi.B2R_ESTATE  # nothing left to promote
    corr = np.zeros(tgt.shape[0], np.int32)  # the parity taps that read the source refuse as well
    assert lib.b2r_get_correspondences(h, corr.ctypes.data_as(C.POINTER(C.c_int32)), corr.shape[0]) == _capi.B2R_ESTATE
    if method != "gicp":
        p6, H = np.zeros(6), np.zeros(36)
        dp = C.POINTER(C.c_double)
        assert lib.b2r_ndt_hessian_at(h, p6.ctypes.data_as(dp), H.ctypes.data_as(dp)) == _capi.B2R_ESTATE
    # the target side still answers: the promoted cloud is searchable
    idx, d2 = reg.nearestKSearch(src[:100])
    assert np.all(idx >= 0) and np.all(d2 == 0)
    # a new source ends the state; the refused align did not touch the final transformation
    a = cloud_of(np.random.default_rng(9), 5000, 32)
    reg.setInputSource(a)
    rc, buf = get_aligned(reg, 5000, 32)
    assert rc == 0
    check_records(buf, transform_ref(T, a[:, :3]), 32)
    reg.setInputSource(tgt)
    reg.align(np.eye(4, dtype=f32))
    fresh = pkg.select_registration_method(dict(METHODS[method]))
    fresh.setInputTarget(src)
    fresh.setInputSource(tgt)
    fresh.align(np.eye(4, dtype=f32))
    assert np.array_equal(reg.getFinalTransformation(), fresh.getFinalTransformation()) and reg.nr_iterations == fresh.nr_iterations
    fresh.close()
    del keep


@pytest.mark.parametrize("method", ["gicp", "ndt_omp"])
def test_inside_the_odometry_mirror_the_aligned_cloud_is_the_filtered_one(synth, method):
    frames = [synth.scan("vlp16_16k", frame=k, stride=8) for k in range(4)]
    reg = pkg.select_registration_method(dict(METHODS[method]))
    filt = pkg.select_registration_method(dict(METHODS["gicp"]))
    # NDT_OMP moves these scans by millimetres per frame: its keyframe switches on time, GICP's on distance
    odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=1.5, keyframe_delta_angle=1.0, keyframe_delta_time=0.15 if method == "ndt_omp" else 10000.0,
                                   downsample_method=pkg.B2R_DOWNSAMPLE_VOXELGRID, downsample_resolution=0.25)
    seen_plain = seen_switch = 0
    for k, c in enumerate(frames):
        if k + 1 < len(frames):
            odo.prefetch_raw(frames[k + 1].ctypes.data, frames[k + 1].shape[0], 32)
        st = odo.matching(0.1 * k, c)
        f = filt.voxelGridFilter(c, 0.25)
        if k == 0:
            continue
        if st["keyframe_updated"]:  # the frame has become the target: there is no source
            assert get_aligned(reg, f.shape[0], 32)[0] == _capi.B2R_ESTATE
            seen_switch += 1
            continue
        assert get_aligned(reg, c.shape[0], 32)[0] == _capi.B2R_EINVAL  # the raw cloud's size is not the source's
        rc, buf = get_aligned(reg, f.shape[0], 32)
        assert rc == 0
        check_records(buf, transform_ref(st["trans"], f[:, :3]), 32)
        seen_plain += 1
    assert seen_plain >= 1 and seen_switch >= 1
    odo.close()
    reg.close()
    filt.close()
