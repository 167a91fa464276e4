"""GPU: b2r_approximate_voxelgrid / _device and b2r_prefilter's APPROX_VOXELGRID option against the sequential reference of
pcl::ApproximateVoxelGrid (tests/approx_voxelgrid_ref.cpp): records, their order and the counts bit for bit (NaN payloads aside,
see approx_voxelgrid_ref.bits)."""
import numpy as np
import pytest
import torch  # before the engine library: it links the system NCCL, and torch's CUDA libraries must resolve against their own first
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi

from approx_voxelgrid_ref import Reference, CASES, case, decorate, records, same_bits

pytestmark = pytest.mark.gpu

LEAVES = (0.1, 0.25, 1.0)
SCANS = {"vlp16": "vlp16", "hdl32e": "hdl32e", "kitti": "kitti", "262k": (64, 4096)}


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("avg_ref"))


@pytest.fixture(scope="module")
def reg():
    r = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    yield r
    r.close()


@pytest.fixture(scope="module")
def clouds(synth):
    """name -> decorated cloud (32-byte records): four scans and a map-scale cloud of ten KITTI-shape scans (1.2 M points)"""
    out = {k: decorate(synth.scan(v, frame=i, stride=8), seed=i) for i, (k, v) in enumerate(SCANS.items())}
    parts = []
    for f in range(10):
        c = synth.scan("kitti", frame=f, stride=8)
        T = synth.pose_matrix(f).astype(np.float32)
        c[:, :3] = (c[:, :3] @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
        parts.append(c)
    out["map_1.2M"] = decorate(np.concatenate(parts), seed=99)
    return out


def check(reg, ref, cloud, leaf):
    got, cnt = reg.approximateVoxelGridFilter(cloud, leaf, with_counts=True)
    want, wcnt = ref.approximate_voxelgrid(cloud, leaf)
    assert got.shape == want.shape
    assert same_bits(got, want)
    assert np.array_equal(cnt, wcnt)
    return got


def to_device(cloud):
    d = torch.from_numpy(np.ascontiguousarray(cloud)).cuda()
    torch.cuda.synchronize()
    return d


def from_device(ptr, m, stride_f):
    """copy m records at an engine-owned device pointer to the host"""
    from cuda.bindings import runtime as cudart
    copy = torch.empty((m, stride_f), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    if m:
        err, = cudart.cudaMemcpy(copy.data_ptr(), ptr, m * stride_f * 4, cudart.cudaMemcpyKind.cudaMemcpyDeviceToDevice)
        assert int(err) == 0
    return copy.cpu().numpy()


@pytest.mark.parametrize("stride", [4, 8])
@pytest.mark.parametrize("leaf", LEAVES)
@pytest.mark.parametrize("name", list(SCANS) + ["map_1.2M"])
def test_scans_equal_reference(reg, ref, clouds, name, leaf, stride):
    cloud = np.ascontiguousarray(clouds[name][:, :stride])
    got = check(reg, ref, cloud, leaf)
    assert 0 < got.shape[0] < cloud.shape[0]


@pytest.mark.parametrize("n", [0, 1, 2, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 65537])
def test_sizes(reg, ref, synth, n):
    cloud = decorate(synth.scan("kitti", frame=3, stride=8), seed=3)[:n] if n > 6 else synth.scan("kitti", frame=3, stride=8)[:n]
    got = check(reg, ref, cloud, 0.25)
    assert (got.shape[0] == 0) == (n == 0)


@pytest.mark.parametrize("stride", [3, 4, 8])
@pytest.mark.parametrize("name", CASES)
def test_edge_cases(reg, ref, name, stride):
    cloud, leaf = case(name, stride)
    got = check(reg, ref, cloud, leaf)
    if name == "same_bucket_alternating":
        assert got.shape[0] == cloud.shape[0]
    elif name == "one_cell":
        assert got.shape[0] == 1
    elif name == "every_bucket":
        assert got.shape[0] == 512


@pytest.mark.parametrize("name", ["kitti", "map_1.2M"])
def test_device_entry_equals_host_entry_and_repeats(reg, ref, clouds, name):
    cloud = clouds[name]
    host = reg.approximateVoxelGridFilter(cloud, 0.25)
    d = to_device(cloud)
    ptr, m = reg.approximateVoxelGridFilterDevice(d.data_ptr(), d.shape[0], d.shape[1] * 4, 0.25)
    first = from_device(ptr, m, cloud.shape[1])
    ptr2, m2 = reg.approximateVoxelGridFilterDevice(d.data_ptr(), d.shape[0], d.shape[1] * 4, 0.25)
    again = from_device(ptr2, m2, cloud.shape[1])
    assert m == host.shape[0] == m2
    assert np.array_equal(first.view(np.uint32), host.view(np.uint32))
    assert np.array_equal(again.view(np.uint32), first.view(np.uint32))
    assert reg.approximateVoxelGridFilterDevice(d.data_ptr(), 0, 32, 0.25)[1] == 0


def test_invalid_arguments(reg):
    cloud = records(np.zeros((10, 3)), 8)
    for leaf in (0.0, -0.1, float("nan"), float("inf")):
        with pytest.raises(pkg.B2RError) as e:
            reg.approximateVoxelGridFilter(cloud, leaf)
        assert e.value.code == _capi.B2R_EINVAL
        with pytest.raises(pkg.B2RError) as e:
            reg.approximateVoxelGridFilterDevice(0, 0, 32, leaf)
        assert e.value.code == _capi.B2R_EINVAL
        with pytest.raises(pkg.B2RError) as e:
            reg.prefilter(cloud, downsample_method=pkg.B2R_DOWNSAMPLE_APPROX_VOXELGRID, downsample_resolution=leaf)
        assert e.value.code == _capi.B2R_EINVAL
    import ctypes as C
    lib = _capi.load()
    out, m = np.zeros_like(cloud), C.c_size_t()
    for stride in (8, 14, 0):
        rc = lib.b2r_approximate_voxelgrid(reg._h, cloud.ctypes.data_as(C.c_void_p), 10, stride, 0.1, out.ctypes.data_as(C.c_void_p), C.byref(m), None)
        assert rc == _capi.B2R_EINVAL
        d_out = C.c_void_p()
        rc = lib.b2r_approximate_voxelgrid_device(reg._h, None, 0, stride, 0.1, C.byref(d_out), C.byref(m))
        assert rc == _capi.B2R_EINVAL


def host_chain(oracle, ref, raw, deskew_w=None, near=1.0, far=100.0, leaf=0.1, outlier="STATISTICAL", radius=0.8, min_nb=2):
    c = raw if deskew_w is None else oracle.deskew(raw, 0.1, deskew_w)
    c = c[oracle.distance_filter(c, near, far)]
    ds, _ = ref.approximate_voxelgrid(c, leaf)
    if outlier == "STATISTICAL":
        ds = ds[oracle.statistical_outlier(ds, 20, 1.0)[0]]
    elif outlier == "RADIUS":
        ds = ds[oracle.radius_outlier(ds, radius, min_nb)]
    return ds


def test_prefilter_default_parameters(reg, ref, synth, oracle):
    """b2r_prefilter with downsample_method = APPROX_VOXELGRID and the nodelet's defaults == the stages chained on the host"""
    raw = synth.scan("vlp16", frame=9, stride=8)
    out, dptr, m = reg.prefilter(raw, downsample_method=pkg.B2R_DOWNSAMPLE_APPROX_VOXELGRID)
    want = host_chain(oracle, ref, raw)
    assert m == want.shape[0] and dptr
    assert np.array_equal(out.view(np.uint32), want.view(np.uint32))
    # the cloud is downsampled, not passed through: fewer points than without a downsample stage
    _, _, m_none = reg.prefilter(raw, downsample_method=pkg.B2R_DOWNSAMPLE_NONE, want_host=False)
    assert m < m_none


@pytest.mark.parametrize("outlier", ["STATISTICAL", "RADIUS", "NONE"])
def test_prefilter_chain_equals_stagewise_reference(reg, ref, synth, oracle, outlier):
    raw = synth.scan("hdl32e", frame=4, stride=8)
    w = (0.01, -0.02, 0.3)
    method = {"NONE": 0, "STATISTICAL": 1, "RADIUS": 2}[outlier]
    out, dptr, m = reg.prefilter(raw, deskewing=1, scan_period=0.1, angular_velocity=w, distance_near_thresh=1.0, distance_far_thresh=60.0,
                                 downsample_method=pkg.B2R_DOWNSAMPLE_APPROX_VOXELGRID, downsample_resolution=0.25, outlier_removal_method=method,
                                 radius_radius=0.5, radius_min_neighbors=2)
    want = host_chain(oracle, ref, raw, deskew_w=w, near=1.0, far=60.0, leaf=0.25, outlier=outlier, radius=0.5, min_nb=2)
    assert m == want.shape[0] and dptr
    assert np.array_equal(out.view(np.uint32), want.view(np.uint32))


def test_prefilter_device_output_feeds_odometry(synth):
    """raw KITTI-shape scans -> b2r_prefilter (APPROX_VOXELGRID) on the device -> b2r_odometry_matching_device where the cloud lies, against
    the same odometry fed host copies of the filtered clouds: every status field bitwise equal"""
    pre = dict(use_distance_filter=1, distance_near_thresh=0.1, distance_far_thresh=100.0, downsample_method=pkg.B2R_DOWNSAMPLE_APPROX_VOXELGRID,
               downsample_resolution=0.25, outlier_removal_method=2, radius_radius=0.5, radius_min_neighbors=2)
    par = {"registration_method": "FAST_GICP", "reg_transformation_epsilon": 0.1, "reg_max_correspondence_distance": 2.0}
    raws = [synth.scan("kitti", frame=f, stride=8) for f in range(4)]
    reg = pkg.select_registration_method(dict(par))
    odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=5.0, keyframe_delta_angle=2.0, keyframe_delta_time=10000.0)
    host_out = []
    for k, raw in enumerate(raws):
        filt, _, m = reg.prefilter(raw, **pre)
        host_out.append(odo.matching(0.1 * k, filt.copy()))
    odo.close()
    reg.close()
    reg = pkg.select_registration_method(dict(par))
    odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=5.0, keyframe_delta_angle=2.0, keyframe_delta_time=10000.0)
    for k, raw in enumerate(raws):
        d = to_device(raw)
        _, dptr, m = reg.prefilter_raw(d.data_ptr(), d.shape[0], d.shape[1] * 4, device=True, **pre)
        st = odo.matching_raw(0.1 * k, dptr, m, raw.shape[1] * 4, device=True)
        h = host_out[k]
        for key in ("odom", "trans"):
            assert np.array_equal(st[key].view(np.uint32), h[key].view(np.uint32)), (k, key)
        for key in ("converged", "iterations", "keyframe_updated", "frame_rejected"):
            assert st[key] == h[key], (k, key)
        assert np.float64(st["matching_error"]).tobytes() == np.float64(h["matching_error"]).tobytes()
        assert np.float32(st["inlier_fraction"]).tobytes() == np.float32(h["inlier_fraction"]).tobytes()
    odo.close()
    reg.close()
