"""GPU: the ingest seam (row f-4) byte for byte.  b2r_ingest_pointcloud2 / b2r_ingest_pcd write 32-byte pcl::PointXYZI records into an
engine-owned device buffer; every test reads that buffer back and compares its raw bits with the PCL field-mapping restatement of
tests/ingest_ref.py (intensity only from FLOAT32, else 0; words 3, 5-7 constant) — every intensity datatype in both byte orders,
misaligned and overlapping layouts, sizes around the unpack kernel's block and grid-stride boundaries, special float bit patterns,
the layout refusals, PCD bodies, a pinned caller buffer overwritten as soon as the call returns, and the chains the device cloud
feeds (prefilter, odometry, batch), compared bitwise with the same entry points on the decoded host cloud."""
import ctypes as C
import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi
from ingest_ref import (NO_FIELD, FLOAT32, UINT16, DATATYPE_SIZE, PCD_CASES, as_cloud, decode_pointcloud2, layout, parse_pcd_header,
                        pcd_header)

pytestmark = pytest.mark.gpu

_SPECIAL = np.array([0x7FC00000, 0x7FC00001, 0xFFC12345, 0x7F800001, 0x7FBFFFFF, 0x7F800000, 0xFF800000, 0x80000000, 0x00000000,
                     0x00000001, 0x807FFFFF, 0x00800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x3F800000, 0xBF800000], np.uint32)


@pytest.fixture(scope="module")
def reg():
    r = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    yield r
    r.close()


def readback(r, ptr, n):
    """the engine's (n, 8) PointXYZI output as raw bits; the handle's streams are non-blocking, so synchronise them first"""
    from cuda.bindings import runtime as cudart
    r.synchronize()
    out = np.empty((n, 8), np.uint32)
    if n:
        err, = cudart.cudaMemcpy(out.ctypes.data, ptr, out.nbytes, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
        assert int(err) == 0
    return out


def ingest_rc(r, data, n, lay):
    """b2r_ingest_pointcloud2 with its return code (data may be None): (rc, device pointer)"""
    L = _capi.PointLayout(lay["point_step"], lay["off_x"], lay["off_y"], lay["off_z"], lay["off_intensity"], lay["intensity_datatype"],
                          int(lay["is_bigendian"]))
    out = C.c_void_p()
    ptr = None if data is None else data.ctypes.data_as(C.c_void_p)
    rc = r._lib.b2r_ingest_pointcloud2(r._h, ptr, n, C.byref(L), C.byref(out))
    return rc, out.value


def random_blob(n, step, seed):
    return np.random.default_rng(seed).integers(0, 256, n * step, dtype=np.uint8)


def check_exact(r, blob, n, lay):
    ptr = r.ingestPointCloud2(blob, n, **lay)
    got = readback(r, ptr, n)
    want = decode_pointcloud2(blob, n, lay)
    assert np.array_equal(got, want), f"first differing record {np.flatnonzero((got != want).any(1))[:1]}"
    return got


@pytest.mark.parametrize("big", [False, True], ids=["le", "be"])
@pytest.mark.parametrize("dt", [1, 2, 3, 4, 5, 6, 7, 8, None], ids=lambda d: "none" if d is None else f"dt{d}")
def test_intensity_datatypes_and_byte_orders(reg, dt, big):
    """random bytes in a 23-byte record (x@1 y@5 z@9 intensity@13): only a FLOAT32 intensity reaches the point, as in PCL"""
    lay = layout(23, 1, 5, 9, NO_FIELD if dt is None else 13, 7 if dt is None else dt, big)
    got = check_exact(reg, random_blob(3001, 23, dt or 0), 3001, lay)
    if dt != FLOAT32:
        assert not got[:, 4].any()


_LAYOUTS = {
    "step13_odd": layout(13, 1, 5, 9, 2, FLOAT32),                # intensity overlaps x and y
    "step23_f64_odd": layout(23, 3, 7, 11, 15, 8),                # FLOAT64 at an odd offset, ending on point_step
    "reversed_xyz": layout(37, 30, 17, 3, 33, FLOAT32),           # z before y before x, intensity ending on point_step
    "all_at_zero": layout(12, 0, 0, 0, 0, FLOAT32),               # every field on the same four bytes
    "step257_tail": layout(257, 250, 253, 246, 249, FLOAT32),     # fields near the end of a long record, overlapping
    "step48_u16": layout(48, 6, 10, 14, 26, UINT16),
}


@pytest.mark.parametrize("big", [False, True], ids=["le", "be"])
@pytest.mark.parametrize("name", list(_LAYOUTS))
def test_misaligned_and_overlapping_layouts(reg, name, big):
    lay = dict(_LAYOUTS[name], is_bigendian=big)
    check_exact(reg, random_blob(2049, lay["point_step"], sum(name.encode())), 2049, lay)


def _stride():
    from cuda.bindings import runtime as cudart
    err, sms = cudart.cudaDeviceGetAttribute(cudart.cudaDeviceAttr.cudaDevAttrMultiProcessorCount, 0)
    assert int(err) == 0
    return 256 * 16 * sms


@pytest.mark.parametrize("n", ["0", "1", "255", "256", "257", "stride-1", "stride", "stride+1", "1300000"])
def test_sizes_across_block_and_grid_stride(reg, n):
    """k_unpack_points runs min(ceil(n/256), 16*SMs) blocks of 256 threads in a grid-stride loop: n on both sides of one block and of
    one full grid stride (the SM count read from the device), and a 1.3 M-point cloud"""
    s = _stride()
    n = {"stride-1": s - 1, "stride": s, "stride+1": s + 1}.get(n) or int(n)
    lay = layout(32, 0, 4, 8, 16, FLOAT32)
    blob = random_blob(n, 32, n)
    if n == 0:
        rc, ptr = ingest_rc(reg, blob, 0, lay)
        assert rc == 0 and not ptr
        return
    check_exact(reg, blob, n, lay)


@pytest.mark.parametrize("big", [False, True], ids=["le", "be"])
def test_special_bit_patterns(reg, big):
    """NaN payloads (quiet and signalling), +-0, denormals, +-inf and the float extremes in x, y, z and intensity come through bit for bit"""
    k = _SPECIAL.size
    idx = np.array(np.meshgrid(*[np.arange(k)] * 2, indexing="ij")).reshape(2, -1).T   # every ordered pair
    words = np.stack([_SPECIAL[idx[:, 0]], _SPECIAL[idx[:, 1]], _SPECIAL[idx[::-1, 0]], _SPECIAL[idx[::-1, 1]]], 1)
    blob = np.ascontiguousarray(words.astype(">u4" if big else "<u4")).view(np.uint8).reshape(-1)
    lay = layout(16, 0, 4, 8, 12, FLOAT32, big)
    got = check_exact(reg, blob, words.shape[0], lay)
    assert np.array_equal(got[:, [0, 1, 2, 4]], words)


@pytest.mark.parametrize("field", ["x", "y", "z"] + [f"i{dt}" for dt in range(1, 9)])
def test_layout_bounds(reg, field):
    """a field ending exactly on point_step is accepted (and read correctly); one byte further is B2R_EINVAL"""
    step = 29
    size = 4 if field in "xyz" else DATATYPE_SIZE[int(field[1:])]
    base = layout(step, 0, 4, 8, 12, FLOAT32) if field in "xyz" else layout(step, 0, 4, 8, 0, int(field[1:]))
    key = f"off_{field}" if field in "xyz" else "off_intensity"
    blob = random_blob(300, step, 7)
    check_exact(reg, blob, 300, dict(base, **{key: step - size}))
    rc, _ = ingest_rc(reg, blob, 300, dict(base, **{key: step - size + 1}))
    assert rc == _capi.B2R_EINVAL
    check_exact(reg, blob, 300, dict(base, **{key: step - size}))   # the handle still works


def test_layout_refusals(reg):
    blob = random_blob(100, 32, 3)
    assert ingest_rc(reg, blob, 100, layout(11, 0, 4, 4))[0] == _capi.B2R_EINVAL
    for dt in (0, 9):
        assert ingest_rc(reg, blob, 100, layout(32, 0, 4, 8, 16, dt))[0] == _capi.B2R_EINVAL
    assert ingest_rc(reg, None, 100, layout(32))[0] == _capi.B2R_EINVAL
    # without an intensity field the datatype is not looked at
    check_exact(reg, blob, 100, layout(32, 0, 4, 8, NO_FIELD, 0))


def write_pcd(path, kw, seed):
    hdr = pcd_header(kw)
    ref = parse_pcd_header(hdr)
    body = random_blob(ref["points"], ref["layout"]["point_step"], seed)
    path.write_bytes(hdr + body.tobytes())
    return ref, body


_PCD_OK = [c for c in PCD_CASES if c[2] == "ok"]
_PCD_BAD = [c for c in PCD_CASES if c[2] != "ok"]


@pytest.mark.parametrize("name,kw,want", [(c[0], dict(c[1], width=c[1].get("width", 1) * 911), c[2]) for c in _PCD_OK],
                         ids=[c[0] for c in _PCD_OK])
def test_pcd_body_matches_reference(reg, tmp_path, name, kw, want):
    ref, body = write_pcd(tmp_path / "c.pcd", kw, len(name))
    ptr, n = reg.ingestPcd(tmp_path / "c.pcd")
    assert n == ref["points"]
    assert np.array_equal(readback(reg, ptr, n), decode_pointcloud2(body, n, ref["layout"]))


@pytest.mark.parametrize("name,kw,want", _PCD_BAD, ids=[c[0] for c in _PCD_BAD])
def test_pcd_refusals(reg, tmp_path, name, kw, want):
    p = tmp_path / "c.pcd"
    p.write_bytes(pcd_header(kw) + bytes(64))
    with pytest.raises(pkg.B2RError) as e:
        reg.ingestPcd(p)
    assert e.value.code == {"EINVAL": _capi.B2R_EINVAL, "EUNSUPPORTED": _capi.B2R_EUNSUPPORTED}[want]


def test_pcd_short_body_then_growing_files(reg, tmp_path):
    """a body shorter than POINTS says is B2R_EINVAL and leaves the handle usable; a small file followed by ever larger ones (the
    pinned staging buffer is reallocated) reads every body exactly"""
    kw = dict(fields="x y z intensity".split(), size=[4] * 4, typ="FFFF", width=1000)
    p = tmp_path / "short.pcd"
    p.write_bytes(pcd_header(kw) + bytes(16 * 1000 - 1))
    with pytest.raises(pkg.B2RError) as e:
        reg.ingestPcd(p)
    assert e.value.code == _capi.B2R_EINVAL
    for i, w in enumerate((10, 5000, 200000, 30)):
        ref, body = write_pcd(tmp_path / f"g{i}.pcd", dict(kw, width=w), i)
        ptr, n = reg.ingestPcd(tmp_path / f"g{i}.pcd")
        assert n == w and np.array_equal(readback(reg, ptr, n), decode_pointcloud2(body, n, ref["layout"]))


def test_pinned_caller_buffer_is_released_on_return():
    """b2r_ingest_pointcloud2 is synchronous: with the handle's stream held busy (64 GiB of memset queued ahead of the copy), a pinned
    blob overwritten the moment the call returns still yields the original bytes"""
    from cuda.bindings import runtime as cudart
    r = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    n, lay = 4096, layout(32, 0, 4, 8, 16, FLOAT32)
    orig = random_blob(n, 32, 11)
    err, host = cudart.cudaMallocHost(orig.size)
    assert int(err) == 0
    err, busy = cudart.cudaMalloc(1 << 30)
    assert int(err) == 0
    try:
        buf = np.ctypeslib.as_array((C.c_uint8 * orig.size).from_address(host))
        buf[:] = orig
        st = cudart.cudaStream_t(r.getStream())
        for _ in range(64):
            err, = cudart.cudaMemsetAsync(busy, 0, 1 << 30, st)
            assert int(err) == 0
        ptr = r.ingestPointCloud2(buf, n, **lay)
        buf[:] = 0xEE
        got = readback(r, ptr, n)
    finally:
        r.synchronize()
        cudart.cudaFree(busy)
        cudart.cudaFreeHost(host)
        r.close()
    assert np.array_equal(got, decode_pointcloud2(orig, n, lay))


def velodyne_blob(cloud, seed, big=False):
    """x y z intensity FLOAT32 (0, 4, 8, 16) and ring UINT16 @20, point_step 32; random intensities"""
    e = ">" if big else "<"
    dt = np.dtype({"names": ["x", "y", "z", "intensity", "ring"], "formats": [e + "f4"] * 4 + [e + "u2"], "offsets": [0, 4, 8, 16, 20],
                   "itemsize": 32})
    rec = np.zeros(cloud.shape[0], dt)
    rec["x"], rec["y"], rec["z"] = cloud[:, 0], cloud[:, 1], cloud[:, 2]
    rec["intensity"] = np.random.default_rng(seed).uniform(0, 255, cloud.shape[0]).astype(np.float32)
    rec["ring"] = np.arange(cloud.shape[0]) % 16
    return rec.view(np.uint8).reshape(-1).copy(), layout(32, 0, 4, 8, 16, FLOAT32, big)


@pytest.mark.parametrize("big", [False, True], ids=["le", "be"])
def test_pointcloud2_prefilter_chain(reg, synth, big):
    """PointCloud2 -> b2r_prefilter(device_input=1) with the defaults (VOXELGRID + STATISTICAL) == b2r_prefilter on the decoded host
    cloud, bit for bit, intensity averages included"""
    cloud = synth.scan("vlp16_16k", frame=5)
    blob, lay = velodyne_blob(cloud, 5, big)
    n = cloud.shape[0]
    ptr = reg.ingestPointCloud2(blob, n, **lay)
    _, dptr, m = reg.prefilter_raw(ptr, n, 32, device=True)
    got = readback(reg, dptr, m)
    host, _, m_host = reg.prefilter(as_cloud(decode_pointcloud2(blob, n, lay)))
    assert m == m_host and m > 100
    assert np.array_equal(got, host.view(np.uint32))
    assert got[:, 4].any()


def test_uint16_intensity_is_zero_through_the_voxel_grid(reg, synth):
    """an UINT16 intensity is not mapped (PCL leaves PointXYZI's intensity at 0): zero from the unpack to the voxel-grid averages"""
    cloud = synth.scan("vlp16_16k", frame=6)
    n = cloud.shape[0]
    dt = np.dtype({"names": ["x", "y", "z", "intensity"], "formats": ["<f4", "<f4", "<f4", "<u2"], "offsets": [1, 5, 9, 13], "itemsize": 15})
    rec = np.zeros(n, dt)
    rec["x"], rec["y"], rec["z"] = cloud[:, 0], cloud[:, 1], cloud[:, 2]
    rec["intensity"] = np.arange(1, n + 1) % 65535 + 1
    blob = rec.view(np.uint8).reshape(-1).copy()
    lay = layout(15, 1, 5, 9, 13, UINT16)
    ptr = reg.ingestPointCloud2(blob, n, **lay)
    assert not readback(reg, ptr, n)[:, 4].any()
    _, dptr, m = reg.prefilter_raw(ptr, n, 32, device=True)
    got = readback(reg, dptr, m)
    assert m > 100 and not got[:, 4].any()
    host, _, _ = reg.prefilter(as_cloud(decode_pointcloud2(blob, n, lay)))
    assert np.array_equal(got, host.view(np.uint32))


def test_pointcloud2_odometry_chain(synth):
    """PointCloud2 -> b2r_odometry_matching_device over 4 frames == b2r_odometry_matching on the decoded clouds"""
    frames = [synth.scan("vlp16_16k", frame=f) for f in range(4)]
    r_dev, r_host = (pkg.select_registration_method({"registration_method": "FAST_GICP"}) for _ in range(2))
    o_dev, o_host = pkg.ScanMatchingOdometry(r_dev), pkg.ScanMatchingOdometry(r_host)
    for k, cloud in enumerate(frames):
        blob, lay = velodyne_blob(cloud, k)
        n = cloud.shape[0]
        ptr = r_dev.ingestPointCloud2(blob, n, **lay)
        a = o_dev.matching_raw(0.1 * k, ptr, n, 32, device=True)
        b = o_host.matching(0.1 * k, as_cloud(decode_pointcloud2(blob, n, lay)))
        assert np.array_equal(a["odom"], b["odom"]) and np.array_equal(a["trans"], b["trans"])
        assert (a["converged"], a["iterations"], a["keyframe_updated"]) == (b["converged"], b["iterations"], b["keyframe_updated"])
    for o in (o_dev, o_host):
        o.close()
    for r in (r_dev, r_host):
        r.close()


def test_pcd_batch_chain(synth, tmp_path):
    """PCD -> b2r_batch_add_cloud_device -> b2r_batch_align == b2r_batch_add_cloud of the decoded cloud, as source and as target"""
    cloud = synth.scan("vlp16_16k", frame=7)
    n = cloud.shape[0]
    kw = dict(fields="x y z _ intensity ring".split(), size=[4, 4, 4, 1, 4, 2], typ="FFFUFU", count=[1] * 6, width=n)
    hdr = pcd_header(kw)
    ref = parse_pcd_header(hdr)
    dt = np.dtype({"names": ["x", "y", "z", "intensity"], "formats": ["<f4"] * 4, "offsets": [0, 4, 8, 13], "itemsize": 19})
    rec = np.zeros(n, dt)
    rec["x"], rec["y"], rec["z"] = cloud[:, 0], cloud[:, 1], cloud[:, 2]
    rec["intensity"] = np.random.default_rng(1).uniform(0, 100, n).astype(np.float32)
    body = rec.view(np.uint8).reshape(-1)
    (tmp_path / "k.pcd").write_bytes(hdr + body.tobytes())
    assert ref["layout"]["point_step"] == 19 and ref["layout"]["off_intensity"] == 13
    decoded = as_cloud(decode_pointcloud2(body, n, ref["layout"]))
    lb = pkg.RegistrationBatch(params={"registration_method": "FAST_GICP"})
    ptr, m = lb.engine.ingestPcd(tmp_path / "k.pcd")
    assert m == n
    i_dev = lb.addCloudRaw(ptr, n, 32, device=True)
    i_host = lb.addCloud(decoded)
    other = lb.addCloud(synth.scan("vlp16_16k", frame=8))
    eye = np.eye(4, dtype=np.float32)
    res = lb.align([(i_dev, other, eye), (i_host, other, eye), (other, i_dev, eye), (other, i_host, eye)], True)
    lb.close()
    for a, b in ((res[0], res[1]), (res[2], res[3])):
        assert np.array_equal(a["T"], b["T"]) and a["fitness"] == b["fitness"]
        assert (a["converged"], a["iterations"]) == (b["converged"], b["iterations"])
