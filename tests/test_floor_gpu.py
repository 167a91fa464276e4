"""GPU: b2r_floor_detect against the sequential reference of FloorDetectionNodelet::detect (tests/floor_ref.cpp), bit for bit: the
filtered cloud, RANSAC's iterations, model indices and coefficients, the inlier cloud, reason and detected."""
import ctypes as C
import math

import numpy as np
import pytest
import torch  # before the engine library: it links the system NCCL, and torch's CUDA libraries must resolve against their own first
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi

from floor_ref import Reference, LAUNCH, assert_same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("floor_ref"))


@pytest.fixture(scope="module")
def reg():
    r = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    yield r
    r.close()


def shifted(c, dz):
    c = c.copy()
    c[:, 2] += np.float32(dz)
    return c


@pytest.mark.parametrize("sensor", ["vlp16", "hdl32e", "kitti"])
@pytest.mark.parametrize("launch", ["hdl", "501", "kitti"])
def test_raw_scans(ref, reg, synth, sensor, launch):
    c = synth.scan(sensor, frame=2, stride=8)
    if launch == "kitti":
        c = shifted(c, -1.2)  # sensor_height 3.0: put the ground at z = -3.0, inside that band
    got = reg.floor_detect(c, **LAUNCH[launch])
    want = ref.detect(c, **LAUNCH[launch])
    assert_same(got, want)
    assert got["detected"]


@pytest.mark.parametrize("sensor", ["vlp16", "hdl32e", "kitti"])
def test_prefiltered_scans(ref, reg, synth, sensor):
    """b2r_prefilter's defaults first (the KITTI shape through the 0.25 m voxel grid), then the floor call on its device output"""
    c = synth.scan(sensor, frame=5, stride=8)
    res = 0.25 if sensor == "kitti" else 0.1
    host, dptr, m = reg.prefilter(c, want_host=True, downsample_resolution=res)
    got = reg.floor_detect(ptr=dptr, n=m, stride_bytes=32, device=True, **LAUNCH["hdl"])
    assert_same(got, ref.detect(host, **LAUNCH["hdl"]))
    assert_same(reg.floor_detect(host, **LAUNCH["hdl"]), got)


@pytest.mark.parametrize("tilt", [-20.0, -5.0, 5.0, 20.0])
def test_tilted_sensor(ref, reg, synth, tilt):
    c = synth.scan("vlp16", frame=1, stride=8, pitch=math.radians(tilt))
    for t in (tilt, -tilt, 0.0):
        got = reg.floor_detect(c, **dict(LAUNCH["hdl"], tilt_deg=t))
        assert_same(got, ref.detect(c, **dict(LAUNCH["hdl"], tilt_deg=t)))


@pytest.mark.parametrize("stride", [3, 4, 5, 8, 12])
def test_strides_and_fields(ref, reg, synth, stride):
    c = synth.scan("vlp16", frame=3, stride=8)
    a = np.zeros((c.shape[0], stride), np.float32)
    a[:, :min(stride, 8)] = c[:, :min(stride, 8)]
    if stride > 8:
        a[:, 8:] = np.arange(stride - 8, dtype=np.float32) + 0.5
    got = reg.floor_detect(a, **LAUNCH["hdl"])
    assert_same(got, ref.detect(a, **LAUNCH["hdl"]))


def test_host_and_device_input_and_repeat(ref, reg, synth):
    c = synth.scan("hdl32e", frame=7, stride=8)
    a = reg.floor_detect(c)
    t = torch.from_numpy(c).cuda()
    b = reg.floor_detect(ptr=t.data_ptr(), n=c.shape[0], stride_bytes=32, device=True)
    again = reg.floor_detect(c)  # the seed restarts per call, as a fresh PCL model's does
    assert_same(a, b)
    assert_same(a, again)
    assert_same(a, ref.detect(c))
    # the device outputs hold the same clouds as the host copies: read them back through a prefilter with every stage off
    for key, n in (("d_filtered", a["n_filtered"]), ("d_inliers", a["n_inliers"])):
        out = np.zeros((n, 8), np.float32)
        p = _capi.PrefilterParams()
        _capi.check(reg._lib.b2r_prefilter_params_default(C.byref(p)))
        p.use_distance_filter, p.downsample_method, p.outlier_removal_method = 0, 0, 0
        m = C.c_size_t()
        _capi.check(reg._lib.b2r_prefilter(reg._h, C.c_void_p(again[key]), n, 32, 1, C.byref(p), out.ctypes.data_as(C.c_void_p), None, C.byref(m)))
        assert m.value == n
        assert np.array_equal(out.view(np.uint32), (a["filtered"] if key == "d_filtered" else a["inliers"]).view(np.uint32))
