"""CPU-only: ScanMatchingOdometry's downsample arguments reach b2r_odometry_params (the ctypes mirror of the header's struct)
unchanged, and leaving them out means NONE.  The library is replaced by a stub that records the struct b2r_odometry_create receives."""
import ctypes as C

import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi, registration


class _StubLib:
    def __init__(self):
        self.params = None

    def b2r_odometry_create(self, h, p_ref, out_ref):
        self.params = _capi.OdometryParams.from_buffer_copy(p_ref._obj)
        out_ref._obj.value = 1
        return 0

    def b2r_odometry_destroy(self, o):
        pass


class _StubRegistration:
    _h = C.c_void_p(1)


def _create(monkeypatch, **kw):
    lib = _StubLib()
    monkeypatch.setattr(registration._capi, "load", lambda: lib)
    odo = pkg.ScanMatchingOdometry(_StubRegistration(), **kw)
    odo.close()
    return lib.params


def test_downsample_arguments_reach_the_params_struct(monkeypatch):
    p = _create(monkeypatch, keyframe_delta_trans=2.0, publish_status=True, downsample_method=pkg.B2R_DOWNSAMPLE_APPROX_VOXELGRID,
                downsample_resolution=0.25)
    assert p.downsample_method == _capi.B2R_DOWNSAMPLE_APPROX_VOXELGRID == 2
    assert p.downsample_resolution == 0.25
    assert p.keyframe_delta_trans == 2.0 and p.publish_status == 1  # the fields before them are where they were
    p = _create(monkeypatch, downsample_method=pkg.B2R_DOWNSAMPLE_VOXELGRID, downsample_resolution=0.1)
    assert p.downsample_method == 1 and p.downsample_resolution == C.c_float(0.1).value


def test_default_is_no_downsample(monkeypatch):
    p = _create(monkeypatch)
    assert p.downsample_method == pkg.B2R_DOWNSAMPLE_NONE == 0
    assert p.downsample_resolution == C.c_float(0.1).value
    assert (p.keyframe_delta_trans, p.keyframe_delta_angle, p.keyframe_delta_time) == (0.25, 0.15, 1.0)


def test_params_layout_appends_the_two_fields():
    names = [f[0] for f in _capi.OdometryParams._fields_]
    assert names[-2:] == ["downsample_method", "downsample_resolution"]
    assert _capi.OdometryParams.downsample_method.offset == 52 and _capi.OdometryParams.downsample_resolution.offset == 56
    assert C.sizeof(_capi.OdometryParams) == 64
