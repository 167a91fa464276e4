"""CPU: b2r_pcd_read_header (host-only, no GPU needed) against the PCD header restatement in tests/ingest_ref.py — field order,
COUNT > 1 and padding fields in the offsets, every intensity type (only F 4 COUNT 1 is mapped, as pcl::PointXYZI's field mapping
does), CRLF / tabs / comments, a missing POINTS line, organized clouds, and the refusals."""
import ctypes as C
import pytest
from hdl_graph_slam_b200 import _capi
from ingest_ref import PCD_CASES, NO_FIELD, FLOAT32, PcdError, parse_pcd_header, pcd_header

_CODES = {"EINVAL": _capi.B2R_EINVAL, "EUNSUPPORTED": _capi.B2R_EUNSUPPORTED}


def read_header(path):
    lib = _capi.load()
    L, n, off = _capi.PointLayout(), C.c_size_t(), C.c_size_t()
    rc = lib.b2r_pcd_read_header(str(path).encode(), C.byref(L), C.byref(n), C.byref(off))
    lay = dict(point_step=L.point_step, off_x=L.off_x, off_y=L.off_y, off_z=L.off_z, off_intensity=L.off_intensity,
               intensity_datatype=L.intensity_datatype, is_bigendian=bool(L.is_bigendian))
    return rc, dict(layout=lay, points=n.value, data_offset=off.value)


@pytest.mark.parametrize("name,kw,want", PCD_CASES, ids=[c[0] for c in PCD_CASES])
def test_pcd_header_matches_reference(tmp_path, name, kw, want):
    hdr = pcd_header(kw)
    p = tmp_path / "c.pcd"
    p.write_bytes(hdr + bytes(64))
    rc, got = read_header(p)
    if want != "ok":
        with pytest.raises(PcdError) as e:
            parse_pcd_header(hdr)
        assert e.value.kind == want
        assert rc == _CODES[want]
        return
    ref = parse_pcd_header(hdr)
    assert rc == 0
    assert got == ref
    assert got["data_offset"] == len(hdr)


def test_pcd_header_reference_known_answers():
    """the restatement itself on hand-computed headers"""
    r = parse_pcd_header(pcd_header(dict(fields="normal _ x y _ z intensity".split(), size=[4, 1, 4, 4, 2, 4, 4], typ="FUFFIFF",
                                         count=[3, 3, 1, 1, 1, 1, 1])))
    assert (r["layout"]["off_x"], r["layout"]["off_y"], r["layout"]["off_z"], r["layout"]["off_intensity"], r["layout"]["point_step"]) == (15, 19, 25, 29, 33)
    for t, s in (("F", 8), ("U", 1), ("U", 2), ("U", 4), ("U", 8), ("I", 1), ("I", 2), ("I", 4), ("I", 8)):
        r = parse_pcd_header(pcd_header(dict(fields="x y z intensity".split(), size=[4, 4, 4, s], typ=f"FFF{t}")))
        assert r["layout"]["off_intensity"] == NO_FIELD and r["layout"]["point_step"] == 12 + s
    r = parse_pcd_header(pcd_header(dict(fields="x y z intensity".split(), size=[4] * 4, typ="FFFF", width=7, height=3, points=False)))
    assert r["points"] == 21 and r["layout"]["off_intensity"] == 12 and r["layout"]["intensity_datatype"] == FLOAT32

