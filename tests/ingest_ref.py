"""Reference for the ingest seam (row f-4): what pcl::fromROSMsg / pcl::fromPCLPointCloud2 and pcl::io::loadPCDFile produce for
pcl::PointXYZI, restated in numpy from PCL's published behaviour.  No code is shared with the engine or the oracle.

  decode_pointcloud2(blob, n, layout)  -> (n, 8) uint32: the raw bits of the 32-byte PointXYZI records x y z 1 | intensity 0 0 0
  parse_pcd_header(data)               -> the layout, point count and body offset of a binary PCD file

PCL maps a message field into a point field only when name, datatype and count all match (FieldMatches).  PointXYZI's intensity is
one float, so an "intensity" field is taken only when it is FLOAT32; any other datatype is left unmapped and the point keeps its
default intensity, 0.  PCL copies the bytes as they are and ignores is_bigendian; the engine byte-swaps instead (there is no
meaningful reference value for a big-endian message on a little-endian host), and this decoder follows the engine there.

Everything is compared as raw bits (uint32 views), so NaN payloads, -0.0, denormals and infinities are exact."""
import numpy as np

NO_FIELD = 0xFFFFFFFF
INT8, UINT8, INT16, UINT16, INT32, UINT32, FLOAT32, FLOAT64 = range(1, 9)
DATATYPE_SIZE = {INT8: 1, UINT8: 1, INT16: 2, UINT16: 2, INT32: 4, UINT32: 4, FLOAT32: 4, FLOAT64: 8}
ONE_BITS = 0x3F800000  # 1.0f, word 3 of every record


def layout(point_step, off_x=0, off_y=4, off_z=8, off_intensity=NO_FIELD, intensity_datatype=FLOAT32, is_bigendian=False):
    """the fields of b2r_point_layout, as a dict (the keyword arguments of Registration.ingestPointCloud2)"""
    return dict(point_step=point_step, off_x=off_x, off_y=off_y, off_z=off_z, off_intensity=off_intensity,
                intensity_datatype=intensity_datatype, is_bigendian=bool(is_bigendian))


def decode_pointcloud2(blob, n, lay):
    """fromPCLPointCloud2 into PointXYZI for n records of lay["point_step"] bytes (rows contiguous) -> (n, 8) uint32"""
    step = lay["point_step"]
    rec = np.frombuffer(bytes(blob), np.uint8, count=n * step).reshape(n, step)
    word = np.dtype(">u4" if lay["is_bigendian"] else "<u4")

    def field(off):
        return np.ascontiguousarray(rec[:, off:off + 4]).view(word).reshape(n).astype(np.uint32)

    out = np.zeros((n, 8), np.uint32)
    out[:, 0], out[:, 1], out[:, 2] = field(lay["off_x"]), field(lay["off_y"]), field(lay["off_z"])
    out[:, 3] = ONE_BITS
    if lay["off_intensity"] != NO_FIELD and lay["intensity_datatype"] == FLOAT32:
        out[:, 4] = field(lay["off_intensity"])
    return out


def as_cloud(bits):
    """the decoded records as the (n, 8) float32 cloud a host entry point takes"""
    return np.ascontiguousarray(bits).view(np.float32)


class PcdError(ValueError):
    """kind is the engine's error code name for the same input: "EINVAL" or "EUNSUPPORTED" """

    def __init__(self, kind, msg):
        super().__init__(f"{kind}: {msg}")
        self.kind = kind


def parse_pcd_header(data):
    """PCDReader::readHeader for what PointXYZI needs -> dict(layout, points, data_offset).

    Blank lines and lines starting with '#' are skipped; tokens are separated by any whitespace (CRLF and tabs included).  DATA ends
    the header and the body starts right after its line.  COUNT defaults to 1 per field; without POINTS the count is WIDTH * HEIGHT.
    A field's byte offset is the sum of SIZE * COUNT of the fields before it.  x, y, z must each be F 4 COUNT 1; intensity is mapped
    only when it is F 4 COUNT 1.  Only DATA binary is read."""
    fields, size, typ, count = None, None, None, None
    width, height, points, data_kind, pos = 0, 1, None, None, 0
    for raw in data.splitlines(keepends=True):
        pos += len(raw)
        line = raw.decode("latin-1").strip()
        if not line or line.startswith("#"):
            continue
        tok = line.split()
        key, vals = tok[0], tok[1:]
        if key in ("FIELDS", "COLUMNS"):
            fields = vals
        elif key == "SIZE":
            size = [int(v) for v in vals]
        elif key == "TYPE":
            typ = [v[0] for v in vals]
        elif key == "COUNT":
            count = [int(v) for v in vals]
        elif key == "WIDTH" and vals:
            width = int(vals[0])
        elif key == "HEIGHT" and vals:
            height = int(vals[0])
        elif key == "POINTS" and vals:
            points = int(vals[0])
        elif key == "DATA" and vals:
            data_kind = vals[0]
            break
    if data_kind is None or not fields:
        raise PcdError("EINVAL", "not a PCD header")
    if count is None:
        count = [1] * len(fields)
    if not (size is not None and typ is not None and len(size) == len(typ) == len(count) == len(fields)):
        raise PcdError("EINVAL", "SIZE / TYPE / COUNT do not match FIELDS")
    if data_kind != "binary":
        raise PcdError("EUNSUPPORTED", f"DATA {data_kind}")
    offsets = np.concatenate([[0], np.cumsum([s * c for s, c in zip(size, count)])]).astype(int)
    f32 = {f: int(offsets[i]) for i, f in enumerate(fields) if typ[i] == "F" and size[i] == 4 and count[i] == 1}
    if not all(k in f32 for k in "xyz"):
        raise PcdError("EINVAL", "no float32 x / y / z")
    lay = layout(int(offsets[-1]), f32["x"], f32["y"], f32["z"], f32.get("intensity", NO_FIELD), FLOAT32, False)
    return dict(layout=lay, points=width * height if points is None else points, data_offset=pos)


def pcd_bytes(fields, size, typ, count=None, width=1, height=1, points=True, data="binary", eol="\n", sep=" ", extra=()):
    """a PCD header as bytes: the lists are written as given (so their lengths may disagree), `points` False leaves POINTS out,
    `extra` lines (comments, blank lines) go after VERSION"""
    n = width * height
    lines = ["# .PCD v0.7 - Point Cloud Data file format", "VERSION 0.7", *extra, sep.join(["FIELDS", *fields]),
             sep.join(["SIZE", *map(str, size)]), sep.join(["TYPE", *typ])]
    if count is not None:
        lines.append(sep.join(["COUNT", *map(str, count)]))
    lines += [f"WIDTH{sep}{width}", f"HEIGHT{sep}{height}", "VIEWPOINT 0 0 0 1 0 0 0"]
    if points:
        lines.append(f"POINTS{sep}{n}")
    lines.append(f"DATA{sep}{data}")
    return (eol.join(lines) + eol).encode()


# (id, header keyword arguments of pcd_bytes, expected result: "ok" / "EINVAL" / "EUNSUPPORTED")
_PCD_TYPES = [("F", 4), ("F", 8), ("U", 1), ("U", 2), ("U", 4), ("U", 8), ("I", 1), ("I", 2), ("I", 4), ("I", 8)]
PCD_CASES = [
    ("xyzi_f4", dict(fields="x y z intensity".split(), size=[4] * 4, typ="FFFF", count=[1] * 4), "ok"),
    ("zyx_order", dict(fields="z intensity y x".split(), size=[4] * 4, typ="FFFF", count=[1] * 4), "ok"),
    ("yxz_no_intensity", dict(fields="y x z".split(), size=[4] * 3, typ="FFF"), "ok"),
    ("lead_count3_and_padding", dict(fields="normal _ x y _ z intensity".split(), size=[4, 1, 4, 4, 2, 4, 4], typ="FUFFIFF",
                                     count=[3, 3, 1, 1, 1, 1, 1]), "ok"),
    ("intensity_count2", dict(fields="x y z intensity".split(), size=[4] * 4, typ="FFFF", count=[1, 1, 1, 2]), "ok"),
    *[(f"intensity_{t}{s}", dict(fields="x intensity y z".split(), size=[4, s, 4, 4], typ=f"F{t}FF", count=[1] * 4), "ok") for t, s in _PCD_TYPES],
    ("crlf_tabs_comments", dict(fields="x y z intensity".split(), size=[4] * 4, typ="FFFF", count=[1] * 4, eol="\r\n", sep="\t",
                                extra=["# a comment", "", "\t", "#another"]), "ok"),
    ("no_points_line", dict(fields="x y z intensity".split(), size=[4] * 4, typ="FFFF", width=7, height=3, points=False), "ok"),
    ("organized_height4", dict(fields="x y z intensity".split(), size=[4] * 4, typ="FFFF", width=5, height=4), "ok"),
    ("data_ascii", dict(fields="x y z".split(), size=[4] * 3, typ="FFF", data="ascii"), "EUNSUPPORTED"),
    ("data_binary_compressed", dict(fields="x y z".split(), size=[4] * 3, typ="FFF", data="binary_compressed"), "EUNSUPPORTED"),
    ("x_f8", dict(fields="x y z".split(), size=[8, 4, 4], typ="FFF"), "EINVAL"),
    ("x_count2", dict(fields="x y z".split(), size=[4] * 3, typ="FFF", count=[2, 1, 1]), "EINVAL"),
    ("x_unsigned", dict(fields="x y z".split(), size=[4] * 3, typ="UFF"), "EINVAL"),
    ("missing_z", dict(fields="x y intensity".split(), size=[4] * 3, typ="FFF"), "EINVAL"),
    ("size_too_short", dict(fields="x y z intensity".split(), size=[4] * 3, typ="FFFF"), "EINVAL"),
    ("type_too_long", dict(fields="x y z".split(), size=[4] * 3, typ="FFFF"), "EINVAL"),
    ("count_too_short", dict(fields="x y z intensity".split(), size=[4] * 4, typ="FFFF", count=[1, 1, 1]), "EINVAL"),
    ("no_data_line", dict(fields="x y z".split(), size=[4] * 3, typ="FFF", data=None), "EINVAL"),
]


def pcd_header(case_kwargs):
    kw = dict(case_kwargs)
    if kw.get("data", "binary") is None:  # a header that never says DATA
        kw["data"] = "binary"
        return pcd_bytes(**kw).rsplit(b"DATA", 1)[0]
    return pcd_bytes(**kw)
