"""GPU: the front-end drop-in (adapter/b200_frontend.hpp) EXECUTED through tests/frontend_harness.cpp and the test-only stand-ins
adapter/pcl_shim.hpp + backend_shim.hpp + frontend_shim.hpp, the way PrefilteringNodelet and FloorDetectionNodelet call it.

B200Prefilter, under the code defaults and the prefilter rosparams of launch/hdl_graph_slam{,_400,_501,_kitti}.launch:
  - every output is byte for byte b2r_prefilter called directly with a b2r_prefilter_params built here from the reference lines
    (prefiltering_nodelet.cpp:50-99, 106-136, 182-243): deskew on and off, base_link transform given and not, every downsample and
    outlier name (unknown ones too), use_distance_filter false (the distance filter still runs), scan_period changed between calls;
  - on one VLP-16 and one KITTI scan the output equals the oracle's stage-wise chain (distance filter, voxel grid, outlier filter);
  - header, frame_id, width, height and is_dense follow the header's rules; an empty input gives nullptr.
The PointCloud2 overloads, on velodyne-style, Ouster-style organized (NaN records, 1.3 M points), big-endian, padded-row and UINT8 /
no-intensity messages: bitwise the pcl overloads on the cloud tests/frontend_ref.py decodes row by row.  b2r_ingest_pointcloud2_rows
is bitwise b2r_ingest_pointcloud2 at height 1 and on contiguous organized messages, and refuses a short row_step.
B200FloorDetector on prefiltered VLP-16, HDL-32E and KITTI scans with the hdl, 501 and kitti floor parameters: bitwise
b2r_floor_detect, and tests/floor_ref.cpp's coefficients, model indices and clouds; filtered() on every frame it was asked for,
inliers() only with a floor; the size gate, not-vertical and empty cases.  A prefilter and a floor detector on two threads give the
serial answers."""
import ctypes as C
import os
import struct
import subprocess
import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi
from ingest_ref import FLOAT32, as_cloud, decode_pointcloud2
from frontend_ref import decode_rows, layout_of, message
from floor_ref import LAUNCH as FLOOR_LAUNCH, Reference, assert_same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PREFILTER, FLOOR = 1, 2
OK, INVALID_ARGUMENT, RUNTIME_ERROR = 0, 1, 2

# the prefilter rosparams of each launch file (the nodelet's <param> lines); "defaults" sets none
PREFILTER_LAUNCH = {
    "defaults": {},
    "hdl": dict(base_link_frame="base_link", use_distance_filter="false", distance_near_thresh="0.1", distance_far_thresh="1000.0",
                downsample_method="VOXELGRID", downsample_resolution="0.1", outlier_removal_method="NONE", statistical_mean_k="30",
                statistical_stddev="1.2", radius_radius="0.5", radius_min_neighbors="2"),
    "400": dict(base_link_frame="base_link", use_distance_filter="true", distance_near_thresh="0.1", distance_far_thresh="100.0",
                downsample_method="VOXELGRID", downsample_resolution="0.1", outlier_removal_method="RADIUS", statistical_mean_k="30",
                statistical_stddev="1.2", radius_radius="0.5", radius_min_neighbors="2"),
    "501": dict(base_link_frame="base_link", use_distance_filter="true", distance_near_thresh="0.5", distance_far_thresh="100.0",
                downsample_method="VOXELGRID", downsample_resolution="0.1", outlier_removal_method="RADIUS", statistical_mean_k="30",
                statistical_stddev="1.2", radius_radius="0.5", radius_min_neighbors="2"),
    "kitti": dict(base_link_frame="base_link", use_distance_filter="true", distance_near_thresh="0.1", distance_far_thresh="100.0",
                  downsample_method="VOXELGRID", downsample_resolution="0.25", outlier_removal_method="RADIUS", statistical_mean_k="30",
                  statistical_stddev="1.2", radius_radius="0.5", radius_min_neighbors="2"),
}
IMU = np.array([0.02, -0.05, 0.6], np.float32)  # rad/s, as the IMU message gives it
TF = np.array([[0.99, -0.141, 0.0, 0.3], [0.141, 0.99, 0.0, -0.1], [0.0, 0.0, 1.0, 1.2], [0, 0, 0, 1]], np.float32)  # sensor -> base_link


def reference_params(ros, imu=None, tf=None, scan_period=None):
    """b2r_prefilter_params as PrefilteringNodelet's lines set them up: initialize_params (:50-99) for a rosparam dict, cloud_callback
    (:112-133) for the call: deskew only with an IMU message (:184-186), the distance filter always (:131)"""
    g = lambda k, d: ros.get(k, d)  # noqa: E731
    ds = g("downsample_method", "VOXELGRID")
    orm = g("outlier_removal_method", "STATISTICAL")
    p = dict(downsample_method={"VOXELGRID": 1, "APPROX_VOXELGRID": 2}.get(ds, 0),
             downsample_resolution=float(g("downsample_resolution", 0.1)),
             outlier_removal_method={"STATISTICAL": 1, "RADIUS": 2}.get(orm, 0),
             use_distance_filter=1, distance_near_thresh=float(g("distance_near_thresh", 1.0)),
             distance_far_thresh=float(g("distance_far_thresh", 100.0)))
    if orm == "STATISTICAL":
        p.update(statistical_mean_k=int(g("statistical_mean_k", 20)), statistical_stddev=float(g("statistical_stddev", 1.0)))
    if orm == "RADIUS":
        p.update(radius_radius=float(g("radius_radius", 0.8)), radius_min_neighbors=int(g("radius_min_neighbors", 2)))
    if imu is not None:
        p.update(deskewing=1, scan_period=float(scan_period if scan_period is not None else g("scan_period", 0.1)), angular_velocity=imu)
    if tf is not None:
        p.update(use_base_link_transform=1, base_link_transform=tf)
    return p


# ---------------------------------------------------------------------------------------------------------------- harness I/O
def _s(s):
    b = s.encode()
    return struct.pack("<i", len(b)) + b


def _kv(d):
    return struct.pack("<i", len(d)) + b"".join(_s(k) + _s(str(v)) for k, v in d.items())


def pcl_input(cloud, header=(7, 1234567890123, "velodyne"), width=None, height=1, is_dense=True):
    cloud = np.ascontiguousarray(cloud, np.float32)
    assert cloud.ndim == 2 and cloud.shape[1] == 8
    return ("pcl", header, cloud, cloud.shape[0] if width is None else width, height, is_dense)


def msg_input(m, header=(7, 1234567890123, "velodyne"), is_dense=False):
    return ("msg", header, m, is_dense)


def encode_call(kind, inp, set_params=None, imu=None, tf=None, want_filtered=True, want_inliers=True):
    b = _kv(set_params or {})
    seq, stamp, frame = inp[1]
    if inp[0] == "pcl":
        _, _, cloud, w, h, dense = inp
        b += struct.pack("<iIQ", 0, seq, stamp) + _s(frame) + struct.pack("<IIiq", w, h, int(dense), cloud.shape[0]) + cloud.tobytes()
    else:
        _, _, m, dense = inp
        b += struct.pack("<iIQ", 1, seq, stamp) + _s(frame)
        b += struct.pack("<IIIIii", m["width"], m["height"], m["point_step"], m["row_step"], int(m["is_bigendian"]), int(dense))
        b += struct.pack("<i", len(m["fields"])) + b"".join(_s(n) + struct.pack("<IiI", o, t, c) for n, o, t, c in m["fields"])
        b += struct.pack("<q", len(m["data"])) + bytes(m["data"])
    if kind == PREFILTER:
        b += struct.pack("<i3f", imu is not None, *(imu if imu is not None else np.zeros(3)))
        b += struct.pack("<i16f", tf is not None, *(np.asarray(tf, np.float32).T.reshape(16) if tf is not None else np.zeros(16)))
    else:
        b += struct.pack("<ii", int(want_filtered), int(want_inliers))
    return b


class _R:
    def __init__(self, b):
        self.b, self.o = b, 0

    def get(self, fmt):
        v = struct.unpack_from("<" + fmt, self.b, self.o)
        self.o += struct.calcsize("<" + fmt)
        return v if len(v) > 1 else v[0]

    def str(self):
        n = self.get("i")
        s = self.b[self.o:self.o + n].decode()
        self.o += n
        return s

    def cloud(self):
        if not self.get("i"):
            return None
        seq, stamp = self.get("I"), self.get("Q")
        frame = self.str()
        w, h, dense, n = self.get("IIiq")
        pts = np.frombuffer(self.b, np.uint32, count=n * 8, offset=self.o).reshape(n, 8).copy()
        self.o += n * 32
        return dict(header=(seq, stamp, frame), width=w, height=h, is_dense=bool(dense), bits=pts)


def decode_call(kind, b):
    r = _R(b)
    status = r.get("i")
    if status != OK:
        return dict(status=status, error=r.str())
    if kind == PREFILTER:
        return dict(status=OK, cloud=r.cloud())
    has, coeffs = r.get("i"), np.array(r.get("4f"), np.float32)
    res = _capi.FloorResult.from_buffer_copy(r.b[r.o:r.o + C.sizeof(_capi.FloorResult)])
    r.o += C.sizeof(_capi.FloorResult)
    return dict(status=OK, coeffs=coeffs if has else None, result=res, filtered=r.cloud(), inliers=r.cloud())


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    from hdl_graph_slam_b200 import build
    build.build_engine()
    exe = str(tmp_path_factory.mktemp("frontend") / "frontend_harness")
    lib = os.path.join(ROOT, "hdl_graph_slam_b200", "_lib")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++14", "-O1", "-Wall", "-pthread",
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "hdl_graph_slam_b200", "adapter"), "-o", exe,
                           os.path.join(ROOT, "tests", "frontend_harness.cpp"), "-L", lib, "-lb200reg", "-Wl,-rpath," + lib])
    return exe


def run_jobs(harness, tmp_path, jobs, mode="serial"):
    """jobs: [(kind, rosparams, [encoded calls])] -> [[decoded answers]] per job"""
    body = struct.pack("<i", len(jobs)) + b"".join(struct.pack("<i", k) + _kv(p) + struct.pack("<i", len(c)) + b"".join(c) for k, p, c in jobs)
    src, dst = tmp_path / f"in_{mode}.bin", tmp_path / f"out_{mode}.bin"
    src.write_bytes(body)
    out = subprocess.run([harness, str(src), str(dst), mode], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr
    b = dst.read_bytes()
    o, answers = 0, []
    for kind, _, calls in jobs:
        (n,) = struct.unpack_from("<q", b, o)
        o += 8
        blk, p, got = b[o:o + n], 0, []
        o += n
        for _ in calls:
            (m,) = struct.unpack_from("<q", blk, p)
            got.append(decode_call(kind, blk[p + 8:p + 8 + m]))
            p += 8 + m
        answers.append(got)
    assert o == len(b)
    return answers


@pytest.fixture(scope="module")
def reg():
    r = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    yield r
    r.close()


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same_cloud(x, y):
    if x is None or y is None:
        return x is None and y is None
    return all(x[k] == y[k] for k in ("header", "width", "height", "is_dense")) and np.array_equal(x["bits"], y["bits"])


def same_answer(a, b):
    """two decoded harness answers, bit for bit"""
    if a["status"] != b["status"]:
        return False
    if a["status"] != OK:
        return a["error"] == b["error"]
    if "cloud" in a:
        return same_cloud(a["cloud"], b["cloud"])
    coeffs_same = (a["coeffs"] is None and b["coeffs"] is None) or (
        a["coeffs"] is not None and b["coeffs"] is not None and np.array_equal(u32(a["coeffs"]), u32(b["coeffs"])))
    return coeffs_same and bytes(a["result"]) == bytes(b["result"]) and same_cloud(a["filtered"], b["filtered"]) and same_cloud(a["inliers"], b["inliers"])


def direct(reg, cloud, p):
    out, _, m = reg.prefilter(cloud, **p)
    return u32(out[:m])


# ---------------------------------------------------------------------------------------------------------------- prefilter
@pytest.mark.parametrize("launch", sorted(PREFILTER_LAUNCH))
def test_prefilter_launch_sets(harness, tmp_path, reg, synth, launch):
    ros = PREFILTER_LAUNCH[launch]
    sensor = "kitti" if launch == "kitti" else "vlp16"
    clouds = [synth.scan(sensor, frame=f, stride=8) for f in (0, 1)]
    variants = [(None, None), (IMU, None), (None, TF), (IMU, TF)]
    calls = [encode_call(PREFILTER, pcl_input(c, header=(3 + i, 1000 + i, "velodyne"), is_dense=True), imu=w, tf=t)
             for i, (c, (w, t)) in enumerate((c, v) for c in clouds for v in variants)]
    (got,) = run_jobs(harness, tmp_path, [(PREFILTER, ros, calls)])
    i = 0
    for c in clouds:
        for w, t in variants:
            g = got[i]
            assert g["status"] == OK
            want = direct(reg, c, reference_params(ros, w, t))
            assert np.array_equal(g["cloud"]["bits"], want), (launch, i)
            frame = ros.get("base_link_frame", "") if t is not None else "velodyne"
            assert g["cloud"]["header"] == (3 + i, 1000 + i, frame)
            assert (g["cloud"]["width"], g["cloud"]["height"]) == (want.shape[0], 1)
            assert g["cloud"]["is_dense"] == (ros.get("downsample_method", "VOXELGRID") == "VOXELGRID")
            i += 1


NAMES = [(d, o) for d in ("VOXELGRID", "APPROX_VOXELGRID", "NONE", "voxelgrid") for o in ("STATISTICAL", "RADIUS", "NONE", "OUTLIER")]


def test_prefilter_every_method_name(harness, tmp_path, reg, synth):
    """every downsample and outlier name, unknown names (read as NONE) included, with non-default parameters"""
    c = synth.scan("vlp16", frame=2, stride=8)
    jobs = []
    for d, o in NAMES:
        ros = dict(downsample_method=d, downsample_resolution="0.2", outlier_removal_method=o, statistical_mean_k="12",
                   statistical_stddev="0.8", radius_radius="0.6", radius_min_neighbors="3", distance_near_thresh="2.0", distance_far_thresh="40.0")
        jobs.append((PREFILTER, ros, [encode_call(PREFILTER, pcl_input(c), imu=IMU)]))
    answers = run_jobs(harness, tmp_path, jobs)
    seen = set()
    for (d, o), ((_, ros, _), (g,)) in zip(NAMES, zip(jobs, answers)):
        want = direct(reg, c, reference_params(ros, IMU))
        assert np.array_equal(g["cloud"]["bits"], want), (d, o)
        assert g["cloud"]["is_dense"] == (d == "VOXELGRID")
        seen.add(want.shape[0])
    assert len(seen) > 6  # the names select different filters


def test_use_distance_filter_false_still_filters(harness, tmp_path, reg, synth):
    c = synth.scan("vlp16", frame=0, stride=8)
    ros = dict(use_distance_filter="false", distance_near_thresh="5.0", distance_far_thresh="30.0", downsample_method="NONE",
               outlier_removal_method="NONE")
    ((g,),) = run_jobs(harness, tmp_path, [(PREFILTER, ros, [encode_call(PREFILTER, pcl_input(c))])])
    norm = np.linalg.norm(c[:, :3], axis=1)
    keep = (norm > 5.0) & (norm < 30.0)
    assert 0 < keep.sum() < c.shape[0]
    assert np.array_equal(g["cloud"]["bits"], u32(c[keep]))
    assert not g["cloud"]["is_dense"]


def test_scan_period_is_read_at_every_deskew(harness, tmp_path, reg, synth):
    c = synth.scan("vlp16", frame=1, stride=8)
    ros = dict(downsample_method="NONE", outlier_removal_method="NONE", scan_period="0.1")
    calls = [encode_call(PREFILTER, pcl_input(c), imu=IMU), encode_call(PREFILTER, pcl_input(c), set_params={"scan_period": "0.35"}, imu=IMU),
             encode_call(PREFILTER, pcl_input(c), imu=None)]
    ((a, b, n),) = run_jobs(harness, tmp_path, [(PREFILTER, ros, calls)])
    assert np.array_equal(a["cloud"]["bits"], direct(reg, c, reference_params(ros, IMU, scan_period=0.1)))
    assert np.array_equal(b["cloud"]["bits"], direct(reg, c, reference_params(ros, IMU, scan_period=0.35)))
    assert not np.array_equal(a["cloud"]["bits"], b["cloud"]["bits"])
    assert np.array_equal(n["cloud"]["bits"], direct(reg, c, reference_params(ros)))


@pytest.mark.parametrize("sensor,launch", [("vlp16", "400"), ("kitti", "kitti")])
def test_prefilter_equals_the_oracle_chain(harness, tmp_path, synth, oracle, sensor, launch):
    ros = PREFILTER_LAUNCH[launch]
    c = synth.scan(sensor, frame=0, stride=8)
    ((g,),) = run_jobs(harness, tmp_path, [(PREFILTER, ros, [encode_call(PREFILTER, pcl_input(c))])])
    keep = oracle.distance_filter(c, float(ros["distance_near_thresh"]), float(ros["distance_far_thresh"]))
    d = c[keep]
    v = oracle.voxelgrid(d, float(ros["downsample_resolution"]))[0]
    full = np.zeros((v.shape[0], 8), np.float32)
    full[:, :3], full[:, 3], full[:, 4] = v[:, :3], 1.0, v[:, 3]
    full = full[oracle.radius_outlier(full, float(ros["radius_radius"]), int(ros["radius_min_neighbors"]))]
    got = g["cloud"]["bits"].view(np.float32)
    assert got.shape[0] == full.shape[0]
    assert np.array_equal(u32(got[:, :3]), u32(full[:, :3])) and np.array_equal(u32(got[:, 4]), u32(full[:, 4]))


def test_empty_inputs_give_nullptr(harness, tmp_path, synth):
    empty = np.zeros((0, 8), np.float32)
    m = message(np.zeros((0, 4), np.float32), width=0)
    calls = [encode_call(PREFILTER, pcl_input(empty), imu=IMU, tf=TF), encode_call(PREFILTER, msg_input(m), imu=IMU, tf=TF)]
    ((a, b),) = run_jobs(harness, tmp_path, [(PREFILTER, {}, calls)])
    assert a["status"] == OK and a["cloud"] is None and b["status"] == OK and b["cloud"] is None


# ---------------------------------------------------------------------------------------------------------------- PointCloud2
def with_nans(cloud, frac, seed):
    c = cloud.copy()
    rows = np.random.default_rng(seed).random(c.shape[0]) < frac
    c[rows, :3] = np.nan
    return c


def xyzi(c):
    return np.ascontiguousarray(np.column_stack([c[:, :3], c[:, 4]]), np.float32)


def decoded_cloud(m):
    lay = layout_of(m["fields"], m["point_step"], m["is_bigendian"])
    return as_cloud(decode_rows(m["data"], m["width"], m["height"], m["row_step"], lay))


def message_cases(synth):
    v = synth.scan("vlp16", frame=3, stride=8)
    o64 = with_nans(synth.scan((64, 1024), frame=4, stride=8), 0.1, 1)
    o128 = with_nans(np.concatenate([synth.scan((64, 10240), frame=f, stride=8) for f in (5, 6)]), 0.05, 2)
    return {
        "velodyne": message(xyzi(v), "velodyne"),
        "ouster64": message(xyzi(o64), "ouster", width=1024, height=64),
        "ouster128_1.3M": message(xyzi(o128), "ouster", width=10240, height=128),
        "big_endian": message(xyzi(v), "velodyne", big=True),
        "padded": message(xyzi(o64), "ouster", width=1024, height=64, pad=24),
        "padded_big_endian_uint8": message(xyzi(o64), "velodyne", width=1024, height=64, pad=7, big=True, intensity="uint8"),
        "no_intensity_padded": message(xyzi(v), "velodyne", width=v.shape[0] // 16, height=16, pad=2, intensity="none"),
    }


def test_pointcloud2_overloads_equal_the_pcl_overloads(harness, tmp_path, synth):
    cases = message_cases(synth)
    ros = PREFILTER_LAUNCH["400"]
    fl = {k: str(v) for k, v in FLOOR_LAUNCH["hdl"].items()}
    fl["use_normal_filtering"] = "true"
    pf_calls, fd_calls = [], []
    for name, m in cases.items():
        c = decoded_cloud(m)
        hdr = (11, 1_600_000_000_250_000, "os_sensor")
        pf_calls += [encode_call(PREFILTER, msg_input(m, hdr), imu=IMU, tf=TF),
                     encode_call(PREFILTER, pcl_input(c, hdr, width=m["width"], height=m["height"], is_dense=False), imu=IMU, tf=TF)]
        fd_calls += [encode_call(FLOOR, msg_input(m, hdr)), encode_call(FLOOR, pcl_input(c, hdr, m["width"], m["height"], is_dense=False))]
    pf, fd = run_jobs(harness, tmp_path, [(PREFILTER, ros, pf_calls), (FLOOR, fl, fd_calls)])
    for k, name in enumerate(cases):
        a, b = pf[2 * k], pf[2 * k + 1]
        assert a["status"] == OK and same_answer(a, b), name
        assert a["cloud"]["header"] == (11, 1_600_000_000_250_000, "base_link") and a["cloud"]["bits"].shape[0] > 0
        a, b = fd[2 * k], fd[2 * k + 1]
        assert a["status"] == OK and same_answer(a, b), name


def test_message_without_float32_xyz_is_refused(harness, tmp_path, synth):
    v = synth.scan("vlp16_16k", frame=0, stride=8)
    m = message(xyzi(v), "velodyne")
    m["fields"] = [(n, o, 8 if n == "z" else t, c) for n, o, t, c in m["fields"]]  # z as FLOAT64
    short = message(xyzi(v), "velodyne", width=v.shape[0] // 16, height=16)
    short["row_step"] -= 1  # shorter than width * point_step
    ((a, b),) = run_jobs(harness, tmp_path, [(PREFILTER, {}, [encode_call(PREFILTER, msg_input(m)), encode_call(PREFILTER, msg_input(short))])])
    assert a["status"] == INVALID_ARGUMENT and "x, y and z" in a["error"]
    assert b["status"] == RUNTIME_ERROR and "row_step" in b["error"]


def readback(r, ptr, n):
    from cuda.bindings import runtime as cudart
    r.synchronize()
    out = np.empty((n, 8), np.uint32)
    if n:
        err, = cudart.cudaMemcpy(out.ctypes.data, ptr, out.nbytes, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
        assert int(err) == 0
    return out


def test_ingest_rows_equals_contiguous_ingest(reg, synth):
    cases = message_cases(synth)
    for name, m in cases.items():
        lay = layout_of(m["fields"], m["point_step"], m["is_bigendian"])
        n = m["width"] * m["height"]
        rows = readback(reg, reg.ingestPointCloud2Rows(m["data"], m["width"], m["height"], m["row_step"], **lay), n)
        assert np.array_equal(rows, decode_rows(m["data"], m["width"], m["height"], m["row_step"], lay)), name
        if m["row_step"] == m["width"] * m["point_step"]:  # contiguous: the same bits as the contiguous entry point
            flat = readback(reg, reg.ingestPointCloud2(m["data"], n, **lay), n)
            assert np.array_equal(rows, flat), name
            one = readback(reg, reg.ingestPointCloud2Rows(m["data"], n, 1, n * m["point_step"], **lay), n)  # height 1
            assert np.array_equal(one, flat), name
            assert np.array_equal(flat, decode_pointcloud2(m["data"], n, lay)), name


def test_ingest_rows_refuses_a_short_row_step_and_accepts_empty(reg):
    lay = dict(point_step=16, off_x=0, off_y=4, off_z=8, off_intensity=12, intensity_datatype=FLOAT32, is_bigendian=False)
    data = np.zeros(4 * 64, np.uint8)
    with pytest.raises(Exception) as e:
        reg.ingestPointCloud2Rows(data, 4, 4, 63, **lay)
    assert getattr(e.value, "code", None) == _capi.B2R_EINVAL and "row_step" in str(e.value)
    assert reg.ingestPointCloud2Rows(data, 0, 4, 0, **lay) is None
    assert reg.ingestPointCloud2Rows(data, 4, 0, 64, **lay) is None


# ---------------------------------------------------------------------------------------------------------------- floor
@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("floor_ref"))


def prefiltered(reg, synth, sensor):
    raw = synth.scan(sensor, frame=0, stride=8)
    res = 0.25 if sensor == "kitti" else 0.1
    out, _, m = reg.prefilter(raw, use_distance_filter=1, distance_near_thresh=0.1, distance_far_thresh=100.0, downsample_method=1,
                              downsample_resolution=res, outlier_removal_method=2, radius_radius=0.5, radius_min_neighbors=2)
    return np.ascontiguousarray(out[:m])


def floor_ros(launch, **kw):
    d = dict(FLOOR_LAUNCH[launch], **kw)
    return {k: ("true" if v else "false") if k == "use_normal_filtering" else str(v) for k, v in d.items()}


def floor_kw(ros):
    return dict(tilt_deg=float(ros["tilt_deg"]), sensor_height=float(ros["sensor_height"]), height_clip_range=float(ros["height_clip_range"]),
                floor_pts_thresh=int(ros["floor_pts_thresh"]), use_normal_filtering=int(ros["use_normal_filtering"] == "true"),
                floor_normal_thresh=float(ros.get("floor_normal_thresh", 10.0)), normal_filter_thresh=float(ros["normal_filter_thresh"]))


def check_floor(g, direct_res, want, header, want_filtered=True, want_inliers=True, empty_msg=False):
    assert g["status"] == OK
    r = g["result"]
    assert r.detected == direct_res["detected"] and r.reason == _capi.FLOOR_REASONS.index(direct_res["reason"])
    for k in ("n_filtered", "n_inliers", "ransac_iterations"):
        assert getattr(r, k) == direct_res[k], k
    assert tuple(r.model_indices) == direct_res["model_indices"]
    assert np.array_equal(u32(r.coeffs[:]), u32(direct_res["coeffs"]))
    assert (g["coeffs"] is not None) == direct_res["detected"]
    if g["coeffs"] is not None:
        assert np.array_equal(u32(g["coeffs"]), u32(direct_res["coeffs"]))
    got = {"detected": bool(r.detected), "reason": _capi.FLOOR_REASONS[r.reason], "coeffs": np.array(r.coeffs[:], np.float32),
           "n_filtered": r.n_filtered, "n_inliers": r.n_inliers, "ransac_iterations": r.ransac_iterations,
           "model_indices": tuple(r.model_indices), "filtered": direct_res["filtered"], "inliers": direct_res["inliers"]}
    if want is not None:
        assert_same(got, want)
    if want_filtered and not empty_msg:
        f = g["filtered"]
        assert f is not None and f["header"] == header and (f["width"], f["height"]) == (r.n_filtered, 1)
        assert np.array_equal(f["bits"], u32(direct_res["filtered"]))
        if want is not None:
            assert_same(dict(got, filtered=f["bits"].view(np.float32)), want)
    else:
        assert g["filtered"] is None
    if want_inliers and r.detected:
        i = g["inliers"]
        assert i is not None and i["header"] == header and (i["width"], i["height"]) == (r.n_inliers, 1)
        assert np.array_equal(i["bits"], u32(direct_res["inliers"]))
        if want is not None:
            assert_same(dict(got, inliers=i["bits"].view(np.float32)), want)
    else:
        assert g["inliers"] is None


@pytest.mark.parametrize("sensor", ["vlp16", "hdl32e", "kitti"])
@pytest.mark.parametrize("launch", ["hdl", "501", "kitti"])
def test_floor_detector_on_prefiltered_scans(harness, tmp_path, reg, ref, synth, sensor, launch):
    c = prefiltered(reg, synth, sensor)
    ros = floor_ros(launch)
    hdr = (5, 42_000_001, "base_link")
    m = message(xyzi(c), "velodyne")
    calls = [encode_call(FLOOR, pcl_input(c, hdr, is_dense=False)), encode_call(FLOOR, pcl_input(c, hdr), want_inliers=False),
             encode_call(FLOOR, pcl_input(c, hdr), want_filtered=False), encode_call(FLOOR, msg_input(m, hdr))]
    ((a, b, d, e),) = run_jobs(harness, tmp_path, [(FLOOR, ros, calls)])
    kw = floor_kw(ros)
    direct_res = reg.floor_detect(c, **kw)
    want = ref.detect(c, **kw)
    check_floor(a, direct_res, want, hdr)
    check_floor(b, direct_res, None, hdr, want_inliers=False)
    check_floor(d, direct_res, None, hdr, want_filtered=False)
    check_floor(e, direct_res, want, hdr)
    assert not a["filtered"]["is_dense"]  # normal filtering or the input's flag (false)
    if ros["use_normal_filtering"] == "false":
        assert b["filtered"]["is_dense"]  # the plane clips keep the input's flag


def test_floor_gates_and_empty_inputs(harness, tmp_path, reg, ref, synth):
    c = prefiltered(reg, synth, "vlp16")
    hdr = (1, 2, "base_link")
    empty = np.zeros((0, 8), np.float32)
    cases = [("size_gate", floor_ros("hdl", floor_pts_thresh=10 ** 7), c, "TOO_FEW_FILTERED"),
             ("not_vertical", floor_ros("hdl", tilt_deg=40.0, use_normal_filtering=False, height_clip_range=30.0, floor_normal_thresh=5.0), c,
              "NOT_VERTICAL"),
             ("inlier_gate", floor_ros("hdl", use_normal_filtering=False, height_clip_range=30.0, floor_pts_thresh=int(c.shape[0] * 0.95)), c, "TOO_FEW_INLIERS")]
    jobs = [(FLOOR, ros, [encode_call(FLOOR, pcl_input(x, hdr))]) for _, ros, x, _ in cases]
    jobs.append((FLOOR, floor_ros("hdl"), [encode_call(FLOOR, pcl_input(empty, hdr)), encode_call(FLOOR, msg_input(message(np.zeros((0, 4), np.float32), width=0), hdr))]))
    answers = run_jobs(harness, tmp_path, jobs)
    for (name, ros, x, reason), (g,) in zip(cases, answers[:-1]):
        kw = floor_kw(ros)
        direct_res = reg.floor_detect(x, **kw)
        if reason is not None:
            assert direct_res["reason"] == reason, (name, direct_res["reason"])
        assert not direct_res["detected"], name
        check_floor(g, direct_res, ref.detect(x, **kw), hdr)
    pcl_empty, msg_empty = answers[-1]
    assert pcl_empty["coeffs"] is None and _capi.FLOOR_REASONS[pcl_empty["result"].reason] == "EMPTY_INPUT"
    assert pcl_empty["filtered"]["bits"].shape == (0, 8) and pcl_empty["inliers"] is None  # detect() on an empty cloud publishes it
    assert msg_empty["coeffs"] is None and _capi.FLOOR_REASONS[msg_empty["result"].reason] == "EMPTY_INPUT"
    assert msg_empty["filtered"] is None and msg_empty["inliers"] is None  # cloud_callback returns before detect (:76-78)


# ---------------------------------------------------------------------------------------------------------------- threads
def test_prefilter_and_floor_detector_on_two_threads(harness, tmp_path, synth):
    raws = [synth.scan("hdl32e", frame=f, stride=8) for f in range(3)]
    ros = PREFILTER_LAUNCH["501"]
    pf_calls = [encode_call(PREFILTER, pcl_input(r), imu=IMU, tf=TF) for r in raws]
    pf_calls += [encode_call(PREFILTER, msg_input(message(xyzi(r), "velodyne"))) for r in raws]
    fd_calls = [encode_call(FLOOR, msg_input(message(xyzi(r), "ouster", width=r.shape[0] // 32, height=32, pad=8))) for r in raws]
    fd_calls += [encode_call(FLOOR, pcl_input(r)) for r in raws]
    jobs = [(PREFILTER, ros, pf_calls), (FLOOR, floor_ros("501"), fd_calls)]
    serial = run_jobs(harness, tmp_path, jobs, "serial")
    concurrent = run_jobs(harness, tmp_path, jobs, "concurrent")
    for s, c in zip(serial, concurrent):
        for a, b in zip(s, c):
            assert a["status"] == OK and same_answer(a, b)
