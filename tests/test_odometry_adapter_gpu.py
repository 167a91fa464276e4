"""GPU: the odometry drop-in (adapter/b200_odometry.hpp) EXECUTED through tests/odometry_harness.cpp and the test-only stand-ins, the
way ScanMatchingOdometryNodelet calls it.

- Against the raw mirror: walks of 48 frames (keyframe switches, far jumps that thresholding rejects, msf_delta guesses) under the
  code defaults and the odometry rosparams of launch/hdl_graph_slam{,_400,_501,_kitti}.launch, on FAST_GICP, NDT_OMP and NDT handles,
  with downsample NONE / VOXELGRID / APPROX_VOXELGRID, thresholding on and off: every pose, decision and status is bit for bit
  b2r_odometry_matching given parameters built here from the reference lines (scan_matching_odometry_nodelet.cpp:65-107).
- Against the reference walk: tests/odometry_ref.py's replay with roscpp's delta_time rule, on sec / nsec stamps placed where the
  double rule decides differently; the double entry point switches its keyframe one frame later.  Mixing the two stamp forms on one
  odometry follows b200reg.h's rule.
- PointCloud2 input (velodyne-style of varying size, organized with NaN records, padded rows): bitwise the pcl overload over whole walks,
  the first frame the target of a FAST_GICP handle under NONE.
- aligned(): bit for bit a numpy restatement of pcl::transformPointCloud under odom, on dense and non-dense clouds with NaN / inf
  records; nullptr on first and rejected frames.
- want_status toggled per frame gives the always-on poses and, where asked, the publish_status = 1 status.
- An odometry and a prefilter on two threads give the serial answers."""
import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg
import odometry_ref
from frontend_ref import decode_rows, layout_of, message
from odometry_adapter_io import ODOMETRY, PREFILTER, build_harness, encode_call, msg_input, pcl_input, run_jobs

pytestmark = pytest.mark.gpu

REG = dict(registration_method="FAST_GICP", reg_num_threads="0", reg_maximum_iterations="64", reg_max_optimizer_iterations="20",
           reg_use_reciprocal_correspondences="false", reg_correspondence_randomness="20", reg_resolution="1.0",
           reg_nn_search_method="DIRECT7")
# the odometry nodelet's <param> lines of each launch file; "defaults" sets none
LAUNCH = {
    "defaults": {},
    "hdl": dict(REG, odom_frame_id="odom", keyframe_delta_trans="1.0", keyframe_delta_angle="1.0", keyframe_delta_time="10000.0",
                transform_thresholding="false", max_acceptable_trans="1.0", max_acceptable_angle="1.0", downsample_method="NONE",
                downsample_resolution="0.1", reg_transformation_epsilon="0.01", reg_max_correspondence_distance="2.5"),
    "400": dict(REG, odom_frame_id="odom", keyframe_delta_trans="1.0", keyframe_delta_angle="1.0", keyframe_delta_time="10000.0",
                transform_thresholding="false", max_acceptable_trans="1.0", max_acceptable_angle="1.0", downsample_method="NONE",
                downsample_resolution="0.1", reg_transformation_epsilon="0.1", reg_max_correspondence_distance="2.0"),
    "501": dict(REG, odom_frame_id="odom", keyframe_delta_trans="0.25", keyframe_delta_angle="1.0", keyframe_delta_time="10000.0",
                transform_thresholding="false", max_acceptable_trans="1.0", max_acceptable_angle="1.0", downsample_method="NONE",
                downsample_resolution="0.1", reg_transformation_epsilon="0.1", reg_max_correspondence_distance="2.0"),
    "kitti": dict(REG, odom_frame_id="odom", keyframe_delta_trans="5.0", keyframe_delta_angle="2.0", keyframe_delta_time="10000.0",
                  transform_thresholding="false", max_acceptable_trans="1.0", max_acceptable_angle="1.0", downsample_method="NONE",
                  reg_transformation_epsilon="0.1", reg_max_correspondence_distance="2.0"),
}
BASE_NS = 1436939143126614242
N_FRAMES = 48
JUMPS = (15, 31)  # these frames get the scan 25 frames (7.5 m) ahead: thresholding rejects them
MSF = np.array([[1, 0, 0, 0.3], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float32)  # an msf_delta guess on every fifth frame


def stamp(ns):
    return (ns // 1_000_000_000, ns % 1_000_000_000)


def to_sec(st):
    return float(st[0]) + 1e-9 * float(st[1])  # ros::Time::toSec()


def walk_stamps(n=N_FRAMES, period_ns=97_300_000):
    """97.3 ms apart: no difference lands within a microsecond of any keyframe_delta_time used here, so the ROS and double rules agree"""
    return [stamp(BASE_NS + k * period_ns) for k in range(n)]


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return build_harness(tmp_path_factory.mktemp("odometry") / "odometry_harness")


@pytest.fixture(scope="module")
def frames(synth):
    out = [synth.scan("vlp16_16k", frame=k, step=0.3, stride=8) for k in range(N_FRAMES)]
    for j in JUMPS:
        out[j] = synth.scan("vlp16_16k", frame=j + 25, step=0.3, stride=8)
    return out


def raw_params(ros):
    """b2r_odometry_params as initialize_params (:65-107) sets them up for a rosparam dict"""
    g = lambda k, d: ros.get(k, d)  # noqa: E731
    ds = g("downsample_method", "VOXELGRID")
    return dict(keyframe_delta_trans=float(g("keyframe_delta_trans", 0.25)), keyframe_delta_angle=float(g("keyframe_delta_angle", 0.15)),
                keyframe_delta_time=float(g("keyframe_delta_time", 1.0)), transform_thresholding=g("transform_thresholding", "false") == "true",
                max_acceptable_trans=float(g("max_acceptable_trans", 1.0)), max_acceptable_angle=float(g("max_acceptable_angle", 1.0)),
                downsample_method={"VOXELGRID": pkg.B2R_DOWNSAMPLE_VOXELGRID, "APPROX_VOXELGRID": pkg.B2R_DOWNSAMPLE_APPROX_VOXELGRID}.get(ds, 0),
                downsample_resolution=float(g("downsample_resolution", 0.1)))


def reg_params(ros):
    return {k: v for k, v in ros.items() if k == "registration_method" or k.startswith("reg_")}


def raw_walk(ros, clouds, stamps, msf=None, ros_stamps=False):
    """b2r_odometry_matching (publish_status = 1) with the doubles toSec(stamp), or b2r_odometry_matching_ros"""
    reg = pkg.select_registration_method(reg_params(ros))
    odo = pkg.ScanMatchingOdometry(reg, publish_status=True, **raw_params(ros))
    out = []
    for k, (c, st) in enumerate(zip(clouds, stamps)):
        d = None if msf is None else msf(k)
        out.append(odo.matching_ros(st[0], st[1], c, d, want_status=True) if ros_stamps else odo.matching(to_sec(st), c, d))
        out[-1]["aligned_raw"] = None if k == 0 or out[-1]["frame_rejected"] else odo.aligned(c.shape[0], 32)
    odo.close()
    reg.close()
    return out


def msf_every_fifth(k):
    return MSF if k % 5 == 4 else None


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32).tobytes()


def aligned_ref(cloud, odom, is_dense):
    """pcl::transformPointCloud(*cloud, *aligned, odom) as the engine states it: record copied, x y z = ((m0 x + m1 y) + m2 z) + m3 in
    float32 (numpy rounds every operation), 1.0f at float 3; a non-dense cloud's records with a non-finite x, y or z stay as they are"""
    f = np.array(cloud, np.float32).reshape(-1, 8)
    M = np.asarray(odom, np.float32)
    x, y, z = f[:, 0].copy(), f[:, 1].copy(), f[:, 2].copy()
    keep = np.ones(len(f), bool) if is_dense else (np.isfinite(x) & np.isfinite(y) & np.isfinite(z))
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(3):
            v = ((M[r, 0] * x + M[r, 1] * y) + M[r, 2] * z) + M[r, 3]
            f[keep, r] = v[keep]
    f[keep, 3] = np.float32(1.0)
    return f


def assert_aligned(got_bits, cloud, odom, is_dense):
    want = aligned_ref(cloud, odom, is_dense)
    got = got_bits.view(np.float32).reshape(-1, 8)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)  # the NaN a product of inf and 0 makes has no fixed payload
    assert np.array_equal(got.view(np.uint32)[~nan], want.view(np.uint32)[~nan])


def assert_walk(ans, raw, clouds, ros, want_status, want_aligned, is_dense=True, widths=None):
    kp = np.eye(4, dtype=np.float32)
    for k, (a, r) in enumerate(zip(ans, raw)):
        assert not isinstance(a, tuple), (k, a)
        assert bits(a["odom"]) == bits(r["odom"]), k
        assert (a["keyframe_updated"], a["frame_rejected"]) == (r["keyframe_updated"], r["frame_rejected"]), k
        assert bits(a["keyframe_pose"]) == bits(kp), k  # :238, before this frame's switch
        if a["keyframe_updated"]:
            kp = a["odom"]
        if want_status(k) and k > 0:
            assert a["converged"] == r["converged"] and bits(a["trans"]) == bits(r["trans"]), k
            assert np.float64(a["matching_error"]).tobytes() == np.float64(r["matching_error"]).tobytes(), k
            assert np.float32(a["inlier_fraction"]).tobytes() == np.float32(r["inlier_fraction"]).tobytes(), k
        if not want_aligned(k) or k == 0 or a["frame_rejected"]:
            assert a["aligned"] is None, k
            continue
        al = a["aligned"]
        assert al["header"][2] == ros.get("odom_frame_id", "odom") and al["is_dense"] == is_dense, k
        assert (al["width"], al["height"]) == ((clouds[k].shape[0], 1) if widths is None else widths[k]), k
        assert_aligned(al["bits"], clouds[k], a["odom"], is_dense)
        if r.get("aligned_raw") is not None and is_dense:
            assert al["bits"].tobytes() == r["aligned_raw"].view(np.uint32).tobytes(), k  # b2r_odometry_aligned through Python


WALKS = [  # (registration_method, launch set, downsample_method, transform_thresholding)
    ("FAST_GICP", "defaults", None, True),
    ("FAST_GICP", "hdl", "NONE", False),
    ("FAST_GICP", "400", "VOXELGRID", True),
    ("FAST_GICP", "501", "APPROX_VOXELGRID", False),
    ("FAST_GICP", "kitti", "NONE", True),
    ("NDT_OMP", "hdl", "NONE", True),
    ("NDT_OMP", "501", "VOXELGRID", False),
    ("NDT", "400", "APPROX_VOXELGRID", True),
    ("NDT", "kitti", "NONE", False),
]


def walk_ros(method, launch, downsample, thresholding):
    ros = dict(LAUNCH[launch])
    ros["registration_method"] = method
    if downsample is not None:
        ros["downsample_method"] = downsample
    if thresholding:
        ros.update(transform_thresholding="true", max_acceptable_trans="0.5")
    return ros


@pytest.mark.parametrize("method,launch,downsample,thresholding", WALKS)
def test_walk_equals_the_raw_mirror(harness, tmp_path, frames, method, launch, downsample, thresholding):
    ros = walk_ros(method, launch, downsample, thresholding)
    stamps = walk_stamps()
    calls = [encode_call(ODOMETRY, pcl_input(c), st, msf=msf_every_fifth(k)) for k, (c, st) in enumerate(zip(frames, stamps))]
    ((ans,), _) = run_jobs(harness, tmp_path, [(ODOMETRY, ros, calls)])
    raw = raw_walk(ros, frames, stamps, msf_every_fifth)
    assert_walk(ans, raw, frames, ros, lambda k: True, lambda k: True)
    # the NDT handles' steps on these scans are too short to be sure of a switch or a rejection; kitti's keyframes are 5 m apart
    if method == "FAST_GICP":
        assert sum(a["keyframe_updated"] for a in ans) >= (1 if launch == "kitti" else 2)
        if thresholding:
            assert any(a["frame_rejected"] for a in ans)


# ---- roscpp's delta_time against the reference replay
def ros_stamps_near_threshold(n=40):
    """frames 100 ms apart, except that frame 10 is 1.000000207 s after frame 0 (1436939143.126614242 -> 1436939144.126614449): more
    than keyframe_delta_time = 1.0, while the two stamps as doubles differ by exactly 1.0"""
    ns = [BASE_NS + k * 100_000_000 for k in range(10)]
    t10 = BASE_NS + 1_000_000_207
    ns += [t10 + (k - 10) * 100_000_000 for k in range(10, n)]
    return [stamp(t) for t in ns]


def ros_wants_keyframe(trans, stamp_, keyframe_stamp, keyframe_delta_trans, keyframe_delta_angle, keyframe_delta_time):
    """odometry_ref.wants_keyframe with :243's (stamp - keyframe_stamp).toSec() on ros::Time stamps (sec, nsec), in Python integers"""
    dt, da = odometry_ref.norm3(trans), odometry_ref.angle(trans)
    s, ns = stamp_[0] - keyframe_stamp[0], stamp_[1] - keyframe_stamp[1]
    s += ns // 1_000_000_000
    ns %= 1_000_000_000
    dtime = float(s) + 1e-9 * float(ns)
    return (dt > keyframe_delta_trans) | (da > keyframe_delta_angle) | (dtime > keyframe_delta_time), dt, da, dtime


def engine_align(params):
    reg = pkg.select_registration_method(params)

    def align(cloud, target, guess):
        reg.setInputTarget(target)
        reg.setInputSource(cloud)
        reg.align(guess)
        return dict(T=reg.getFinalTransformation(), converged=reg.hasConverged(), iterations=reg.nr_iterations)
    return reg, align


@pytest.mark.parametrize("method", ["FAST_GICP", "NDT_OMP"])
def test_ros_rule_matches_the_reference_replay(harness, tmp_path, frames, monkeypatch, method):
    ros = dict(LAUNCH["hdl"], registration_method=method, keyframe_delta_trans="1000000.0", keyframe_delta_angle="1000000.0",
               keyframe_delta_time="1.0")
    clouds = [frames[k] if k not in JUMPS else frames[k - 1] for k in range(40)]
    stamps = ros_stamps_near_threshold(len(clouds))
    calls = [encode_call(ODOMETRY, pcl_input(c), st) for c, st in zip(clouds, stamps)]
    ((ans,), _) = run_jobs(harness, tmp_path, [(ODOMETRY, ros, calls)])
    reg, align = engine_align(reg_params(ros))
    monkeypatch.setattr(odometry_ref, "wants_keyframe", ros_wants_keyframe)
    rep = odometry_ref.Replay(align, **raw_params(ros))
    want = [rep.matching(st, c) for c, st in zip(clouds, stamps)]
    reg.close()
    assert [a["keyframe_updated"] for a in ans] == [bool(w["keyframe_updated"]) for w in want]
    assert [a["frame_rejected"] for a in ans] == [bool(w["frame_rejected"]) for w in want]
    for k, (a, w) in enumerate(zip(ans, want)):
        assert np.allclose(a["odom"], w["odom"], atol=1e-4), k
    assert ans[10]["keyframe_updated"] and not ans[11]["keyframe_updated"]
    # the raw sec / nsec entry point gives the adapter's walk bit for bit; the double entry point switches one frame later
    ros_raw = raw_walk(ros, clouds, stamps, ros_stamps=True)
    assert [bits(r["odom"]) for r in ros_raw] == [bits(a["odom"]) for a in ans]
    dbl = raw_walk(ros, clouds, stamps)
    assert not dbl[10]["keyframe_updated"] and dbl[11]["keyframe_updated"]
    assert any(bits(d["odom"]) != bits(a["odom"]) for d, a in zip(dbl, ans))


def test_mixing_stamp_forms(frames):
    """the keyframe keeps the form of the call that made it; roscpp's rule only when both stamps are sec / nsec"""
    clouds = [frames[k] for k in range(4)]
    p = dict(keyframe_delta_trans=1e6, keyframe_delta_angle=1e6, keyframe_delta_time=1.0)
    t0, t1 = stamp(BASE_NS), stamp(BASE_NS + 1_000_000_207)
    assert to_sec(t1) - to_sec(t0) == 1.0

    def run(first_ros, second_ros):
        reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
        odo = pkg.ScanMatchingOdometry(reg, **p)
        a = odo.matching_ros(*t0, clouds[0]) if first_ros else odo.matching(to_sec(t0), clouds[0])
        b = odo.matching_ros(*t1, clouds[1]) if second_ros else odo.matching(to_sec(t1), clouds[1])
        odo.close()
        reg.close()
        assert a["keyframe_updated"] and b["converged"] and not b["frame_rejected"]
        return b["keyframe_updated"]
    assert run(True, True)        # 1.000000207 > 1.0
    assert not run(False, True)   # a double keyframe stamp: toSec(t1) - toSec(t0) == 1.0
    assert not run(True, False)   # a double frame stamp
    assert not run(False, False)


# ---- PointCloud2 input
def organized_with_nan(cloud, rows=16):
    """an organized (rows x n / rows) cloud with every 7th record and one whole column NaN, as a driver publishes missing returns"""
    c = np.array(cloud, np.float32)
    c[::7, :3] = np.nan
    c[3::(c.shape[0] // rows), :3] = np.nan
    return c


def msg_walks(frames):
    """per kind: (messages, the pcl clouds fromROSMsg gives, (width, height), is_dense)"""
    out = {}
    # velodyne-style, height 1, a different size every frame (the ingest buffers are reallocated as the walk goes)
    msgs, clouds, wh = [], [], []
    for k, f in enumerate(frames):
        m = message(f[:f.shape[0] - 97 * (k % 5), [0, 1, 2, 4]], kind="velodyne", seed=k)
        msgs.append(m)
        clouds.append(decode_rows(m["data"], m["width"], 1, m["row_step"], layout_of(m["fields"], m["point_step"])).view(np.float32))
        wh.append((m["width"], 1))
    out["velodyne"] = (msgs, clouds, wh, True)
    for kind, pad in (("organized", 0), ("padded", 6)):
        msgs, clouds, wh = [], [], []
        for k, f in enumerate(frames):
            c = organized_with_nan(f)
            m = message(c[:, [0, 1, 2, 4]], kind="ouster", width=c.shape[0] // 16, height=16, pad=pad, seed=k)
            dec = decode_rows(m["data"], m["width"], m["height"], m["row_step"], layout_of(m["fields"], m["point_step"]))
            msgs.append(m)
            clouds.append(dec.view(np.float32))
            wh.append((m["width"], m["height"]))
        out[kind] = (msgs, clouds, wh, False)
    return out


@pytest.mark.parametrize("method,downsample", [("FAST_GICP", "NONE"), ("FAST_GICP", "VOXELGRID"), ("NDT_OMP", "NONE")])
def test_pointcloud2_walks_equal_the_pcl_walks(harness, tmp_path, frames, method, downsample):
    ros = dict(LAUNCH["hdl"], registration_method=method, downsample_method=downsample, transform_thresholding="true",
               max_acceptable_trans="0.5", keyframe_delta_trans="0.5")
    stamps = walk_stamps()
    jobs, meta = [], []
    for kind, (msgs, clouds, wh, dense) in msg_walks(frames).items():
        want_aligned = (lambda k: True) if kind != "padded" else (lambda k: k % 2 == 0)
        mc = [encode_call(ODOMETRY, msg_input(m, dense), st, msf=msf_every_fifth(k), want_aligned=want_aligned(k))
              for k, (m, st) in enumerate(zip(msgs, stamps))]
        pc = [encode_call(ODOMETRY, pcl_input(c, width=w, height=h, is_dense=dense), st, msf=msf_every_fifth(k), want_aligned=want_aligned(k))
              for k, (c, (w, h), st) in enumerate(zip(clouds, wh, stamps))]
        jobs += [(ODOMETRY, ros, mc), (ODOMETRY, ros, pc)]
        meta.append((kind, clouds, wh, dense, want_aligned))
    answers, blocks = run_jobs(harness, tmp_path, jobs)
    for i, (kind, clouds, wh, dense, want_aligned) in enumerate(meta):
        assert blocks[2 * i] == blocks[2 * i + 1], kind
        ans = answers[2 * i]
        raw = raw_walk(ros, clouds, stamps, msf_every_fifth)
        assert_walk(ans, raw, clouds, ros, lambda k: True, want_aligned, is_dense=dense, widths=wh)
        if method == "FAST_GICP":
            assert any(a["frame_rejected"] for a in ans) and sum(a["keyframe_updated"] for a in ans) >= 2, kind


def test_message_without_float32_xyz_is_refused(harness, tmp_path, frames):
    m = message(frames[0][:, [0, 1, 2, 4]], kind="velodyne")
    m["fields"] = [f if f[0] != "z" else ("z", 8, 8, 1) for f in m["fields"]]
    ((ans,), _) = run_jobs(harness, tmp_path, [(ODOMETRY, {"downsample_method": "NONE"}, [encode_call(ODOMETRY, msg_input(m), stamp(BASE_NS))])])
    assert ans[0][0] == "error" and ans[0][1] == 1 and "FLOAT32 x, y and z" in ans[0][2]


def test_aligned_on_non_dense_and_dense_clouds_with_non_finite_records(harness, tmp_path, frames):
    """NaN and inf records in a host cloud, declared dense and non-dense: accepted, keyframe and rejected frames"""
    ros = dict(LAUNCH["hdl"], transform_thresholding="true", max_acceptable_trans="0.5", keyframe_delta_trans="0.5")
    clouds = []
    for k, f in enumerate(frames):
        c = np.array(f, np.float32)
        c[5::41, 0] = np.nan
        c[9::53, 1] = np.inf
        c[13::67, 2] = -np.inf
        c[:, 5:] = np.float32(k)  # bytes after the intensity are copied too
        clouds.append(c)
    stamps = walk_stamps()
    jobs = [(ODOMETRY, ros, [encode_call(ODOMETRY, pcl_input(c, is_dense=dense), st) for c, st in zip(clouds, stamps)]) for dense in (False, True)]
    (nd, de), _ = run_jobs(harness, tmp_path, jobs)
    raw = raw_walk(ros, clouds, stamps)
    assert_walk(nd, raw, clouds, ros, lambda k: True, lambda k: True, is_dense=False)
    assert_walk(de, raw, clouds, ros, lambda k: True, lambda k: True, is_dense=True)
    assert any(a["frame_rejected"] for a in nd) and sum(a["keyframe_updated"] for a in nd) >= 3


def test_want_status_toggled_per_frame(harness, tmp_path, frames):
    ros = dict(LAUNCH["501"], downsample_method="VOXELGRID")
    stamps = walk_stamps()
    on = [encode_call(ODOMETRY, pcl_input(c), st) for c, st in zip(frames, stamps)]
    toggled = [encode_call(ODOMETRY, pcl_input(c), st, want_status=k % 3 == 1, want_aligned=k % 4 == 2) for k, (c, st) in enumerate(zip(frames, stamps))]
    (a_on, a_tg), _ = run_jobs(harness, tmp_path, [(ODOMETRY, ros, on), (ODOMETRY, ros, toggled)])
    raw = raw_walk(ros, frames, stamps)
    assert_walk(a_on, raw, frames, ros, lambda k: True, lambda k: True)
    assert_walk(a_tg, raw, frames, ros, lambda k: k % 3 == 1, lambda k: k % 4 == 2)
    for x, y in zip(a_on, a_tg):
        assert bits(x["odom"]) == bits(y["odom"])


def test_odometry_and_prefilter_on_two_threads(harness, tmp_path, frames):
    ros = dict(LAUNCH["hdl"])
    stamps = walk_stamps()
    jobs = [(ODOMETRY, ros, [encode_call(ODOMETRY, pcl_input(c), st) for c, st in zip(frames, stamps)]),
            (PREFILTER, {"downsample_method": "VOXELGRID", "outlier_removal_method": "RADIUS"},
             [encode_call(PREFILTER, pcl_input(c), st) for c, st in zip(frames, stamps)])]
    _, serial = run_jobs(harness, tmp_path, jobs, "serial")
    _, concurrent = run_jobs(harness, tmp_path, jobs, "concurrent")
    assert serial == concurrent
