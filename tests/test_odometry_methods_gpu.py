"""GPU: the odometry drop-in (adapter/b200_odometry.hpp, through tests/odometry_harness.cpp) on every registration branch the factory
serves, and the registration-parameter forwarding (adapter/b200_select.hpp) that both drop-ins share.

- 24-frame walks (keyframe switches by distance and time, far jumps and sideways msf_delta guesses that thresholding rejects) on pcl
  GICP, pclomp GICP, pcl ICP, FastVGICP, FastVGICPCuda, NDT_OMP's KDTREE and DIRECT1 searches, and FastGICP /
  NDT_OMP / pcl NDT, with downsample NONE, VOXELGRID and (one GICP-family and one NDT-family method) APPROX_VOXELGRID:
  - every answer bit for bit b2r_odometry_matching with parameters built from the reference lines;
  - every align of the walk bitwise a fresh single handle's from the same guess on the same keyframe and registered frame;
  - the same keyframe switches and rejections as tests/odometry_ref.py's replay with each method's sequential reference as the align,
    the same iterations and flag, the pose within that method's tolerance (tests/method_refs.py; pcl GICP and pclomp GICP: the rule
    stated at the comparison); every walk switches and rejects at least once and accepts without a switch at least once;
  - the status exactly: matching_error bitwise b2r_fitness at the returned pose on a fresh handle and within 1e-12 of the oracle's
    fitness there, inlier_fraction bitwise float(inliers) / float(size of the registered, downsampled frame) with the oracle's count.
- PointCloud2 walks (velodyne records in 16 padded rows) bitwise the pcl overload's, one per method family.
- An empty frame's status: inlier_fraction is 0/0 = NaN, as the reference's division gives it.
- Parameter forwarding: under every reg_* key a branch reads, set to a non-default value, the handles of B200KeyframeCache and
  B200ScanMatchingOdometry are configured field for field as b2r_select_registration_method configures one from the same dict, and a
  short walk is bitwise the raw mirror's and differs from the default set's; NDT_OMP with KDTREE is refused by both drop-ins with the
  engine's B2R_EUNSUPPORTED message, B200_NDT_KDTREE with the same key is served."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg
import odometry_ref
from frontend_ref import decode_rows, layout_of, message
from method_refs import METHODS, NDT_FAMILY, NON_DEFAULT, References, pose_close, pose_tolerance
from odometry_adapter_io import ODOMETRY, ROOT, build_harness, encode_call, msg_input, pcl_input, run_jobs
from test_odometry_adapter_gpu import assert_walk, bits, raw_params, raw_walk, reg_params, stamp, to_sec, BASE_NS

pytestmark = pytest.mark.gpu
DBL_MAX = np.finfo(np.float64).max
N_FRAMES = 24
JUMPS = (7, 15)    # these frames get the scan 25 frames (7.5 m) ahead
JOLTS = (11, 20)   # these frames get a 1.2 m sideways msf_delta: an align that stays near its guess is rejected
MSF = np.array([[1, 0, 0, 0.3], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float32)
JOLT = np.array([[1, 0, 0, 0], [0, 1, 0, 1.2], [0, 0, 1, 0], [0, 0, 0, 1]], np.float32)
LEAF = 0.25
# keyframes 0.5 m or 0.35 s apart (the NDT aligns move little on these scans, so time switches them too), thresholding at 0.5 m
ODOM = dict(odom_frame_id="odom", keyframe_delta_trans="0.5", keyframe_delta_angle="1.0", keyframe_delta_time="0.35",
            transform_thresholding="true", max_acceptable_trans="0.5", max_acceptable_angle="1.0", downsample_resolution=str(LEAF))

WALKS = [(m, ds) for m in ("GICP", "B200_GICP_OMP", "B200_ICP", "FAST_VGICP", "B200_VGICP_CUDA", "B200_NDT_KDTREE", "NDT_OMP_DIRECT1")
         for ds in ("NONE", "VOXELGRID")]
WALKS += [("GICP", "APPROX_VOXELGRID"), ("B200_NDT_KDTREE", "APPROX_VOXELGRID"),
          ("FAST_GICP", "VOXELGRID"), ("NDT_OMP", "VOXELGRID"), ("NDT", "NONE")]


def msf_of(k):
    return JOLT if k in JOLTS else (MSF if k % 5 == 4 else None)


def walk_stamps(n=N_FRAMES, period_ns=97_300_000):
    return [stamp(BASE_NS + k * period_ns) for k in range(n)]


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return build_harness(tmp_path_factory.mktemp("odometry") / "odometry_harness")


@pytest.fixture(scope="module")
def refs(tmp_path_factory, oracle):
    r = References(tmp_path_factory, oracle)
    yield r
    r.close()


@pytest.fixture(scope="module")
def filt():
    r = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    yield r
    r.close()


@pytest.fixture(scope="module")
def frames(synth):
    out = [synth.scan("vlp16_16k", frame=k, step=0.3, stride=8) for k in range(N_FRAMES)]
    for j in JUMPS:
        out[j] = synth.scan("vlp16_16k", frame=j + 25, step=0.3, stride=8)
    return out


PCL_GICP = ("GICP", "B200_GICP_OMP")


def walk_ros(case, downsample):
    ros = dict(ODOM, downsample_method=downsample, **METHODS[case])
    if case in PCL_GICP:
        # at 0.5 m a jump's rejection strands these walks: every later frame is aligned from a stale guess to a keyframe more than
        # 0.5 m behind and rejected, and the BFGS end points of such aligns hang on the line search's last bits (see the replay below)
        ros["max_acceptable_trans"] = "1.0"
    return ros


def registered(filt, clouds, downsample):
    """the clouds the mirror registers: its own downsample stage, restated by the engine's filters (bitwise the stage's, see
    test_odometry_branches_gpu / test_odometry_downsample_gpu)"""
    if downsample == "VOXELGRID":
        return [filt.voxelGridFilter(c, LEAF) for c in clouds]
    if downsample == "APPROX_VOXELGRID":
        return [filt.approximateVoxelGridFilter(c, LEAF) for c in clouds]
    return list(clouds)


def taken_and_not(flags, what):
    flags = list(flags)
    assert any(flags) and not all(flags), (what, flags)


def assert_status_exact(ans, reg_clouds, params, oracle):
    """matching_error bitwise b2r_fitness at the engine's own returned pose on a fresh handle of the method and within 1e-12 of the
    oracle there; inlier_fraction bitwise float(oracle's inliers) / float(registered frame size) (:321, static_cast<float> / size())"""
    fresh = pkg.select_registration_method(params)
    kf = reg_clouds[0]
    for k in range(1, len(ans)):
        a, src = ans[k], reg_clouds[k]
        fresh.setInputTarget(kf)
        fresh.setInputSource(src)
        score, _, inl_engine = fresh.getFitnessScore(DBL_MAX, T=a["trans"], inlier_thresh_sq=0.25, full=True)
        assert np.float64(a["matching_error"]).tobytes() == np.float64(score).tobytes(), k
        want, used, inl = oracle.fitness(kf, src, a["trans"], DBL_MAX, 0.25)
        assert used > 0 and abs(a["matching_error"] - want) <= 1e-12 * want, (k, a["matching_error"], want)
        assert inl_engine == inl, k
        frac = np.float32(inl) / np.float32(src.shape[0])
        assert np.float32(a["inlier_fraction"]).tobytes() == frac.tobytes(), (k, a["inlier_fraction"], frac)
        if a["keyframe_updated"]:
            kf = src
    fresh.close()


def engine_guesses(ros, raw, reg_clouds, stamps):
    """each frame's guess prev_trans * msf_delta (:210) and target as the engine's walk had them: odometry_ref's replay fed the
    engine's own align results (its gate is bitwise the engine's, test_odometry_gate)"""
    it = iter(raw[1:])
    mirror = odometry_ref.Replay(lambda c, kf, g: (lambda r: dict(T=r["trans"], converged=r["converged"], iterations=r["iterations"]))(next(it)),
                                 **raw_params(ros))
    out = [mirror.matching(to_sec(st), c, msf_of(k)) for k, (c, st) in enumerate(zip(reg_clouds, stamps))]
    return [r.get("guess") for r in mirror.log], [o["keyframe"] for o in out]


def assert_aligns_are_single_aligns(raw, reg_clouds, guesses, keyframes, params):
    """every align of the walk, whose target is a promoted source and whose source may have been prefetched, is bitwise a fresh single
    handle's set_target(keyframe) / set_source(frame) / align(guess)"""
    fresh = pkg.select_registration_method(params)
    for k in range(1, len(raw)):
        fresh.setInputTarget(keyframes[k])
        fresh.setInputSource(reg_clouds[k])
        fresh.align(guesses[k])
        assert (fresh.hasConverged(), fresh.nr_iterations) == (raw[k]["converged"], raw[k]["iterations"]), k
        assert bits(fresh.getFinalTransformation()) == bits(raw[k]["trans"]), k
    fresh.close()


@pytest.mark.parametrize("case,downsample", WALKS)
def test_walk_on_every_method(harness, tmp_path, frames, refs, filt, oracle, case, downsample):
    ros = walk_ros(case, downsample)
    stamps = walk_stamps()
    calls = [encode_call(ODOMETRY, pcl_input(c), st, msf=msf_of(k)) for k, (c, st) in enumerate(zip(frames, stamps))]
    ((ans,), _) = run_jobs(harness, tmp_path, [(ODOMETRY, ros, calls)])
    raw = raw_walk(ros, frames, stamps, msf_of)
    assert_walk(ans, raw, frames, ros, lambda k: True, lambda k: True)
    taken_and_not([a["keyframe_updated"] for a in ans[1:]], "keyframe switch")
    taken_and_not([a["frame_rejected"] for a in ans[1:]], "thresholding rejection")
    assert any(a["converged"] and a["frame_rejected"] for a in ans[1:]), "a rejection by the thresholds, not by convergence"

    reg_clouds = registered(filt, frames, downsample)
    if downsample != "NONE":
        assert all(r.shape[0] < c.shape[0] for r, c in zip(reg_clouds, frames))
    assert_status_exact(ans, reg_clouds, reg_params(ros), oracle)
    guesses, keyframes = engine_guesses(ros, raw, reg_clouds, stamps)
    assert_aligns_are_single_aligns(raw, reg_clouds, guesses, keyframes, reg_params(ros))

    # the reference walk: odometry_ref's replay of matching() with the method's sequential reference as the align.  Every align
    # starts from the engine's own guess of that frame (the replay's guess agrees with it to the pose tolerance): an align stops once a
    # step moves less than transformation_epsilon, so its end point is not continuous in the guess, and a walk would carry a
    # difference far below the tolerance into a different stop a few frames on
    h = pkg.select_registration_method(reg_params(ros))
    cfg = h.config
    h.close()

    def align(c, kf, g):
        k = len(rep.log)
        # the replay's prev_trans is the reference's pose of an earlier frame, held to the method's tolerance below
        tol = 5e-3 if case in PCL_GICP else pose_tolerance(case)
        assert np.max(np.abs(g - guesses[k])) <= 4 * tol, (k, np.max(np.abs(g - guesses[k])))
        return refs.align(case, cfg, c, kf, guesses[k])
    rep = odometry_ref.Replay(align, **raw_params(ros))
    want = [rep.matching(to_sec(st), c, msf_of(k)) for k, (c, st) in enumerate(zip(reg_clouds, stamps))]
    for k, (a, r, w) in enumerate(zip(ans, raw, want)):
        assert (a["keyframe_updated"], a["frame_rejected"]) == (bool(w["keyframe_updated"]), bool(w["frame_rejected"])), k
        if k == 0:
            continue
        if case in PCL_GICP:
            # pcl GICP / pclomp GICP: the walk's aligns are bitwise single aligns (above), so what is left between engine and
            # reference is their BFGS: the line search compares f values that agree to the last bits, and a fixed-tree sum against an
            # index-order one may take another step there.  From the same guess on these sparse 2048-point scans the two end points
            # lie up to 3e-3 apart on frames the walk accepts, and far apart on frames a jump puts metres from the keyframe (both
            # rejected).  Pinned: the same decisions and flag on every frame; on an accepted frame at most one outer iteration apart,
            # every pose entry within 5e-3, and the oracle's fitness at the two end points within 5e-3 relative (measured: up to 3.4e-3)
            assert r["converged"] == w["converged"], k
            if not r["frame_rejected"]:
                assert abs(r["iterations"] - w["iterations"]) <= 1, (k, r["iterations"], w["iterations"])
                assert np.max(np.abs(r["trans"] - w["trans"])) <= 5e-3, (k, np.max(np.abs(r["trans"] - w["trans"])))
                fe = oracle.fitness(w["keyframe"], reg_clouds[k], r["trans"], DBL_MAX, 0.25)[0]
                fr = oracle.fitness(w["keyframe"], reg_clouds[k], w["trans"], DBL_MAX, 0.25)[0]
                assert abs(fe - fr) <= 5e-3 * fr, (k, fe, fr)
            continue
        assert (r["converged"], r["iterations"]) == (w["converged"], w["iterations"]), (k, r["iterations"], w["iterations"])
        assert pose_close(case, r["trans"], w["trans"]), (k, np.max(np.abs(r["trans"] - w["trans"])))
        if case not in NDT_FAMILY and case != "B200_ICP":
            # the status against the oracle at the REFERENCE's pose (a different question from the exact check above)
            score, _, inl = oracle.fitness(w["keyframe"], reg_clouds[k], w["trans"], DBL_MAX, 0.25)
            assert abs(a["matching_error"] - score) <= 1e-6 * score and abs(a["inlier_fraction"] - inl / reg_clouds[k].shape[0]) < 1e-6, k


@pytest.mark.parametrize("case", ["GICP", "FAST_VGICP", "B200_NDT_KDTREE"])
def test_pointcloud2_walk_equals_the_pcl_walk(harness, tmp_path, frames, case):
    """velodyne records (x y z intensity ring time, 22 bytes) in 16 rows with 6 bytes of padding after each"""
    ros = walk_ros(case, "VOXELGRID")
    stamps = walk_stamps()
    mc, pc = [], []
    for k, (f, st) in enumerate(zip(frames, stamps)):
        m = message(f[:, [0, 1, 2, 4]], kind="velodyne", width=f.shape[0] // 16, height=16, pad=6, seed=k)
        assert m["row_step"] > m["width"] * m["point_step"]
        c = decode_rows(m["data"], m["width"], m["height"], m["row_step"], layout_of(m["fields"], m["point_step"])).view(np.float32)
        mc.append(encode_call(ODOMETRY, msg_input(m, True), st, msf=msf_of(k)))
        pc.append(encode_call(ODOMETRY, pcl_input(c, width=m["width"], height=16, is_dense=True), st, msf=msf_of(k)))
    (am, ap), blocks = run_jobs(harness, tmp_path, [(ODOMETRY, ros, mc), (ODOMETRY, ros, pc)])
    assert blocks[0] == blocks[1]
    taken_and_not([a["keyframe_updated"] for a in am[1:]], "keyframe switch")
    taken_and_not([a["frame_rejected"] for a in am[1:]], "thresholding rejection")


@pytest.mark.parametrize("case", ["FAST_GICP", "B200_ICP", "NDT_OMP"])
def test_empty_frame_status(harness, tmp_path, frames, case):
    """an empty frame registers nothing: the align does not converge, the frame is rejected, getFitnessScore has no neighbour
    (DBL_MAX), and inlier_fraction is static_cast<float>(0) / 0 = NaN; the walk goes on from the state before it"""
    ros = walk_ros(case, "NONE")
    clouds = [frames[0], frames[1], np.zeros((0, 8), np.float32), frames[2], frames[3]]
    stamps = walk_stamps(len(clouds))
    calls = [encode_call(ODOMETRY, pcl_input(c), st) for c, st in zip(clouds, stamps)]
    ((ans,), _) = run_jobs(harness, tmp_path, [(ODOMETRY, ros, calls)])
    raw = raw_walk(ros, clouds, stamps)
    assert_walk(ans, raw, clouds, ros, lambda k: k != 2, lambda k: True)
    e = ans[2]
    assert not e["converged"] and e["frame_rejected"] and not e["keyframe_updated"]
    assert e["matching_error"] == DBL_MAX and np.isnan(e["inlier_fraction"]) and np.isnan(raw[2]["inlier_fraction"])
    assert e["aligned"] is None
    assert bits(ans[3]["odom"]) == bits(raw[3]["odom"]) and ans[3]["converged"] and not ans[3]["frame_rejected"]


# ---- registration-parameter forwarding (adapter/b200_select.hpp)
FIELD = {"reg_maximum_iterations": "max_iterations", "reg_transformation_epsilon": "transformation_epsilon",
         "reg_max_correspondence_distance": "max_correspondence_distance", "reg_correspondence_randomness": "k_correspondences",
         "reg_max_optimizer_iterations": "max_optimizer_iterations", "reg_use_reciprocal_correspondences": "use_reciprocal_correspondences",
         "reg_resolution": "ndt_resolution", "reg_nn_search_method": "ndt_search_method"}


@pytest.fixture(scope="module")
def select_harness(tmp_path_factory):
    from hdl_graph_slam_b200 import build
    build.build_engine()
    exe = str(tmp_path_factory.mktemp("select") / "select_harness")
    lib = os.path.join(ROOT, "hdl_graph_slam_b200", "_lib")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++14", "-O1", "-Wall", "-pthread",
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "hdl_graph_slam_b200", "adapter"), "-o", exe,
                           os.path.join(ROOT, "tests", "select_harness.cpp"), "-L", lib, "-lb200reg", "-Wl,-rpath," + lib])
    return exe


def dropin_configs(exe, tmp_path, params):
    """(the keyframe cache's, the odometry's) handle configuration, each a b2r_config or the text the constructor threw"""
    src, dst = tmp_path / "select_in.bin", tmp_path / "select_out.bin"
    body = b"".join(struct.pack("<i", len(s)) + s for k, v in params.items() for s in (k.encode(), str(v).encode()))
    src.write_bytes(struct.pack("<i", len(params)) + body)
    out = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    b, o, res = dst.read_bytes(), 0, []
    Config = type(pkg.default_config(pkg.B2R_METHOD_GICP))
    for _ in range(2):
        (st,) = struct.unpack_from("<i", b, o)
        o += 4
        if st == 0:
            res.append(Config.from_buffer_copy(b[o:o + ctypes.sizeof(Config)]))
            o += ctypes.sizeof(Config)
        else:
            (n,) = struct.unpack_from("<i", b, o)
            res.append(b[o + 4:o + 4 + n].decode())
            o += 4 + n
    assert o == len(b)
    return res


def fields(cfg):
    return {name: getattr(cfg, name) for name, _ in cfg._fields_}


@pytest.mark.parametrize("branch", list(NON_DEFAULT))
def test_dropins_configure_the_handle_as_the_factory(select_harness, tmp_path, branch):
    params = NON_DEFAULT[branch]
    cache, odom = dropin_configs(select_harness, tmp_path, params)
    h = pkg.select_registration_method(params)
    want = fields(h.config)
    h.close()
    assert not isinstance(cache, str) and not isinstance(odom, str), (cache, odom)
    assert fields(cache) == want and fields(odom) == want
    d = pkg.select_registration_method({"registration_method": params["registration_method"]})
    default = fields(d.config)
    d.close()
    for k in params:  # every key that was set moved its field: a key the forwarding dropped would leave the default
        if k != "registration_method":
            assert want[FIELD[k]] != default[FIELD[k]], (branch, k)
    # the default set through the drop-ins is the factory default
    cache_d, odom_d = dropin_configs(select_harness, tmp_path, {"registration_method": params["registration_method"]})
    assert fields(cache_d) == default and fields(odom_d) == default


def test_kdtree_is_refused_on_ndt_omp_and_served_on_b200_ndt_kdtree(select_harness, tmp_path):
    params = {"registration_method": "NDT_OMP", "reg_resolution": "1.0", "reg_nn_search_method": "KDTREE"}
    with pytest.raises(pkg.B2RError) as e:
        pkg.select_registration_method(params)
    assert e.value.code == -5  # B2R_EUNSUPPORTED
    cache, odom = dropin_configs(select_harness, tmp_path, params)
    assert isinstance(cache, str) and isinstance(odom, str), (cache, odom)
    assert cache == odom and cache.startswith("b200reg: ") and "KDTREE" in cache, cache
    ok = dict(params, registration_method="B200_NDT_KDTREE")
    cache, odom = dropin_configs(select_harness, tmp_path, ok)
    h = pkg.select_registration_method(ok)
    want = fields(h.config)
    h.close()
    assert fields(cache) == want == fields(odom) and want["method"] == pkg.B2R_METHOD_NDT_KDTREE


@pytest.mark.parametrize("branch", list(NON_DEFAULT))
def test_non_default_walk_is_the_raw_walk(harness, tmp_path, frames, branch):
    """a short walk under the non-default set is bitwise the raw mirror's with that dict, and differs from the default set's walk"""
    clouds, stamps = frames[:8], walk_stamps(8)
    ros = dict(ODOM, downsample_method="NONE", **NON_DEFAULT[branch])
    ros_d = dict(ODOM, downsample_method="NONE", registration_method=NON_DEFAULT[branch]["registration_method"])
    jobs = [(ODOMETRY, r, [encode_call(ODOMETRY, pcl_input(c), st, msf=msf_of(k)) for k, (c, st) in enumerate(zip(clouds, stamps))])
            for r in (ros, ros_d)]
    (ans, ans_d), (blk, blk_d) = run_jobs(harness, tmp_path, jobs)
    assert_walk(ans, raw_walk(ros, clouds, stamps, msf_of), clouds, ros, lambda k: True, lambda k: True)
    assert_walk(ans_d, raw_walk(ros_d, clouds, stamps, msf_of), clouds, ros_d, lambda k: True, lambda k: True)
    assert blk != blk_d
