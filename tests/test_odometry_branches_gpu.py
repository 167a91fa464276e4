"""GPU: every branch of the odometry mirror's matching() (apps/scan_matching_odometry_nodelet.cpp:165-262) against ONE test-side replay
of those lines (tests/odometry_ref.py: first frame, guess = prev_trans * msf_delta, not converged, transform thresholding, the three
keyframe criteria, all four branches of the quaternion conversion), with the align taken from the oracle.  Same converged flag and
iteration count, pose <= 1e-6 (GICP) / 1e-4 (NDT), keyframe_updated / frame_rejected equal on every frame.  Every case asserts that
the branch it is about was taken at least once AND not taken at least once, and is repeated bitwise with every next frame
announced (b2r_odometry_prefetch) and with the mirror's own VOXELGRID downsample."""
import numpy as np
import pytest
import torch  # before the engine library: it links the system NCCL, and torch's CUDA libraries must resolve against their own first
import hdl_graph_slam_b200 as pkg
from common import rot_err, trans_err, perturb

import odometry_ref as ref
from ndt_pcl_ref import Reference

pytestmark = pytest.mark.gpu
f32 = np.float32
BIG = 1e9
GICP = {"registration_method": "FAST_GICP"}
NDT_OMP = {"registration_method": "NDT_OMP", "reg_resolution": 1.0}
NDT_PCL = {"registration_method": "NDT", "reg_resolution": 1.0}
LEAF = 0.25


def status_key(st):
    """every field of a status, as bits"""
    return (st["odom"].view(np.uint32).tobytes(), st["trans"].view(np.uint32).tobytes(), st["iterations"], st["converged"], st["keyframe_updated"],
            st["frame_rejected"], np.float64(st["matching_error"]).tobytes(), np.float32(st["inlier_fraction"]).tobytes())


def assert_same(a, b):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert status_key(x) == status_key(y), k


def engine_walk(params, odo_kw, clouds, stamps, msf=None, device=False, announce=False, downsample=False):
    """statuses of the mirror over the sequence; device: the _device entry point on device copies; announce: every next frame is
    announced before the call; downsample: the mirror's own VOXELGRID stage on the raw clouds"""
    reg = pkg.select_registration_method(dict(params))
    kw = dict(odo_kw)
    if downsample:
        kw.update(downsample_method=pkg.B2R_DOWNSAMPLE_VOXELGRID, downsample_resolution=LEAF)
    odo = pkg.ScanMatchingOdometry(reg, **kw)
    if device:
        clouds = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for c in clouds]
        torch.cuda.synchronize()
    ptr = (lambda c: c.data_ptr()) if device else (lambda c: c.ctypes.data)
    out = []
    for k, c in enumerate(clouds):
        if announce and k + 1 < len(clouds):
            nxt = clouds[k + 1]
            odo.prefetch_raw(ptr(nxt), nxt.shape[0], nxt.shape[1] * 4, device=device)
        out.append(odo.matching_raw(stamps[k], ptr(c), c.shape[0], c.shape[1] * 4, None if msf is None else msf[k], device=device))
    odo.close()
    reg.close()
    return out


def replay_walk(align, odo_kw, clouds, stamps, msf=None):
    r = ref.Replay(align, **odo_kw)
    return [r.matching(stamps[k], c, None if msf is None else msf[k]) for k, c in enumerate(clouds)], r.log


def compare(sts, want, tol, fitness=None):
    """engine statuses against the replay's, frame by frame; fitness(keyframe, cloud, T) -> (score, inlier fraction) checks the
    status fields, which are those of the align's final pose on rejected frames too (:212-214 run before the convergence check)"""
    assert len(sts) == len(want)
    for k, (s, w) in enumerate(zip(sts, want)):
        assert (s["keyframe_updated"], s["frame_rejected"]) == (w["keyframe_updated"], w["frame_rejected"]), k
        if k == 0:
            assert np.array_equal(s["odom"], np.eye(4, dtype=f32)) and np.array_equal(s["trans"], np.eye(4, dtype=f32))
            continue
        assert s["converged"] == w["converged"] and s["iterations"] == w["iterations"], k
        assert trans_err(s["trans"], w["trans"]) < tol and rot_err(s["trans"], w["trans"]) < tol, k
        scale = max(1.0, float(np.max(np.abs(w["odom"][:3, 3]))))
        assert trans_err(s["odom"], w["odom"]) < 4 * tol * scale and rot_err(s["odom"], w["odom"]) < 4 * tol, k
        if fitness is not None:
            score, frac = fitness(w["keyframe"], w["cloud"], w["trans"])
            assert abs(s["matching_error"] - score) <= 1e-6 * score and abs(s["inlier_fraction"] - frac) < 1e-6, k


def taken_and_not(flags, what):
    flags = list(flags)
    assert any(flags) and not all(flags), (what, flags)


def variants_agree(params, odo_kw, clouds, stamps, base, msf=None, filter_handle=None):
    """the same walk with every next frame announced, host and device, is bitwise the plain one; and the mirror's own VOXELGRID stage
    on the raw clouds, announced or not, is bitwise the plain mirror on the clouds filtered beforehand"""
    assert_same(engine_walk(params, odo_kw, clouds, stamps, msf, announce=True), base)
    assert_same(engine_walk(params, odo_kw, clouds, stamps, msf, device=True, announce=True), base)
    if filter_handle is not None:
        filt = [filter_handle.voxelGridFilter(c, LEAF) for c in clouds]
        pre = engine_walk(params, odo_kw, filt, stamps, msf)
        taken_and_not([s["frame_rejected"] or s["keyframe_updated"] for s in pre[1:]], "a rejection or a switch in the downsampled walk")
        assert_same(engine_walk(params, odo_kw, clouds, stamps, msf, downsample=True), pre)
        assert_same(engine_walk(params, odo_kw, clouds, stamps, msf, downsample=True, announce=True), pre)
        assert_same(engine_walk(params, odo_kw, clouds, stamps, msf, device=True, downsample=True, announce=True), pre)


# ---- sequences
def line_frames(synth, idx, sensor="vlp16_16k"):
    """frames of the circuit (1 m and 1.4 degrees apart) in the order idx"""
    return [synth.scan(sensor, frame=k, stride=8) for k in idx]


def yaw_frames(synth, yaws_deg):
    """scans from one place, turned by yaws_deg"""
    x, y, th = synth.pose(0)
    return [synth.scan("vlp16_16k", frame=0, stride=8, xyyaw=(x, y, th + np.deg2rad(a))) for a in yaws_deg]


def stamps_of(n):
    return [0.1 * k for k in range(n)]


@pytest.fixture(scope="module")
def filt():
    r = pkg.select_registration_method(dict(GICP))
    yield r
    r.close()


def gicp_align(oracle, **kw):
    return lambda c, kf, g: oracle.gicp_align(c, kf, g, **kw)


def gicp_fitness(oracle):
    def f(keyframe, cloud, T):
        fs, _, fi = oracle.fitness(keyframe, cloud, T)
        return fs, fi / cloud.shape[0]
    return f


def with_clouds(want, clouds):
    for w, c in zip(want, clouds):
        w["cloud"] = c
    return want


KF_OFF = dict(keyframe_delta_trans=BIG, keyframe_delta_angle=BIG, keyframe_delta_time=BIG)


# ---- msf_delta
def test_msf_delta_is_the_guess(synth, oracle, filt):
    idx = list(range(9))
    clouds = line_frames(synth, idx)
    stamps = stamps_of(len(idx))
    odo_kw = dict(keyframe_delta_trans=2.5, keyframe_delta_angle=BIG, keyframe_delta_time=BIG)
    # the true motion between consecutive frames: a rotation and a translation, so a transposed read is another matrix
    good = [np.eye(4, dtype=f32)] + [(np.linalg.inv(synth.pose_matrix(a)) @ synth.pose_matrix(b)).astype(f32) for a, b in zip(idx, idx[1:])]
    poor = [perturb(70 + k, 0.6, 4.0).astype(f32) for k in range(len(idx))]
    assert not np.allclose(good[1], good[1].T, atol=1e-3)
    iters = {}
    for name, msf in (("identity", None), ("good", good), ("poor", poor)):
        want, log = replay_walk(gicp_align(oracle), odo_kw, clouds, stamps, msf)
        sts = engine_walk(GICP, odo_kw, clouds, stamps, msf)
        compare(sts, want, 1e-6)
        taken_and_not([w["keyframe_updated"] for w in want[1:]], "keyframe switch")
        iters[name] = [w["iterations"] for w in want[1:]]
        assert_same(engine_walk(GICP, odo_kw, clouds, stamps, msf, device=True), sts)
        if name == "good":
            variants_agree(GICP, odo_kw, clouds, stamps, sts, msf, filt)
            # a mirror reading the delta untransposed would hand the align another guess: the oracle started from it differs from this
            # walk by more than `compare` tolerates (iteration count, or pose beyond the tolerance) on some frame
            wrong, _ = replay_walk(gicp_align(oracle), odo_kw, clouds, stamps, [m.T.copy() for m in msf])
            assert any(a["iterations"] != b["iterations"] or trans_err(a["trans"], b["trans"]) > 1e-5 or rot_err(a["trans"], b["trans"]) > 1e-5
                       for a, b in zip(want[1:], wrong[1:]))
    # a mirror that ignored the argument would report the identity run's iteration counts
    assert iters["good"] != iters["identity"] and iters["poor"] != iters["identity"]


# ---- not converged
def test_not_converged_frames_leave_the_state_alone(synth, oracle, filt):
    params, max_it = GICP, 4
    # 1 m steps converge from the previous pose within the cap of 4 iterations, the 3 m jump 6 -> 9 does not, and the frame after the
    # rejection is aligned from the OLD prev_trans against the OLD keyframe
    idx = [0, 1, 2, 5, 3, 4, 5, 6, 9, 7]
    clouds = line_frames(synth, idx)
    stamps = stamps_of(len(idx))
    odo_kw = dict(keyframe_delta_trans=2.5, keyframe_delta_angle=BIG, keyframe_delta_time=BIG, publish_status=True)
    p = dict(params, reg_maximum_iterations=max_it)
    want, log = replay_walk(gicp_align(oracle, max_iterations=max_it), odo_kw, clouds, stamps)
    taken_and_not([not w["converged"] for w in want[1:]], "not converged")
    taken_and_not([w["keyframe_updated"] for w in want[1:]], "keyframe switch")
    assert all(w["frame_rejected"] == (not w["converged"]) for w in want[1:])
    k = next(i for i, w in enumerate(want) if i and w["frame_rejected"])
    assert k + 1 < len(want) and want[k + 1]["keyframe"] is want[k]["keyframe"] and np.array_equal(log[k + 1]["guess"], log[k]["guess"])
    sts = engine_walk(p, odo_kw, clouds, stamps)
    compare(sts, with_clouds(want, clouds), 1e-6, gicp_fitness(oracle))  # publish_status on rejected frames: the failed align's pose
    assert all(np.isfinite(s["matching_error"]) for s in sts[1:])
    variants_agree(p, odo_kw, clouds, stamps, sts, None, filt)


# ---- transform thresholding
def test_thresholding_by_translation(synth, oracle, filt):
    idx = [0, 1, 2, 4, 3, 4, 5, 7, 6, 7]  # steps of 1 m and, twice, 2 m: the limit lies midway
    clouds = line_frames(synth, idx)
    stamps = stamps_of(len(idx))
    odo_kw = dict(keyframe_delta_trans=3.5, keyframe_delta_angle=BIG, keyframe_delta_time=BIG, transform_thresholding=True,
                  max_acceptable_trans=1.5, max_acceptable_angle=BIG)
    want, log = replay_walk(gicp_align(oracle), odo_kw, clouds, stamps)
    assert all(w["converged"] for w in want[1:])
    dx = [r["dx"] for r in log[1:]]
    taken_and_not([d > 1.5 for d in dx], "dx over the limit")
    assert min(abs(d - 1.5) for d in dx) > 0.3  # midway between the two groups of observed steps
    assert [w["frame_rejected"] for w in want[1:]] == [d > 1.5 for d in dx]
    taken_and_not([w["keyframe_updated"] for w in want[1:]], "keyframe switch")
    sts = engine_walk(GICP, odo_kw, clouds, stamps)
    compare(sts, want, 1e-6)
    variants_agree(GICP, odo_kw, clouds, stamps, sts, None, filt)
    # switched off, tiny limits reject nothing
    off = dict(odo_kw, transform_thresholding=False, max_acceptable_trans=1e-9, max_acceptable_angle=1e-9)
    sts_off = engine_walk(GICP, off, clouds, stamps)
    compare(sts_off, replay_walk(gicp_align(oracle), off, clouds, stamps)[0], 1e-6)
    assert not any(s["frame_rejected"] for s in sts_off)


YAWS = [0, 2, 4, 12, 6, 8, 10, 18, 12, 14]  # turns of 2 degrees and, twice, 8 degrees


def test_thresholding_by_angle(synth, oracle, filt):
    clouds = yaw_frames(synth, YAWS)
    stamps = stamps_of(len(YAWS))
    lim = np.deg2rad(5.0) / 2  # acos(w) is half the rotation angle: between the 2 and the 8 degree turns
    odo_kw = dict(KF_OFF, transform_thresholding=True, max_acceptable_trans=BIG, max_acceptable_angle=lim)
    want, log = replay_walk(gicp_align(oracle), odo_kw, clouds, stamps)
    assert all(w["converged"] for w in want[1:])
    da = [r["da"] for r in log[1:]]
    taken_and_not([a > lim for a in da], "da over the limit")
    assert [w["frame_rejected"] for w in want[1:]] == [a > lim for a in da]
    sts = engine_walk(GICP, odo_kw, clouds, stamps)
    compare(sts, want, 1e-6)
    variants_agree(GICP, odo_kw, clouds, stamps, sts)


# ---- the three keyframe criteria
def test_keyframe_switch_by_angle_alone(synth, oracle, filt):
    yaws = [3 * k for k in range(9)]
    clouds = yaw_frames(synth, yaws)
    stamps = stamps_of(len(yaws))
    odo_kw = dict(keyframe_delta_trans=BIG, keyframe_delta_angle=np.deg2rad(7.0) / 2, keyframe_delta_time=BIG)
    want, log = replay_walk(gicp_align(oracle), odo_kw, clouds, stamps)
    taken_and_not([r["by_angle"] for r in log[1:]], "switch by angle")
    assert not any(r["by_trans"] or r["by_time"] for r in log[1:])
    sts = engine_walk(GICP, odo_kw, clouds, stamps)
    compare(sts, want, 1e-6)
    assert [s["keyframe_updated"] for s in sts[1:]] == [r["by_angle"] for r in log[1:]]
    variants_agree(GICP, odo_kw, clouds, stamps, sts, None, filt)


def test_keyframe_switch_by_time_alone_and_by_two_criteria(synth, oracle, filt):
    idx = list(range(8))
    clouds = line_frames(synth, idx)
    stamps = stamps_of(len(idx))
    by_time = dict(keyframe_delta_trans=BIG, keyframe_delta_angle=BIG, keyframe_delta_time=0.25)
    want, log = replay_walk(gicp_align(oracle), by_time, clouds, stamps)
    taken_and_not([r["by_time"] for r in log[1:]], "switch by time")
    assert not any(r["by_trans"] or r["by_angle"] for r in log[1:])
    sts = engine_walk(GICP, by_time, clouds, stamps)
    compare(sts, want, 1e-6)
    variants_agree(GICP, by_time, clouds, stamps, sts, None, filt)
    both = dict(keyframe_delta_trans=1.5, keyframe_delta_angle=BIG, keyframe_delta_time=0.15)
    want, log = replay_walk(gicp_align(oracle), both, clouds, stamps)
    assert any(r["by_trans"] and r["by_time"] for r in log[1:]) and any(not (r["by_trans"] or r["by_time"]) for r in log[1:])
    compare(engine_walk(GICP, both, clouds, stamps), want, 1e-6)


# ---- a large cloud
def test_branches_at_65536_points(synth, oracle):
    idx = [0, 1, 2, 4, 3, 4, 5, 7]
    clouds = line_frames(synth, idx, "vlp16")
    assert clouds[0].shape[0] == 65536
    stamps = stamps_of(len(idx))
    odo_kw = dict(keyframe_delta_trans=2.5, keyframe_delta_angle=BIG, keyframe_delta_time=BIG, transform_thresholding=True,
                  max_acceptable_trans=1.5, max_acceptable_angle=BIG)
    want, log = replay_walk(gicp_align(oracle), odo_kw, clouds, stamps)
    taken_and_not([w["frame_rejected"] for w in want[1:]], "rejection")
    taken_and_not([w["keyframe_updated"] for w in want[1:]], "keyframe switch")
    sts = engine_walk(GICP, odo_kw, clouds, stamps)
    compare(sts, want, 1e-6)
    assert_same(engine_walk(GICP, odo_kw, clouds, stamps, device=True, announce=True), sts)


# ---- NDT handles: a rejected frame leaves the voxel-map target in place
@pytest.mark.parametrize("method", ["ndt_omp", "ndt"])
def test_ndt_walks(synth, oracle, filt, tmp_path, method):
    idx = [0, 1, 2, 4, 3, 4]
    clouds = line_frames(synth, idx)
    stamps = stamps_of(len(idx))
    if method == "ndt_omp":
        params = NDT_OMP
        align = lambda c, kf, g: oracle.NdtMap(kf, 1.0).align(c, g)  # noqa: E731
    else:
        params = NDT_PCL
        pcl = Reference(tmp_path)
        align = lambda c, kf, g: pcl.map(kf, 1.0).align(c, g)  # noqa: E731
    # these aligns move by different amounts per frame (millimetres); the keyframes switch on time, and the limit is put midway between
    # two neighbouring steps that a walk without thresholding observes: the first such limit whose own walk rejects some frames,
    # accepts others and keeps every step further from the limit than the pose tolerance
    free = dict(keyframe_delta_trans=BIG, keyframe_delta_angle=BIG, keyframe_delta_time=0.25)
    _, log = replay_walk(align, free, clouds, stamps)
    dx = sorted(r["dx"] for r in log[1:] if r["converged"])
    want = None
    for lo, hi in zip(dx, dx[1:]):
        odo_kw = dict(free, transform_thresholding=True, max_acceptable_trans=0.5 * (lo + hi), max_acceptable_angle=BIG)
        w, log = replay_walk(align, odo_kw, clouds, stamps)
        rej = [x["frame_rejected"] for x in w[1:]]
        if any(rej) and not all(rej) and min(abs(r["dx"] - odo_kw["max_acceptable_trans"]) for r in log[1:] if r["converged"]) > 3e-4:
            want = w
            break
    assert want is not None, dx
    taken_and_not([w["frame_rejected"] for w in want[1:]], "rejection")
    taken_and_not([w["keyframe_updated"] for w in want[1:]], "keyframe switch")
    k = next(i for i, w in enumerate(want) if i and w["frame_rejected"])
    assert k + 1 < len(want) and want[k + 1]["keyframe"] is want[k]["keyframe"]
    sts = engine_walk(params, odo_kw, clouds, stamps)
    compare(sts, want, 1e-4)
    variants_agree(params, odo_kw, clouds, stamps, sts, None, filt if method == "ndt_omp" else None)
