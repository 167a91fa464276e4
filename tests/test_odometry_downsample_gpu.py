"""GPU: the odometry mirror's own downsample stage (ScanMatchingOdometryNodelet::downsample, downsample_method VOXELGRID /
APPROX_VOXELGRID / NONE, apps/scan_matching_odometry_nodelet.cpp:83-103,147-177).

- against the oracle: matching() replayed on the oracle's filtered clouds (voxel grid) or the sequential reference's
  (approximate voxel grid, tests/approx_voxelgrid_ref.cpp);
- bitwise against the same filter run first through b2r_voxelgrid_device / b2r_approximate_voxelgrid_device and the mirror
  with NONE, for host and device input, GICP and NDT handles;
- bitwise equal with and without b2r_odometry_prefetch, including an announced cloud that is not the one then passed and a
  host buffer rewritten in place after its announcement;
- b2r_prefilter's device output (which lives in the handle's voxel-grid buffer) fed to the mirror on the same handle;
- the leaf-too-small pass-through, unknown method values, invalid leaves, an all-non-finite frame and 262 144-point clouds."""
import numpy as np
import pytest
import torch  # before the engine library: it links the system NCCL, and torch's CUDA libraries must resolve against their own first
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi
from common import rot_err, trans_err

from approx_voxelgrid_ref import Reference

pytestmark = pytest.mark.gpu

VG, AVG, NONE = pkg.B2R_DOWNSAMPLE_VOXELGRID, pkg.B2R_DOWNSAMPLE_APPROX_VOXELGRID, pkg.B2R_DOWNSAMPLE_NONE
GICP = {"registration_method": "FAST_GICP"}
NDT = {"registration_method": "NDT_OMP", "reg_resolution": 1.0}
KF = dict(keyframe_delta_trans=1.5, keyframe_delta_angle=1.0, keyframe_delta_time=10000.0, publish_status=True)
# NDT_OMP moves these scans by millimetres per frame (small steps, transformation_epsilon 0.01): its keyframes switch on time
# (stamps 0.1 k: every third frame)
NDT_KF = dict(keyframe_delta_time=0.25)


def kf_of(params):
    return NDT_KF if params is NDT else {}


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("avg_ref"))


@pytest.fixture(scope="module")
def frames(synth):
    return [synth.scan("vlp16_16k", frame=k, stride=8) for k in range(7)]


def quat_w(R):
    return 0.5 * np.sqrt(max(np.float32(R[0, 0] + R[1, 1] + R[2, 2]) + np.float32(1.0), 0))


def to_device(cloud):
    d = torch.from_numpy(np.ascontiguousarray(cloud)).cuda()
    torch.cuda.synchronize()
    return d


def status_key(st):
    """every field of a status, as bits"""
    return (st["odom"].view(np.uint32).tobytes(), st["trans"].view(np.uint32).tobytes(), st["iterations"], st["converged"], st["keyframe_updated"],
            st["frame_rejected"], np.float64(st["matching_error"]).tobytes(), np.float32(st["inlier_fraction"]).tobytes())


def assert_switches(sts):
    """the first keyframe and at least one keyframe switch"""
    assert sum(s["keyframe_updated"] for s in sts) >= 2, [(s["converged"], s["iterations"], float(np.linalg.norm(s["trans"][:3, 3]))) for s in sts]


def assert_same(a, b):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert status_key(x) == status_key(y), k


def mirror(params, method, leaf, clouds, device=False, announce=None, **kw):
    """statuses of one odometry over `clouds`; announce(k) -> the cloud announced during call k (None: no announcement)"""
    reg = pkg.select_registration_method(dict(params))
    odo = pkg.ScanMatchingOdometry(reg, downsample_method=method, downsample_resolution=leaf, **dict(KF, **kw))
    keep = []
    out = []
    for k, c in enumerate(clouds):
        if announce is not None:
            nxt = announce(k)
            if nxt is not None:
                keep.append(nxt)
                if device:
                    odo.prefetch_raw(nxt.data_ptr(), nxt.shape[0], nxt.shape[1] * 4, device=True)
                else:
                    odo.prefetch_raw(nxt.ctypes.data, nxt.shape[0], nxt.shape[1] * 4)
        if device:
            out.append(odo.matching_raw(0.1 * k, c.data_ptr(), c.shape[0], c.shape[1] * 4, device=True))
        else:
            out.append(odo.matching(0.1 * k, c))
    odo.close()
    reg.close()
    return out


def host_chained(params, method, leaf, raws, **kw):
    """b2r_voxelgrid_device / b2r_approximate_voxelgrid_device, then the mirror with NONE on the filter's device output"""
    reg = pkg.select_registration_method(dict(params))
    odo = pkg.ScanMatchingOdometry(reg, **dict(KF, **kw))
    out = []
    for k, raw in enumerate(raws):
        d = to_device(raw)
        n, sb = d.shape[0], d.shape[1] * 4
        if method == VG:
            ptr, m, _ = reg.voxelGridFilterDevice(d.data_ptr(), n, sb, leaf)
        else:
            ptr, m = reg.approximateVoxelGridFilterDevice(d.data_ptr(), n, sb, leaf)
        out.append(odo.matching_raw(0.1 * k, ptr, m, sb, device=True))
        del d
    odo.close()
    reg.close()
    return out


# ---- 1. against the oracle
@pytest.mark.parametrize("method,leaf", [(VG, 0.1), (VG, 0.25), (AVG, 0.1), (AVG, 0.25)])
def test_gicp_sequence_matches_oracle(frames, oracle, ref, method, leaf):
    filt = [oracle.voxelgrid(f, leaf)[0] if method == VG else ref.approximate_voxelgrid(f, leaf)[0] for f in frames]
    sts = mirror(GICP, method, leaf, frames)
    keyframe, keyframe_pose, prev_trans = None, np.eye(4, dtype=np.float32), np.eye(4, dtype=np.float32)
    switches = 0
    for k, (cloud, st) in enumerate(zip(filt, sts)):
        if keyframe is None:
            keyframe = cloud
            assert st["keyframe_updated"] and np.array_equal(st["odom"], np.eye(4, dtype=np.float32))
            continue
        o = oracle.gicp_align(cloud, keyframe, prev_trans)
        assert st["converged"] == o["converged"] and st["iterations"] == o["iterations"], k
        assert trans_err(st["trans"], o["T"]) < 1e-6 and rot_err(st["trans"], o["T"]) < 1e-6, k
        fs, fn, fi = oracle.fitness(keyframe, cloud, o["T"])
        assert abs(st["matching_error"] - fs) <= 1e-6 * fs, k
        assert abs(st["inlier_fraction"] - fi / cloud.shape[0]) < 1e-6, k  # aligned->size() (:321): the filtered count
        trans = o["T"]
        odom = keyframe_pose @ trans
        prev_trans = trans
        if np.linalg.norm(trans[:3, 3]) > KF["keyframe_delta_trans"] or np.arccos(min(quat_w(trans[:3, :3]), 1.0)) > 1.0:
            keyframe, keyframe_pose, prev_trans = cloud, odom, np.eye(4, dtype=np.float32)
            switches += 1
            assert st["keyframe_updated"], k
        else:
            assert not st["keyframe_updated"], k
    assert switches >= 1


def test_ndt_sequence_matches_oracle(frames, oracle):
    leaf = 0.25
    filt = [oracle.voxelgrid(f, leaf)[0] for f in frames[:5]]
    sts = mirror(NDT, VG, leaf, frames[:5], publish_status=False, **NDT_KF)
    keyframe, kf_stamp, prev_trans = None, 0.0, np.eye(4, dtype=np.float32)
    switches = 0
    for k, (cloud, st) in enumerate(zip(filt, sts)):
        if keyframe is None:
            keyframe = cloud
            continue
        o = oracle.NdtMap(keyframe, 1.0).align(cloud, prev_trans)
        assert st["converged"] == o["converged"] and st["iterations"] == o["iterations"], k
        assert trans_err(st["trans"], o["T"]) < 1e-4 and rot_err(st["trans"], o["T"]) < 1e-4, k
        assert o["converged"]
        prev_trans = o["T"]
        if (np.linalg.norm(o["T"][:3, 3]) > KF["keyframe_delta_trans"] or np.arccos(min(quat_w(o["T"][:3, :3]), 1.0)) > 1.0
                or 0.1 * k - kf_stamp > NDT_KF["keyframe_delta_time"]):
            keyframe, kf_stamp, prev_trans = cloud, 0.1 * k, np.eye(4, dtype=np.float32)
            switches += 1
            assert st["keyframe_updated"], k
        else:
            assert not st["keyframe_updated"], k
    assert switches >= 1


# ---- 2. in-mirror == host-chained
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("params", [GICP, NDT], ids=["gicp", "ndt"])
@pytest.mark.parametrize("method", [VG, AVG], ids=["voxelgrid", "approx"])
def test_in_mirror_equals_host_chained(frames, method, params, device):
    clouds = [to_device(f) for f in frames] if device else frames
    got = mirror(params, method, 0.25, clouds, device=device, **kf_of(params))
    want = host_chained(params, method, 0.25, frames, **kf_of(params))
    assert_switches(got)
    assert_same(got, want)


# ---- 3. prefetch changes nothing
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("params", [GICP, NDT], ids=["gicp", "ndt"])
@pytest.mark.parametrize("method", [VG, AVG], ids=["voxelgrid", "approx"])
def test_prefetch_changes_nothing(frames, method, params, device):
    clouds = [to_device(f) for f in frames] if device else [f.copy() for f in frames]
    kw = kf_of(params)
    base = mirror(params, method, 0.25, clouds, device=device, **kw)
    assert_switches(base)
    # every next frame announced
    assert_same(mirror(params, method, 0.25, clouds, device=device, announce=lambda k: clouds[k + 1] if k + 1 < len(clouds) else None, **kw), base)
    # during call 2 a different cloud is announced than the one call 3 passes (same size and stride): it must be filtered afresh
    decoy = to_device(frames[5]) if device else frames[5].copy()
    assert_same(mirror(params, method, 0.25, clouds, device=device,
                       announce=lambda k: decoy if k == 2 else (clouds[k + 1] if k + 1 < len(clouds) else None), **kw), base)
    if not device:
        # one recycled host buffer: announced holding frame 5, rewritten in place with frame 4 before call 4 reads it
        buf = frames[5].copy()
        seq = list(clouds)
        seq[4] = buf
        reg = pkg.select_registration_method(dict(params))
        odo = pkg.ScanMatchingOdometry(reg, downsample_method=method, downsample_resolution=0.25, **dict(KF, **kw))
        got = []
        for k, c in enumerate(seq):
            if k + 1 < len(seq):
                nxt = seq[k + 1]
                odo.prefetch_raw(nxt.ctypes.data, nxt.shape[0], nxt.shape[1] * 4)
            got.append(odo.matching(0.1 * k, c) if c is not buf else odo.matching_raw(0.1 * k, buf.ctypes.data, buf.shape[0], buf.shape[1] * 4))
            if k == 3:
                buf[:] = frames[4]
        odo.close()
        reg.close()
        assert_same(got, base)


# ---- 4. the prefilter -> odometry chain on one handle
@pytest.mark.parametrize("method", [VG, AVG], ids=["voxelgrid", "approx"])
def test_prefilter_output_feeds_downsampling_mirror_on_one_handle(frames, method):
    """b2r_prefilter's device output lies in the handle's voxel-grid buffer (no outlier stage after the downsample): the mirror's
    own downsample on the same handle must not write there"""
    pre = dict(use_distance_filter=1, distance_near_thresh=1.0, distance_far_thresh=100.0, downsample_method=VG, downsample_resolution=0.1,
               outlier_removal_method=0)
    outs = []
    for copy in (False, True):
        reg = pkg.select_registration_method(dict(GICP))
        odo = pkg.ScanMatchingOdometry(reg, downsample_method=method, downsample_resolution=0.25, **KF)
        res = []
        for k, raw in enumerate(frames):
            d = to_device(raw)
            _, dptr, m = reg.prefilter_raw(d.data_ptr(), d.shape[0], d.shape[1] * 4, device=True, **pre)
            if copy:
                sep = torch.empty((max(m, 1), raw.shape[1]), dtype=torch.float32, device="cuda")
                torch.cuda.synchronize()
                from cuda.bindings import runtime as cudart
                err, = cudart.cudaMemcpy(sep.data_ptr(), dptr, m * raw.shape[1] * 4, cudart.cudaMemcpyKind.cudaMemcpyDeviceToDevice)
                assert int(err) == 0
                dptr = sep.data_ptr()
            res.append(odo.matching_raw(0.1 * k, dptr, m, raw.shape[1] * 4, device=True))
        outs.append(res)
        odo.close()
        reg.close()
    assert_switches(outs[1])
    assert_same(outs[0], outs[1])


# ---- 5. edge cases
def test_leaf_too_small_and_unknown_method_equal_none(frames):
    base = mirror(GICP, NONE, 0.1, frames)
    assert_same(mirror(GICP, VG, 1e-4, frames), base)  # extent / leaf overflows the int32 voxel index: the cloud passes through
    assert_same(mirror(GICP, VG, 1e-4, [to_device(f) for f in frames], device=True), base)
    assert_same(mirror(GICP, 7, 0.1, frames), base)    # unknown downsample_method: PassThrough
    assert_same(mirror(GICP, 7, float("nan"), frames), base)


def test_invalid_leaf_is_refused_at_create():
    reg = pkg.select_registration_method(dict(GICP))
    for method, leaf in [(AVG, 0.0), (AVG, float("nan")), (AVG, float("inf")), (AVG, -0.1), (VG, 0.0), (VG, float("nan"))]:
        with pytest.raises(_capi.B2RError) as e:
            pkg.ScanMatchingOdometry(reg, downsample_method=method, downsample_resolution=leaf)
        assert e.value.code == _capi.B2R_EINVAL
    reg.close()


@pytest.mark.parametrize("params", [GICP, NDT], ids=["gicp", "ndt"])
def test_all_nonfinite_frame_is_an_empty_source(frames, params):
    bad = frames[2].copy()
    bad[:, :3] = np.nan
    bad[::3, 0] = np.inf
    raws = [frames[0], frames[1], bad, frames[3]]
    got = mirror(params, VG, 0.25, raws, **kf_of(params))
    assert got[2]["frame_rejected"] and not got[2]["converged"]
    # the mirror with NONE on the filtered clouds, the all-non-finite frame's output being empty
    reg = pkg.select_registration_method(dict(GICP))
    filt = [reg.voxelGridFilter(f, 0.25) for f in raws]
    reg.close()
    assert filt[2].shape[0] == 0
    assert_same(got, mirror(params, NONE, 0.25, filt, **kf_of(params)))


def test_262k_clouds_take_the_launch_chain(synth):
    """262 144-point inputs: the voxel grid's multi-launch chain (beyond the one-cluster limit), with and without the prefetch"""
    raws = [synth.scan((64, 4096), frame=k, stride=8) for k in range(4)]
    want = host_chained(GICP, VG, 0.1, raws)
    clouds = [to_device(r) for r in raws]
    assert_same(mirror(GICP, VG, 0.1, clouds, device=True), want)
    assert_same(mirror(GICP, VG, 0.1, clouds, device=True, announce=lambda k: clouds[k + 1] if k + 1 < len(clouds) else None), want)
    assert_same(mirror(GICP, VG, 0.1, raws, announce=lambda k: raws[k + 1] if k + 1 < len(raws) else None), want)
