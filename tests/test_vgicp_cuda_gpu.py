"""GPU: B200_VGICP_CUDA (B2R_METHOD_VGICP_CUDA, fast_gicp::FastVGICPCuda) against the sequential reference tests/vgicp_cuda_ref.cpp, and
every entry point against the single handle.  Covariances, voxel cells, counts, means, covariances and per-point correspondences are
bit-exact; H / b / cost within rel 1e-9; aligns have the reference's iteration count and flag and a pose within 1e-6; fitness is
b2r_fitness's bit for bit."""
import numpy as np
import pytest

import hdl_graph_slam_b200 as pkg
import vgicp_cuda_ref as vc
import vgicp_ref as vr
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return vc.Reference(tmp_path_factory.mktemp("vgicp_cuda_ref"))


def handle(res=1.0, **extra):
    p = {"registration_method": "B200_VGICP_CUDA", "reg_resolution": str(res)}
    p.update({k: str(v) for k, v in extra.items()})
    return pkg.select_registration_method(p)


def scene(n_t=12000, n_s=9000, seed=0, T=None, offset=None):
    tgt = vr.room(n_t, seed=seed)
    src = vr.moved(vr.room(n_s, seed=seed + 1), vr.rigid(0.03, [0.25, -0.1, 0.03]) if T is None else T)
    if offset is not None:
        tgt = vr.records(tgt[:, :3].astype(np.float64) + offset)
        src = vr.records(src[:, :3].astype(np.float64) + offset)
    return tgt, src


def test_factory_and_defaults():
    r = handle()
    c = r.config
    assert c.method == pkg.B2R_METHOD_VGICP_CUDA == 6 and c.ndt_resolution == 1.0 and c.max_iterations == 64 and c.k_correspondences == 20
    assert c.transformation_epsilon == 0.01 and c.rotation_epsilon == 2e-3
    r.close()
    r = pkg.select_registration_method({"registration_method": "B200_VGICP_CUDA", "reg_resolution": "0.5", "reg_maximum_iterations": "7",
                                        "reg_transformation_epsilon": "0.001", "reg_correspondence_randomness": "15",
                                        "reg_max_correspondence_distance": "9.0"})
    c = r.config
    assert (c.ndt_resolution, c.max_iterations, c.transformation_epsilon, c.k_correspondences, c.max_correspondence_distance) == (0.5, 7, 0.001, 15, 2.5)
    r.close()
    for name in ("FAST_VGICP_CUDA", "GICP_OMP", "ICP"):
        with pytest.raises(pkg.B2RError):
            pkg.select_registration_method({"registration_method": name})
    with pytest.raises(pkg.B2RError):
        handle(0.0)


@pytest.mark.parametrize("res", [0.25, 0.5, 1.0, 2.0])
def test_voxels_and_linearisation_match_the_reference(ref, res):
    tgt, src = scene(seed=int(res * 4) % 7)
    r = handle(res)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    tcov = r.getCovariances(1, tgt.shape[0])
    scov = r.getCovariances(0, src.shape[0])
    assert np.array_equal(tcov, ref.covariances(tgt)) and np.array_equal(scov, ref.covariances(src))
    m = ref.map(tgt, res, tcov)
    want = m.voxels()
    got = r.vgicpGetVoxels()
    for key in ("cells", "counts", "mean", "cov"):
        assert np.array_equal(got[key], want[key]), key
    for T in (np.eye(4), vr.rigid(0.02, [0.2, -0.05, 0.01])):
        H, b, cost, nc, vox = r.vgicpLinearizeAt(T, src.shape[0])
        Hr, br, cr, vr_ = m.linearize(src, T, scov)
        assert np.array_equal(vox, vr_) and nc == int((vr_ >= 0).sum()) and nc > 0
        assert abs(cost - cr) <= 1e-9 * abs(cr)
        assert np.max(np.abs(H - Hr)) <= 1e-9 * np.max(np.abs(Hr)) and np.max(np.abs(b - br)) <= 1e-9 * np.max(np.abs(br))
        assert np.array_equal(r.getCorrespondences(src.shape[0]), vox)
    r.close()


@pytest.mark.parametrize("n_t,n_s,res,offset", [(12000, 9000, 1.0, None), (40000, 30000, 0.5, None), (262144, 131072, 1.0, None),
                                               (12000, 9000, 1.0, (3000.0, -2000.0, 50.0))])
def test_align_matches_the_reference(ref, n_t, n_s, res, offset):
    tgt, src = scene(n_t, n_s, seed=3, offset=None if offset is None else np.array(offset))
    r = handle(res)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    tcov, scov = r.getCovariances(1, tgt.shape[0]), r.getCovariances(0, src.shape[0])
    if n_t <= 40000:
        assert np.array_equal(scov, ref.covariances(src))
    m = ref.map(tgt, res, tcov)
    o = m.align(src, scov=scov)
    r.align(np.eye(4, dtype=np.float32))
    assert r.nr_iterations == o["iterations"] and r.hasConverged() == o["converged"]
    assert np.max(np.abs(r.getFinalTransformation().astype(np.float64) - o["T"])) <= 1e-6
    want = orc.fitness(tgt, src, r.getFinalTransformation(), 2.5)[0]
    assert abs(r.getFitnessScore(2.5) - want) <= 1e-12 * want
    r.close()


def test_far_from_origin_covariances_are_not_fast_vgicps(ref):
    """at (3000, -2000, 50) the float32 raw moments part from FastGICP's covariances (the FAST_VGICP handle's), bit for bit the reference's"""
    _, src = scene(12000, 9000, seed=5, offset=np.array([3000.0, -2000.0, 50.0]))
    a, b = handle(), pkg.select_registration_method({"registration_method": "FAST_VGICP"})
    for r in (a, b):
        r.setInputTarget(src)
        r.setInputSource(src)
    ca, cb = a.getCovariances(0, src.shape[0]), b.getCovariances(0, src.shape[0])
    assert np.array_equal(ca, ref.covariances(src))
    assert np.max(np.abs(ca - cb)) > 0.1
    a.close()
    b.close()


def test_batch_loop_matching_and_single_handle_agree_bitwise():
    clouds = [vr.room(n, seed=s) for n, s in ((12000, 10), (7000, 11), (15000, 12), (3000, 13), (0, 0))]
    clouds[4] = np.zeros((0, 4), np.float32)
    guesses = [np.eye(4, dtype=np.float32), vr.rigid(0.02, [0.1, 0, 0]).astype(np.float32), vr.rigid(-0.03, [0, 0.2, 0]).astype(np.float32),
               np.eye(4, dtype=np.float32)]
    single = []
    for k in range(1, 5):
        r = handle()
        r.setInputTarget(clouds[0])
        r.setInputSource(clouds[k])
        r.align(guesses[k - 1])
        fit = r.getFitnessScore(2.5) if clouds[k].shape[0] else np.finfo(np.float64).max
        single.append((r.getFinalTransformation(), r.hasConverged(), r.nr_iterations, fit))
        r.close()
    b = pkg.RegistrationBatch(params={"registration_method": "B200_VGICP_CUDA"})
    ids = [b.addCloud(c) for c in clouds]
    together = b.align([(ids[k], ids[0], guesses[k - 1]) for k in range(1, 5)], True, 2.5)
    alone = [b.align([(ids[k], ids[0], guesses[k - 1])], True, 2.5)[0] for k in range(1, 5)]
    fits = b.calcFitnessScore([(ids[0], ids[k], single[k - 1][0]) for k in range(1, 4)], 2.5)
    b.close()
    best, loop = pkg.LoopDetector(handle(), fitness_score_max_range=2.5, fitness_score_thresh=10.0).matching(clouds[1:5], clouds[0], guesses)
    for k in range(4):
        T, conv, it, fit = single[k]
        for got in (together[k], alone[k], loop[k]):
            assert np.array_equal(got["T"], T) and got["converged"] == conv and got["iterations"] == it
            assert np.float64(got["fitness"]).tobytes() == np.float64(fit).tobytes()
    for k in range(3):  # InformationMatrixCalculator::calc_fitness_score on the batch's cached clouds
        want = orc.fitness(clouds[0], clouds[k + 1], single[k][0], 2.5)[0]
        assert abs(fits[k] - want) <= 1e-12 * want
    assert best >= 0


@pytest.mark.parametrize("downsample", [0, 1])
@pytest.mark.parametrize("prefetch", [False, True])
def test_odometry_mirror_equals_a_host_loop_of_single_aligns(downsample, prefetch):
    frames = [vr.moved(vr.room(20000, seed=20 + i), vr.rigid(0.01 * i, [0.12 * i, 0.0, 0.0])) for i in range(6)]
    o = pkg.ScanMatchingOdometry(handle(), keyframe_delta_trans=0.25, publish_status=True, downsample_method=downsample, downsample_resolution=0.1)
    got = []
    for i, f in enumerate(frames):
        if prefetch and i + 1 < len(frames):
            o.prefetch_raw(frames[i + 1].ctypes.data, frames[i + 1].shape[0], 16)
        got.append(o.matching(0.1 * i, f))
    o.close()
    vg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    filt = (lambda c: vg.voxelGridFilter(c, 0.1)) if downsample else (lambda c: c)
    r = handle()
    prev = np.eye(4, dtype=np.float32)
    r.setInputTarget(filt(frames[0]))
    for i in range(1, len(frames)):
        c = filt(frames[i])
        r.setInputSource(c)
        r.align(prev)
        T = r.getFinalTransformation()
        g = got[i]
        assert np.array_equal(g["trans"], T) and g["converged"] == r.hasConverged() and g["iterations"] == r.nr_iterations
        assert g["matching_error"] == r.getFitnessScore()
        prev = T
        if g["keyframe_updated"]:
            r.setInputTarget(c)
            prev = np.eye(4, dtype=np.float32)
    assert any(g["keyframe_updated"] for g in got[1:])
    r.close()
    vg.close()
