"""GPU: FAST_VGICP (B2R_METHOD_VGICP) against the sequential reference tests/vgicp_ref.cpp, and every entry point against the single
handle.  Voxel cells, counts, means and per-point correspondences are bit-exact; voxel covariances within 1e-8; H / b / cost within
rel 1e-9; aligns have the reference's iteration count and flag and a pose within 1e-6; fitness is b2r_fitness's bit for bit."""
import numpy as np
import pytest

import hdl_graph_slam_b200 as pkg
import vgicp_ref as vr
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return vr.Reference(tmp_path_factory.mktemp("vgicp_ref"))


def handle(res=1.0, **extra):
    p = {"registration_method": "FAST_VGICP", "reg_resolution": str(res)}
    p.update({k: str(v) for k, v in extra.items()})
    return pkg.select_registration_method(p)


def scene(n_t=12000, n_s=9000, seed=0, T=None):
    tgt = vr.room(n_t, seed=seed)
    src = vr.moved(vr.room(n_s, seed=seed + 1), vr.rigid(0.03, [0.25, -0.1, 0.03]) if T is None else T)
    return tgt, src


def test_factory_and_defaults():
    r = handle()
    c = r.config
    assert c.method == pkg.B2R_METHOD_VGICP and c.ndt_resolution == 1.0 and c.max_iterations == 64 and c.k_correspondences == 20
    assert c.transformation_epsilon == 0.01 and c.rotation_epsilon == 2e-3
    r.close()
    r = pkg.select_registration_method({"registration_method": "FAST_VGICP", "reg_resolution": "0.5", "reg_maximum_iterations": "7",
                                        "reg_correspondence_randomness": "15", "reg_max_correspondence_distance": "9.0"})
    c = r.config
    assert (c.ndt_resolution, c.max_iterations, c.k_correspondences, c.max_correspondence_distance) == (0.5, 7, 15, 2.5)
    r.close()
    with pytest.raises(pkg.B2RError):
        pkg.select_registration_method({"registration_method": "FAST_VGICP_CUDA"})


@pytest.mark.parametrize("res", [0.25, 0.5, 1.0, 2.0])
def test_voxels_and_linearisation_match_the_reference(ref, res):
    tgt, src = scene(seed=res.__hash__() % 7)
    r = handle(res)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    tcov = r.getCovariances(1, tgt.shape[0])
    scov = r.getCovariances(0, src.shape[0])
    m = ref.map(tgt, res, tcov)
    want = m.voxels()
    got = r.vgicpGetVoxels()
    assert np.array_equal(got["cells"], want["cells"]) and np.array_equal(got["counts"], want["counts"])
    assert np.array_equal(got["mean"], want["mean"])
    assert np.max(np.abs(got["cov"] - want["cov"])) <= 1e-8
    for T in (np.eye(4), vr.rigid(0.02, [0.2, -0.05, 0.01])):
        H, b, cost, nc, vox = r.vgicpLinearizeAt(T, src.shape[0])
        Hr, br, cr, vr_ = m.linearize(src, T, scov)
        assert np.array_equal(vox, vr_) and nc == int((vr_ >= 0).sum()) and nc > 0
        assert abs(cost - cr) <= 1e-9 * abs(cr)
        assert np.max(np.abs(H - Hr)) <= 1e-9 * np.max(np.abs(Hr)) and np.max(np.abs(b - br)) <= 1e-9 * np.max(np.abs(br))
        assert np.array_equal(r.getCorrespondences(src.shape[0]), vox)
    r.close()


@pytest.mark.parametrize("n_t,n_s,res", [(12000, 9000, 1.0), (40000, 30000, 0.5), (262144, 131072, 1.0)])
def test_align_matches_the_reference(ref, n_t, n_s, res):
    tgt, src = scene(n_t, n_s, seed=3)
    r = handle(res)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    m = ref.map(tgt, res, r.getCovariances(1, tgt.shape[0]))
    o = m.align(src, scov=r.getCovariances(0, src.shape[0]))
    r.align(np.eye(4, dtype=np.float32))
    assert r.nr_iterations == o["iterations"] and r.hasConverged() == o["converged"]
    assert np.max(np.abs(r.getFinalTransformation().astype(np.float64) - o["T"])) <= 1e-6
    # getFitnessScore after the align: the target nearest-neighbour fitness at the final float pose, against the CPU oracle's
    want = orc.fitness(tgt, src, r.getFinalTransformation(), 2.5)[0]
    assert abs(r.getFitnessScore(2.5) - want) <= 1e-12 * want
    r.close()


def test_batch_loop_matching_and_single_handle_agree_bitwise():
    clouds = [vr.room(n, seed=s) for n, s in ((12000, 10), (7000, 11), (15000, 12), (3000, 13), (0, 0))]
    clouds[4] = np.zeros((0, 4), np.float32)
    guesses = [np.eye(4, dtype=np.float32), vr.rigid(0.02, [0.1, 0, 0]).astype(np.float32), vr.rigid(-0.03, [0, 0.2, 0]).astype(np.float32),
               np.eye(4, dtype=np.float32)]
    # single handle
    single = []
    for k in range(1, 5):
        r = handle()
        r.setInputTarget(clouds[0])
        r.setInputSource(clouds[k])
        r.align(guesses[k - 1])
        fit = r.getFitnessScore(2.5) if clouds[k].shape[0] else np.finfo(np.float64).max
        single.append((r.getFinalTransformation(), r.hasConverged(), r.nr_iterations, fit))
        r.close()
    # batch, co-scheduled (mixed sizes and an empty source) and alone
    b = pkg.RegistrationBatch(params={"registration_method": "FAST_VGICP"})
    ids = [b.addCloud(c) for c in clouds]
    together = b.align([(ids[k], ids[0], guesses[k - 1]) for k in range(1, 5)], True, 2.5)
    alone = [b.align([(ids[k], ids[0], guesses[k - 1])], True, 2.5)[0] for k in range(1, 5)]
    b.close()
    # the loop detector's matching
    best, loop = pkg.LoopDetector(handle(), fitness_score_max_range=2.5, fitness_score_thresh=10.0).matching(clouds[1:5], clouds[0], guesses)
    for k in range(4):
        T, conv, it, fit = single[k]
        for got in (together[k], alone[k], loop[k]):
            assert np.array_equal(got["T"], T) and got["converged"] == conv and got["iterations"] == it
            assert np.float64(got["fitness"]).tobytes() == np.float64(fit).tobytes()
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
    # the same state machine on the host around single aligns (no keyframe promotion: the keyframe is set as a target again)
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
