"""GPU parity of the NDT path (ndt_omp semantics, SURVEY.md A.2/A.3) against the CPU oracle, through the C ABI.

Tolerances: voxel keys / point counts / validity set, voxel means and inverse covariances, and the number of (point, cell) pairs
bit-exact; score, gradient, Hessian of one derivative pass rel <= 1e-9 (the per-pair float32 math follows the
oracle's operation order exactly, only the float64 summation tree differs); final pose <= 1e-4 m / 1e-4 rad and the same
iteration count."""
import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg
from common import rot_err, trans_err, perturb, relrel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pair(synth):
    return synth.scan("vlp16_16k", frame=1, stride=8), synth.scan("vlp16_16k", frame=0, stride=8)


def make(res, search="DIRECT7", **kw):
    params = {"registration_method": "NDT_OMP", "reg_resolution": res, "reg_nn_search_method": search}
    params.update(kw)
    return pkg.select_registration_method(params)


def test_factory_defaults():
    r = pkg.select_registration_method({})  # registrations.cpp:26 default "NDT_OMP", :93 resolution 0.5, :103 DIRECT7
    c = r.config
    assert c.method == pkg.B2R_METHOD_NDT and c.ndt_resolution == 0.5 and c.ndt_search_method == 7
    assert c.max_iterations == 64 and c.transformation_epsilon == 0.01 and c.ndt_step_size == 0.1 and c.ndt_outlier_ratio == 0.55
    r.close()
    with pytest.raises(pkg.B2RError) as e:
        pkg.select_registration_method({"registration_method": "ICP"})
    assert e.value.code == -5
    with pytest.raises(pkg.B2RError):
        pkg.select_registration_method({"registration_method": "NDT_OMP", "reg_nn_search_method": "KDTREE"})


@pytest.mark.parametrize("res", [1.0, 0.5, 0.7])
def test_voxel_map(pair, oracle, res):
    src, tgt = pair
    r = make(res)
    r.setInputTarget(tgt)
    got = r.ndtGetVoxels()
    want = oracle.NdtMap(tgt, res).dump()
    assert np.array_equal(got["min_b"], want["min_b"]) and np.array_equal(got["div_b"], want["div_b"])
    assert np.array_equal(got["keys"], want["keys"])
    assert np.array_equal(got["npts"], want["npts"])
    assert np.max(np.abs(got["mean"] - want["mean"])) == 0.0
    valid = want["npts"] >= 6
    assert valid.sum() > 100
    assert np.array_equal(got["icov"], want["icov"])  # the finalisation is the oracle's unfused float64 sequence
    r.close()


@pytest.mark.parametrize("search", ["DIRECT7", "DIRECT1"])
def test_derivatives(pair, oracle, search):
    src, tgt = pair
    r = make(1.0, search)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    om = oracle.NdtMap(tgt, 1.0)
    sm = 7 if search == "DIRECT7" else 1
    for p in ([0, 0, 0, 0, 0, 0], [0.9, 0.05, -0.02, 0.01, -0.015, 0.03], [1.0, 0.0, 0.0, 3.1, 3.13, -3.1]):
        score, g, H, npairs = r.ndtDerivativesAt(p)
        o = om.derivatives(src, p, search_method=sm)
        assert npairs == o["n_pairs"] and npairs > 1000
        assert abs(score - o["score"]) <= 1e-9 * abs(o["score"])
        assert relrel(g, o["g"]) < 1e-9 and relrel(H, o["H"]) < 1e-9
    r.close()


def test_derivative_pass_is_bitwise_reproducible(synth):
    """The pass hands its 128-point chunks out through a ticket counter (whichever block is free takes the next one); every chunk owns a row
    of sums and the rows are added by a fixed tree, so the result must not depend on the scheduling: repeated passes, passes after a pass on
    a cloud of another size (counters / ticket base carried over), and a second handle all give the same bits."""
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)
    srcs = [synth.scan("vlp16_16k", frame=1, stride=8), synth.scan("vlp16", frame=1, stride=8), synth.scan("vlp16_16k", frame=2, stride=8)]
    p = [0.9, 0.05, -0.02, 0.01, -0.015, 0.03]
    r = make(1.0)
    r.setInputTarget(tgt)
    ref = {}
    for rep in range(3):
        for k, src in enumerate(srcs):
            r.setInputSource(src)
            for _ in range(2):
                score, g, H, npairs = r.ndtDerivativesAt(p)
                got = (np.float64(score).tobytes(), np.asarray(g).tobytes(), np.asarray(H).tobytes(), int(npairs))
                if k in ref:
                    assert got == ref[k], f"pass on cloud {k} differs from its first run (rep {rep})"
                ref[k] = got
    r2 = make(1.0)
    r2.setInputTarget(tgt)
    r2.setInputSource(srcs[1])
    score, g, H, npairs = r2.ndtDerivativesAt(p)
    assert (np.float64(score).tobytes(), np.asarray(g).tobytes(), np.asarray(H).tobytes(), int(npairs)) == ref[1]
    r.close(); r2.close()


@pytest.mark.parametrize("case", [0, 1, 2, 3])
def test_align_matches_oracle(pair, oracle, case):
    src, tgt = pair
    res, search, guess = [(1.0, "DIRECT7", None), (1.0, "DIRECT7", 11), (0.5, "DIRECT1", 12), (1.0, "DIRECT1", 13)][case]
    G = (np.eye(4) if guess is None else perturb(guess, 0.3, 1.5)).astype(np.float32)
    r = make(res, search)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    r.align(G)
    o = oracle.NdtMap(tgt, res).align(src, G, search_method=7 if search == "DIRECT7" else 1)
    T = r.getFinalTransformation()
    assert r.hasConverged() == o["converged"]
    assert r.nr_iterations == o["iterations"]
    assert trans_err(T, o["T"]) < 1e-4 and rot_err(T, o["T"]) < 1e-4
    r.close()


def test_fixed_iterations_and_line_search_switch(pair, oracle):
    src, tgt = pair
    for flag, fixed in ((0, 30), (1, 0)):
        cfg = pkg.default_config(pkg.B2R_METHOD_NDT)
        cfg.ndt_resolution = 1.0
        cfg.ndt_fixed_iterations = fixed
        cfg.ndt_mt_interval_flag = flag
        r = pkg.Registration(cfg)
        r.setInputTarget(tgt)
        r.setInputSource(src)
        G = perturb(21, 0.3, 1.5).astype(np.float32)
        r.align(G)
        o = oracle.NdtMap(tgt, 1.0).align(src, G, fixed_iterations=fixed, mt_interval_flag=flag)
        T = r.getFinalTransformation()
        if fixed:
            assert r.nr_iterations == fixed == o["iterations"]
        else:
            assert r.nr_iterations == o["iterations"]
        assert trans_err(T, o["T"]) < 1e-4 and rot_err(T, o["T"]) < 1e-4
        r.close()


def test_fitness_through_ndt_handle(pair, oracle):
    src, tgt = pair
    r = make(1.0)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    r.align(np.eye(4, dtype=np.float32))
    T = r.getFinalTransformation()
    score, used, inl = r.getFitnessScore(full=True)
    os_, on, oi = oracle.fitness(tgt, src, T)
    assert used == on and inl == oi and abs(score - os_) <= 1e-12 * abs(os_)
    r.close()


def test_large_extent_at_factory_resolution(pair, oracle):
    """reg_resolution = 0.5 (the factory default, registrations.cpp:93) over a 300 m x 300 m extent: 600 x 600 x ~50 = 18 M cells.
    The reference's VoxelGridCovariance keeps its leaves in a map and is limited only by int32 indices; the engine's voxel map is
    sparse too (sorted keys + hash table), so this must simply work — same voxels, same derivative pass, same align."""
    src, tgt = pair
    far = np.zeros((64, tgt.shape[1]), np.float32)
    rng = np.random.default_rng(5)
    far[:, 0] = np.where(np.arange(64) % 2 == 0, 150.0, -150.0) + rng.uniform(-0.2, 0.2, 64)
    far[:, 1] = np.where((np.arange(64) // 2) % 2 == 0, 150.0, -150.0) + rng.uniform(-0.2, 0.2, 64)
    far[:, 2] = rng.uniform(-0.2, 0.2, 64)
    far[:, 3] = 1.0
    big = np.concatenate([tgt, far]).astype(np.float32)
    r = make(0.5)
    r.setInputTarget(big)
    got = r.ndtGetVoxels()
    m = oracle.NdtMap(big, 0.5)
    want = m.dump()
    assert int(np.prod(want["div_b"].astype(np.int64))) > (1 << 23)  # beyond the old dense-table capacity
    assert np.array_equal(got["div_b"], want["div_b"]) and np.array_equal(got["keys"], want["keys"]) and np.array_equal(got["npts"], want["npts"])
    r.setInputSource(src)
    p = np.array([0.1, -0.05, 0.02, 0.005, -0.01, 0.02])
    score, g, H, npairs = r.ndtDerivativesAt(p)
    o = m.derivatives(src, p)
    assert npairs == o["n_pairs"] and abs(score - o["score"]) <= 1e-9 * abs(o["score"])
    assert relrel(g, o["g"]) < 1e-9 and relrel(H, o["H"]) < 1e-9
    r.align(np.eye(4, dtype=np.float32))
    oa = m.align(src, np.eye(4, dtype=np.float32))
    assert r.hasConverged() == oa["converged"] and r.nr_iterations == oa["iterations"]
    assert trans_err(r.getFinalTransformation(), oa["T"]) < 1e-4 and rot_err(r.getFinalTransformation(), oa["T"]) < 1e-4
    r.close()
