"""GPU: the covariance kernels at every k.  At k = 20 GICP and B200_VGICP_CUDA run the register kernel k_pcl_cov_reg; at any other k
(reg_correspondence_randomness takes 1..64) they run the generic k_pcl_cov, whose neighbour lists need more than 48 KB of shared
memory from k = 49 on, and the batch falls back to one build per cloud.  Covariances against tests/gicp_pcl_ref.cpp (GICP, within 1e-8)
and tests/vgicp_cuda_ref.cpp (B200_VGICP_CUDA, bit for bit) at k in {1 .. 64}, at cloud sizes from 1 point to beyond the one-cluster
limit, with non-finite points; then at k = 7 and 49 the prefetched source, promotion and a mixed-size batch against fresh single
handles bit for bit, and aligns of GICP, B200_VGICP_CUDA and FAST_VGICP against their references."""
import numpy as np
import pytest

import gicp_pcl_ref as gr
import hdl_graph_slam_b200 as pkg
import vgicp_cuda_ref as vc
import vgicp_ref as vr
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def refs(tmp_path_factory):
    return dict(GICP=gr.Reference(tmp_path_factory.mktemp("gicp_pcl_ref")), FAST_VGICP=vr.Reference(tmp_path_factory.mktemp("vgicp_ref")),
                B200_VGICP_CUDA=vc.Reference(tmp_path_factory.mktemp("vgicp_cuda_ref")))


def handle(method, k):
    p = {"registration_method": method, "reg_correspondence_randomness": str(k)}
    if "VGICP" in method:
        p["reg_resolution"] = "1.0"
    return pkg.select_registration_method(p)


def cloud(n, seed, bad=True):
    """a structured scene (uniform points below 8), with a few NaN / +-inf points when it has 33 or more"""
    if n < 8:
        rng = np.random.default_rng(seed)
        return np.c_[rng.uniform(-1, 1, (n, 3)), np.ones(n)].astype(np.float32)
    p = gr.scene(n, seed=seed)
    if bad and n >= 33:
        p[3::max(n // 5, 1), 0] = np.nan
        p[7::max(n // 4, 1), 1] = np.inf
        p[11::max(n // 3, 1), 2] = -np.inf
    return p


def check_covariances(refs, method, pts, k, got):
    want = refs[method].covariances(pts, k)
    fin = np.isfinite(pts[:, :3]).all(axis=1)
    assert np.isnan(got[~fin]).all() and np.isnan(want[~fin]).all()
    if method == "GICP":
        assert np.max(np.abs(got[fin] - want[fin]), initial=0.0) <= 1e-8
    else:
        assert np.array_equal(got[fin], want[fin])


@pytest.mark.parametrize("k", [1, 2, 3, 7, 19, 21, 48, 49, 64])
@pytest.mark.parametrize("method", ["GICP", "B200_VGICP_CUDA"])
def test_covariances_at_every_k(refs, method, k):
    pts = cloud(16384, seed=k)
    r = handle(method, k)
    r.setInputSource(pts)
    check_covariances(refs, method, pts, k, r.getCovariances(0, pts.shape[0]))
    r.close()


@pytest.mark.parametrize("n", [1, 5, 33, 1025, 65537, 131073])
@pytest.mark.parametrize("k", [3, 49])
@pytest.mark.parametrize("method", ["GICP", "B200_VGICP_CUDA"])
def test_covariances_at_every_size(refs, method, k, n):
    pts = cloud(n, seed=n % 97)
    r = handle(method, k)
    r.setInputTarget(pts)
    check_covariances(refs, method, pts, k, r.getCovariances(1, n))
    r.close()


def scenes(method, sizes, seed):
    """clouds of the method's usual scene, each seen from a slightly different pose"""
    out = []
    for i, n in enumerate(sizes):
        if method == "GICP":
            out.append(gr.transform(gr.scene(n, seed=seed + i), gr.pose((0.1 * i, -0.05 * i, 0.0), (0.0, 0.0, 0.01 * i))))
        else:
            out.append(vr.moved(vr.room(n, seed=seed + i), vr.rigid(0.01 * i, [0.1 * i, -0.05 * i, 0.0])))
    return out


def aligned(r, guess):
    r.align(guess)
    return r.getFinalTransformation(), r.hasConverged(), r.nr_iterations, r.getFitnessScore(2.5)


def same(a, b):
    return np.array_equal(a[0], b[0]) and a[1:3] == b[1:3] and np.float64(a[3]).tobytes() == np.float64(b[3]).tobytes()


def fresh(method, k, tgt, src, guess):
    r = handle(method, k)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    out = aligned(r, guess), r.getCovariances(0, src.shape[0]), r.getCovariances(1, tgt.shape[0])
    r.close()
    return out


@pytest.mark.parametrize("k", [7, 49])
@pytest.mark.parametrize("method", ["GICP", "B200_VGICP_CUDA", "FAST_VGICP"])
def test_every_path_equals_a_fresh_single_handle(method, k):
    c = scenes(method, (16384, 12000, 9000, 5000), seed=60)
    eye = np.eye(4, dtype=np.float32)
    # the prefetched source (its covariances run on the second stream) and then promotion of that source to the target
    a = handle(method, k)
    a.setInputTarget(c[0])
    a.prefetchSource(c[1])
    a.setInputSource(c[1])
    want, wsc, _ = fresh(method, k, c[0], c[1], eye)
    assert np.array_equal(a.getCovariances(0, c[1].shape[0]), wsc, equal_nan=True)
    assert same(aligned(a, eye), want)
    a.promoteSourceToTarget()
    a.setInputSource(c[2])
    want, _, wtc = fresh(method, k, c[1], c[2], eye)
    assert np.array_equal(a.getCovariances(1, c[1].shape[0]), wtc, equal_nan=True)
    assert same(aligned(a, eye), want)
    a.close()
    # a batch of clouds of four sizes: k != 20 builds each cloud's covariances on its own
    params = {"registration_method": method, "reg_correspondence_randomness": str(k)}
    if "VGICP" in method:
        params["reg_resolution"] = "1.0"
    b = pkg.RegistrationBatch(params=params)
    ids = [b.addCloud(x) for x in c]
    pairs = [(1, 0), (2, 0), (3, 1), (3, 2)]
    res = b.align([(ids[s], ids[t], eye) for s, t in pairs], True, 2.5)
    b.close()
    for (s, t), x in zip(pairs, res):
        want = fresh(method, k, c[t], c[s], eye)[0]
        assert same((x["T"], x["converged"], x["iterations"], x["fitness"]), want), (s, t)


@pytest.mark.parametrize("k", [7, 49])
@pytest.mark.parametrize("method", ["GICP", "B200_VGICP_CUDA", "FAST_VGICP"])
def test_align_matches_the_reference(refs, method, k):
    if method == "GICP":
        tgt = gr.scene(16384, seed=3)
        src = gr.transform(gr.scene(16384, seed=4), np.linalg.inv(gr.pose((0.4, -0.3, 0.05), (0.01, 0.0, 0.06))))
    else:
        tgt = vr.room(12000, seed=3)
        src = vr.moved(vr.room(9000, seed=4), vr.rigid(0.03, [0.25, -0.1, 0.03]))
    r = handle(method, k)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    scov, tcov = r.getCovariances(0, src.shape[0]), r.getCovariances(1, tgt.shape[0])
    guess = np.eye(4, dtype=np.float32)
    r.align(guess)
    T, conv, it = r.getFinalTransformation(), r.hasConverged(), r.nr_iterations
    if method == "GICP":
        assert np.max(np.abs(scov - refs[method].covariances(src, k))) <= 1e-8
        w = refs[method].align(src, tgt, guess, scov=scov, tcov=tcov, k=k)
        assert np.max(np.abs(tcov - refs[method].covariances(tgt, k))) <= 1e-8
        assert (conv, it) == (w["converged"], w["iterations"])
        gr.end_point_is_as_good(T, w["T"])
    else:
        if method == "FAST_VGICP":
            assert np.max(np.abs(scov - vr.covariances(src, k))) <= 1e-8
            m = refs[method].map(tgt, 1.0, tcov)
        else:
            assert np.array_equal(scov, refs[method].covariances(src, k))
            m = refs[method].map(tgt, 1.0, tcov, k)
        o = m.align(src, scov=scov)
        assert (conv, it) == (o["converged"], o["iterations"])
        assert np.max(np.abs(T.astype(np.float64) - o["T"])) <= 1e-6
    assert conv and it >= 1
    want = orc.fitness(tgt, src, T, 2.5)[0]
    assert abs(r.getFitnessScore(2.5) - want) <= 1e-12 * want
    r.close()
