"""GPU edge cases against the oracle: tiny clouds (fewer points than k), duplicated points (exact ties), packed 16-byte
records, non-finite points, far-apart clouds (no correspondence inside max_correspondence_distance), big k."""
import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg
from common import rot_err, trans_err, perturb, relrel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def reg():
    r = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    yield r
    r.close()


def test_fewer_points_than_k(reg, oracle):
    rng = np.random.default_rng(0)
    tgt = np.c_[rng.uniform(-1, 1, (7, 3)), np.ones(7)].astype(np.float32)
    src = np.c_[rng.uniform(-1, 1, (5, 3)), np.ones(5)].astype(np.float32)
    reg.setInputTarget(tgt)
    reg.setInputSource(src)
    for which, cloud in ((0, src), (1, tgt)):
        got = reg.getCovariances(which, cloud.shape[0])
        want = oracle.gicp_covariances(cloud, 20)  # the oracle uses the min(k, n) neighbours it finds
        assert np.max(np.abs(got - want)) < 1e-8
    idx, d2 = reg.nearestKSearch(src)
    oi, od = oracle.knn(tgt, src, 1)
    assert np.array_equal(idx, oi[:, 0]) and np.array_equal(d2, od[:, 0])


def test_duplicate_points_and_ties(reg, oracle, synth):
    base = synth.scan("vlp16_16k", frame=0, stride=8)[::16].copy()
    tgt = np.concatenate([base, base, base[::2]])          # every point 2-3 times: exact ties everywhere
    src = base[::3].copy()                                 # queries coincide with target points: d2 == 0 ties
    reg.setInputTarget(tgt)
    idx, d2 = reg.nearestKSearch(src)
    oi, od = oracle.knn(tgt, src, 1)
    assert np.array_equal(idx, oi[:, 0]) and np.array_equal(d2, od[:, 0]) and np.all(d2 == 0)
    assert np.all(idx < base.shape[0])                     # lowest index among the duplicates
    reg.setInputSource(src)
    H, b, e = reg.gicpLinearizeAt(np.eye(4))
    sc, tc = oracle.gicp_covariances(src, 20), oracle.gicp_covariances(tgt, 20)
    o = oracle.gicp_linearize(src, sc, tgt, tc, np.eye(4), 2.5)
    assert np.array_equal(reg.getCorrespondences(src.shape[0]), o["corr"])


def test_packed_float4_records_equal_pointxyzi_records(synth):
    c8 = synth.scan("vlp16_16k", frame=2, stride=8)
    t8 = synth.scan("vlp16_16k", frame=3, stride=8)
    c4, t4 = np.ascontiguousarray(c8[:, :4]), np.ascontiguousarray(t8[:, :4])
    out = []
    for s, t in ((c8, t8), (c4, t4)):
        r = pkg.select_registration_method({"registration_method": "FAST_GICP"})
        r.setInputTarget(t)
        r.setInputSource(s)
        r.align(np.eye(4, dtype=np.float32))
        out.append((r.getFinalTransformation(), r.nr_iterations, r.getFitnessScore()))
        r.close()
    assert np.array_equal(out[0][0], out[1][0]) and out[0][1:] == out[1][1:]


def test_non_finite_points_are_ignored(reg, oracle, synth):
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)[::4].copy()
    src = synth.scan("vlp16_16k", frame=1, stride=8)[::4].copy()
    tgt_bad = tgt.copy()
    tgt_bad[5, 0] = np.nan
    tgt_bad[77, 2] = np.inf
    keep = np.ones(len(tgt), bool)
    keep[[5, 77]] = False
    reg.setInputTarget(tgt_bad)
    idx, d2 = reg.nearestKSearch(src)
    oi, od = oracle.knn(tgt[keep], src, 1)
    remap = np.nonzero(keep)[0]
    assert np.array_equal(idx, remap[oi[:, 0]]) and np.array_equal(d2, od[:, 0])


def test_no_correspondence_within_range(reg, synth, oracle):
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)
    src = tgt.copy()
    src[:, 0] += 500.0  # far outside max_correspondence_distance
    reg.setInputTarget(tgt)
    reg.setInputSource(src)
    reg.align(np.eye(4, dtype=np.float32))
    assert np.all(reg.getCorrespondences(src.shape[0]) == -1)
    T = reg.getFinalTransformation()
    o = oracle.gicp_align(src, tgt, np.eye(4, dtype=np.float32))
    # singular normal equations: both stop as "lm not converged" with the guess as pose (documented choice, oracle/gicp.cpp)
    assert not reg.hasConverged() and not o["converged"] and o["lm_failed"]
    assert np.array_equal(T, o["T"]) and np.array_equal(T, np.eye(4, dtype=np.float32))


def test_large_k(oracle, synth):
    cloud = synth.scan("vlp16_16k", frame=0, stride=8)[::8].copy()
    r = pkg.select_registration_method({"registration_method": "FAST_GICP", "reg_correspondence_randomness": 40})
    r.setInputTarget(cloud)
    got = r.getCovariances(1, cloud.shape[0])
    want = oracle.gicp_covariances(cloud, 40)
    assert np.max(np.abs(got - want)) < 1e-8
    r.close()


def test_full_size_properties(synth):
    """BASELINE size (65 536 pts): size-independent properties — identity on identical clouds, A->B then B->A ~ inverse,
    permutation invariance of the integer outputs"""
    a = synth.scan("vlp16", frame=0, stride=8)
    b = synth.scan("vlp16", frame=1, stride=8)
    r = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    r.setInputTarget(a)
    r.setInputSource(a)
    r.align(np.eye(4, dtype=np.float32))
    assert r.hasConverged() and trans_err(r.getFinalTransformation(), np.eye(4)) < 1e-5
    corr = r.getCorrespondences(a.shape[0])
    assert np.array_equal(corr, np.arange(a.shape[0]))      # every point matches itself
    r.setInputSource(b)
    r.align(np.eye(4, dtype=np.float32))
    Tab = r.getFinalTransformation().astype(np.float64)
    score_ab, used, inl = r.getFitnessScore(full=True)
    r.setInputTarget(b)
    r.setInputSource(a)
    r.align(np.eye(4, dtype=np.float32))
    Tba = r.getFinalTransformation().astype(np.float64)
    assert trans_err(Tab @ Tba, np.eye(4)) < 0.05 and rot_err(Tab @ Tba, np.eye(4)) < 5e-3
    # permuting the source permutes the correspondences and leaves counts / fitness unchanged
    perm = np.random.default_rng(1).permutation(b.shape[0])
    r.setInputTarget(a)
    r.setInputSource(b)
    H1, b1, e1 = r.gicpLinearizeAt(Tab)
    c1 = r.getCorrespondences(b.shape[0])
    r.setInputSource(b[perm].copy())
    H2, b2, e2 = r.gicpLinearizeAt(Tab)
    c2 = r.getCorrespondences(b.shape[0])
    assert np.array_equal(c1[perm], c2)
    assert relrel(H1, H2) < 1e-9 and abs(e1 - e2) <= 1e-9 * abs(e1)
    r.close()


@pytest.mark.parametrize("n", [1, 31, 1000, 16384, 16385, 40000, 65536, 100000, 131072])
def test_cluster_bvh_build_equals_toolkit_sort_build(synth, n):
    """bvh_build.cuh (the whole build as one kernel on a thread-block cluster, radix sort through distributed shared memory) must
    produce exactly the structure of the bounding-box / keys / cub::DeviceRadixSort / leaves chain it replaces: identical exact
    1-NN answers and bit-identical GICP covariances (which depend on the sorted order only through per-point k-NN sets) for every
    cluster size (1, 2, 4, 8 CTAs), with non-finite points and lattice ties in the cloud."""
    import subprocess, sys, os, json, tempfile
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = r'''
import sys, json, hashlib
import numpy as np
sys.path.insert(0, %r)
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import synth
n = %d
base = synth.scan("hdl32e", frame=3, stride=8)[:n].copy()
base[::97, :3] = np.round(base[::97, :3])          # lattice ties
if n > 10:
    base[5, 0] = np.nan; base[n // 2, 2] = np.inf   # dropped points
q = synth.scan("vlp16_16k", frame=4, stride=8)[:4096]
reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
reg.setInputTarget(base)
idx, d2 = reg.nearestKSearch(q)
cov = reg.getCovariances(1, n)
print(json.dumps({"idx": hashlib.sha1(idx.tobytes()).hexdigest(), "d2": hashlib.sha1(d2.tobytes()).hexdigest(),
                  "cov": hashlib.sha1(np.nan_to_num(cov, nan=-1.0).tobytes()).hexdigest()}))
reg.close()
''' % (root, n)
    outs = []
    for env_extra in ({}, {"B2R_CUB_SORT": "1"}):
        env = dict(os.environ)
        env.update(env_extra)
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        outs.append(json.loads(r.stdout.strip().splitlines()[-1]))
    assert outs[0] == outs[1]


def _gicp_degenerate_clouds():
    """exact degenerate neighbourhoods (coordinates on a 1/8 grid, exact in float32): name -> (cloud, kind, direction)"""
    g = np.arange(-3, 3, dtype=np.float64) / 8.0
    t = np.arange(30, dtype=np.float64) / 8.0 - 2.0
    u, v = [a.reshape(-1) for a in np.meshgrid(g, g, indexing="ij")]
    out = {
        "identical": (np.tile([[1.25, -0.5, 2.0]], (24, 1)), "point", None),
        "line_x": (np.c_[t, np.full(30, 0.5), np.full(30, -1.0)], "line", (1, 0, 0)),
        "line_y": (np.c_[np.full(30, 0.5), t, np.full(30, -1.0)], "line", (0, 1, 0)),
        "line_z": (np.c_[np.full(30, 0.5), np.full(30, -1.0), t], "line", (0, 0, 1)),
        "line_diag": (np.c_[t, t, t], "line", (1, 1, 1)),
        "plane_z": (np.c_[u, v, np.full(u.size, 0.75)], "plane", (0, 0, 1)),
        "plane_x": (np.c_[np.full(u.size, -0.25), u, v], "plane", (1, 0, 0)),
        "plane_diag": (np.c_[u, u - 0.5, v], "plane", (1, -1, 0)),  # x - y = 0.5
    }
    return {k: (np.c_[c, np.ones(c.shape[0])].astype(np.float32), kind, d) for k, (c, kind, d) in out.items()}


@pytest.mark.parametrize("case", list(_gicp_degenerate_clouds()))
def test_degenerate_neighbourhood_covariances(reg, oracle, case):
    """fast_gicp's PLANE regularisation on neighbourhoods whose covariance is degenerate.  A plane has a unique normal: engine ==
    oracle to 1e-8 == I - 0.999 n n^T of the plane's normal, eigenvalues (numpy eigh) {1e-3, 1, 1}.  A zero covariance (all k
    neighbours one point) has every direction as eigenvector: both follow JacobiSVD (U = I, smallest last) -> diag(1, 1, 1e-3).  A
    line leaves the normal free in the plane orthogonal to it: only the properties are pinned (symmetric, eigenvalues {1e-3, 1, 1},
    the 1e-3 direction orthogonal to the line)."""
    cloud, kind, d = _gicp_degenerate_clouds()[case]
    reg.setInputTarget(cloud)
    got = reg.getCovariances(1, cloud.shape[0])
    want = oracle.gicp_covariances(cloud, 20)
    for C in (got, want):
        assert np.max(np.abs(C - np.transpose(C, (0, 2, 1)))) < 1e-15
        w, V = np.linalg.eigh(C)
        assert np.max(np.abs(w - [1e-3, 1.0, 1.0])) < 1e-12
        if kind == "point":
            assert np.max(np.abs(C - np.diag([1.0, 1.0, 1e-3]))) < 1e-12
        elif kind == "line":
            dn = np.asarray(d, np.float64) / np.linalg.norm(d)
            assert np.max(np.abs(V[:, :, 0] @ dn)) < 1e-9
        else:
            n = np.asarray(d, np.float64) / np.linalg.norm(d)
            assert np.max(np.abs(C - (np.eye(3) - 0.999 * np.outer(n, n)))) < 1e-8
    if kind != "line":
        assert np.max(np.abs(got - want)) < 1e-8
