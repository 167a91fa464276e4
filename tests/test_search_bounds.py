"""CPU checks of the brute-force reference and the threshold probes that tests/test_search_bounds_gpu.py holds the engine to: the
numpy k-NN and covariances equal the oracle's, and the statistical-threshold probe rejects a summation order other than PCL's."""
import numpy as np
import pytest
from test_search_bounds_gpu import (bf_knn, bf_covariances, random_cloud, lattice_cloud, wide_range_cloud, sequential_stats,
                                    statistical_probes, threshold, placed_pair, cov_clouds, check_covariances)


@pytest.mark.parametrize("k", [1, 7, 20, 49, 64])
def test_brute_force_knn_equals_oracle(oracle, k):
    for c in (random_cloud(1), random_cloud(2, shift=True), lattice_cloud()):
        idx, d2 = bf_knn(c, c, k)
        oi, od = oracle.knn(c, c, k)
        assert np.array_equal(idx, oi) and np.array_equal(d2, od)
    tiny = random_cloud(3, n=5)[:5]
    tiny[2, 0] = np.nan  # a non-finite point is never a neighbour
    idx, d2 = bf_knn(tiny, tiny[[0, 1, 3]], k)
    oi, od = oracle.knn(tiny, tiny[[0, 1, 3]], k)
    assert np.array_equal(idx, oi) and np.array_equal(d2, od)


@pytest.mark.parametrize("k", [3, 20, 64])
def test_brute_force_covariances_equal_oracle(oracle, k):
    for c in (random_cloud(1), random_cloud(2, shift=True), lattice_cloud()):
        ref, unique = bf_covariances(c, k)
        want = oracle.gicp_covariances(c, k)
        assert unique.sum() > 0.5 * c.shape[0] or c.shape[0] < 1500
        assert np.max(np.abs(ref[unique] - want[unique])) < 1e-8


@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_covariance_check_pins_degenerate_neighbourhoods(oracle, k):
    """the GPU covariance check at small k, where most neighbourhoods are one point or a line: it accepts the oracle's covariances and
    rejects those built from a wrong neighbour (the (k+1)-th nearest in place of the second)"""
    for name, c in cov_clouds().items():
        order = bf_knn(c, c, 8)[0]
        assert check_covariances(oracle.gicp_covariances(c, k), c, k, oracle, name, order) == []
        if k > 1:
            wrong = order.copy()
            wrong[:, 1] = order[:, k]
            assert check_covariances(bf_covariances(c, k, wrong[:, :k])[0], c, k, oracle, name, order) != []


def test_placed_distances_are_exact():
    values = [6.25, float(np.nextafter(np.float32(6.25), np.float32(0))), float(np.float32(0.01)), float(np.float32(0.09)), 1e-6]
    src, tgt = placed_pair(values)  # asserts the brute-force squared distances equal the values
    assert src.shape[0] == len(values) and tgt.shape[0] == 25 * len(values)


def kernel_order_stats(dist, threads=1024, sums=False):
    """the order of k_sor_stats' parallel sums (before, its only order): thread t adds elements t, t + 1024, ... in turn; then an
    xor butterfly inside each warp and one over the 32 warp sums"""
    part = np.zeros(threads), np.zeros(threads)
    s, sq = part
    d = np.asarray(dist, np.float32)
    for i in range(0, len(d), threads):
        chunk = d[i:i + threads]
        s[:len(chunk)] += chunk.astype(np.float64)
        sq[:len(chunk)] += (chunk * chunk).astype(np.float64)

    def butterfly(v):
        lanes = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            v = v + v[..., lanes ^ o]
        return v[..., 0]

    s = butterfly(butterfly(s.reshape(32, 32)))
    sq = butterfly(butterfly(sq.reshape(32, 32)))
    n = len(d)
    return (s, sq) if sums else (s / n, (sq - s * s / n) / (n - 1))


def order_free(dist):
    """k_sor_stats' guard for its parallel sums: every term a multiple of 2^e, computed sum below 2^(e + 53), for the distances and
    their float32 squares"""
    d = np.asarray(dist, np.float32)
    d = d[~(d < 0)]
    ok = True
    for terms in (d, d * d):
        nz = terms[terms > 0]
        if nz.size == 0:
            continue
        e = int(np.min(np.maximum((nz.view(np.uint32) >> 23) & 0xff, 1).astype(np.int64))) - 150
        total = float(np.sum(terms.astype(np.float64)))
        ok &= (not np.isfinite(total)) or total < 2.0 ** (e + 53)
    return ok


def test_parallel_sums_are_taken_only_where_every_order_agrees(oracle, synth):
    """the guard admits scan-like clouds (where the strided sums then equal the sequential ones bit for bit) and refuses the
    wide-range cloud, so the GPU tests run both of k_sor_stats' paths"""
    from hdl_graph_slam_b200 import synth as s
    from test_search_bounds_gpu import filter_clouds, with_stride
    scans = [s.scan("vlp16_16k", frame=6, stride=8)[:3000], s.scan("kitti", frame=0, stride=8)[:40000]]
    scans += [with_stride(c, 8, np.random.default_rng(0)) for c in filter_clouds()[0].values()]
    for c in scans:
        for k in (1, 20, 63):
            dist = oracle.statistical_outlier(c, k, 1.0)[1]
            fin = np.isfinite(c[:, :3]).all(axis=1)
            assert order_free(dist[fin])
            seq = [0.0, 0.0]
            for d in dist[fin]:
                seq[0] += float(d)
                seq[1] += float(d * d)
            emu = kernel_order_stats(dist[fin], sums=True)
            assert np.array_equal(seq, emu, equal_nan=True)
    assert not order_free(oracle.statistical_outlier(wide_range_cloud(), 20, 1.0)[1])


def test_statistical_probe_rejects_the_strided_summation_order(oracle):
    """the GPU probe would pass for the wrong reason if it could not tell PCL's sequential sums from another order: on the same cloud,
    the strided / butterfly order decides at least one probe differently from the sequential sums, while the oracle agrees with them"""
    c = wide_range_cloud()
    _, dist = oracle.statistical_outlier(c, 20, 1.0)
    seq = sequential_stats(dist)
    emu = kernel_order_stats(dist)
    assert seq != emu
    probes = statistical_probes(dist, seq)
    assert len(probes) >= 3
    caught = 0
    for i, mul in probes:
        for m in (mul, float(np.nextafter(mul, -np.inf))):
            keep_seq = not (float(dist[i]) > threshold(*seq, m))
            keep_emu = not (float(dist[i]) > threshold(*emu, m))
            assert oracle.statistical_outlier(c, 20, m)[0][i] == keep_seq
            caught += keep_seq != keep_emu
    assert caught > 0
