"""The shared __host__ __device__ numerics on the device (tests/device_numerics_harness.cu, device build with the library's
NVCC_FLAGS) against their host build (-ffp-contract=off), which the CPU suite holds bit for bit to the references:

  class A  the functions of the bit-exact contracts (correctly rounded float32 / float64 steps, Jacobi / SVD / Umeyama, PCL's
           eigen33, mt19937 and the RANSAC draw, the NDT voxel Gaussian, the VGICP-CUDA covariance): every output bit equal (NaN
           payload and sign aside) on >= 1e6 random and structured inputs each.
  libm     (float)exp/cos/sin((double)x) as the contracts write them: the device's CUDA libm against the host's glibc, exhaustively
           over every float32 input of the ranges the engine evaluates; the engine's shared atan2_rn on 1e9 random pairs and on every
           pair pcl_eigen33 meets on the floor tests' scans.
  class B  the plain-operator helpers the device may contract: the device build meets the same error bounds as the host build.
  LM       the LM state machine (lm_advance) replayed on the device over recorded rounds: every decision equal, lambda / nu / x0
           within 1e-12 relative of the host build."""
import os
import time

import numpy as np
import pytest

import device_numerics_build as dnb
from test_device_numerics import check_class_b, lm_cases, CLASS_B

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(tmp_path_factory):
    return dnb.Harness(dnb.build_device(tmp_path_factory.mktemp("dn_dev")))


@pytest.fixture(scope="module")
def host(oracle, tmp_path_factory):
    return dnb.Harness(dnb.build_host(tmp_path_factory.mktemp("dn_host")))


@pytest.mark.parametrize("fn", sorted(dnb.CLASS_A), ids=lambda f: dnb.CLASS_A[f])
def test_class_a_device_equals_host_bitwise(dev, host, fn):
    assert dev.lib.dn_is_device() == 1 and host.lib.dn_is_device() == 0
    rng = np.random.default_rng(1000 + fn)
    rec = dnb.class_a_inputs(fn, rng, 1_000_000)
    d, h = dev.run(fn, rec), host.run(fn, rec)
    if fn in (9, 10, 11, 12, 16):  # float64 records
        ok = dnb.same_bits64(d, h)
    else:
        ok = dnb.same_bits(d, h, fn)
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, (f"{dnb.CLASS_A[fn]}: {bad.size} of {len(rec)} records differ; first input {rec[bad[0]].tolist()}\n"
                           f"device {d[bad[0]].tolist()}\nhost   {h[bad[0]].tolist()}")


# exp: every float32 x <= 0 (-0 and every negative finite; +0 is exp(0) = 1 on both); cos / sin: every |t| <= 1.1 (both signs), each
# against glibc; atan2: atan2_rn (the engine's own, csrc/atan2_rn.cuh) on 1e9 random pairs a >= 0, b of either sign, magnitudes
# 2^-64 .. 2^64, against its host build.  CUDA's own atan2 differs from glibc's on 2 of these pairs, which is why the engine has atan2_rn.
SWEEPS = [("exp", 60, 0x80000000, 0x7F800000), ("cos", 61, 0, 2 * 0x3F8CCCCE), ("sin", 62, 0, 2 * 0x3F8CCCCE),
          ("atan2", 63, 20261018, 1_000_000_000)]


@pytest.mark.parametrize("name,fn,first,count", SWEEPS, ids=[s[0] for s in SWEEPS])
def test_transcendentals_device_equal_host(dev, name, fn, first, count):
    t = time.time()
    n, bad = dev.libm_sweep(fn, first, count)
    print(f"{name}: {count} inputs, {n} mismatches, {time.time() - t:.1f} s on {os.cpu_count()} cores")
    assert n == 0, f"(float){name}((double)x) differs between device and host on {n} inputs, e.g. (x, y, device, host) = {bad.tolist()}"


def test_floor_scan_eigen33_device_equals_host(dev, host, synth):
    """every (sqrt(-q), half_b) pair pcl_eigen33 meets in the normal filter on the floor tests' scans, and the eigen33 of each of
    those neighbourhoods: device == host bit for bit (and how many of the pairs CUDA's or glibc's own atan2 would round differently
    from atan2_rn, for the record)"""
    C = dnb.floor_scan_covariances(host, synth)
    ab, quad, _, _ = dnb.compute_roots_args(C)
    pairs = np.ascontiguousarray(ab[~quad])
    assert len(C) > 20_000 and len(pairs) > 10_000
    d, h = dev.run(63, pairs.view(np.uint32)), host.run(63, pairs.view(np.uint32))
    assert dnb.same_bits(d, h).all()
    glibc = np.arctan2(pairs[:, 0].astype(np.float64), pairs[:, 1].astype(np.float64)).astype(np.float32)
    print(f"floor scans: {len(C)} neighbourhoods, {len(pairs)} atan2 pairs, {int((glibc != h.view(np.float32)[:, 0]).sum())} where "
          "glibc's float32 atan2 differs from atan2_rn")
    rec = np.ascontiguousarray(C).view(np.uint32)
    assert dnb.same_bits(dev.run(19, rec), host.run(19, rec)).all()


@pytest.mark.parametrize("fn", sorted(CLASS_B), ids=lambda f: CLASS_B[f])
def test_class_b_device_within_bounds(dev, host, fn):
    check_class_b(dev, fn, host=host)


@pytest.mark.parametrize("case", lm_cases())
def test_lm_replay_device_decides_as_host(dev, host, synth, case):
    from test_device_numerics import lm_rounds
    R, x0, cfg = lm_rounds(host, synth, case)
    d = dev.lm_replay(R, x0, *cfg)
    h = host.lm_replay(R, x0, *cfg)
    # modes, li, it, delta_conv, converged, lm_failed, cur (= accept history), wc: identical round by round
    np.testing.assert_array_equal(d[:, :8], h[:, :8])
    # lambda and nu to 1e-12 relative; x0 to 1e-12 relative to the pose's largest entry (its near-zero rotation entries differ in
    # the last bits of the contracted products, ~1e-19 absolute)
    np.testing.assert_allclose(d[:, 8:10], h[:, 8:10], rtol=1e-12, atol=0)
    scale = np.abs(h[:, 10:]).max(1, keepdims=True)
    assert (np.abs(d[:, 10:] - h[:, 10:]) <= 1e-12 * scale).all(), float((np.abs(d[:, 10:] - h[:, 10:]) / scale).max())
