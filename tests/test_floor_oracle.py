"""CPU: the floor-detection reference (tests/floor_ref.cpp) against an independent numpy / scipy restatement: the generator, the sample
stream, the clip masks, the normals, the RANSAC loop and known-plane recovery on synthetic scans."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from hdl_graph_slam_b200 import _capi
from floor_ref import Reference, LAUNCH, HYP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("floor_ref"))


def test_mt19937_known_answers(ref):
    # the standard's check: the 10000th output of a default-seeded (5489) mt19937
    assert ref.mt19937(5489, 10000)[-1] == 4123659995
    # numpy's legacy RandomState seeds MT19937 with the same init_genrand
    raw = np.random.RandomState(12345)._bit_generator.random_raw(2000).astype(np.uint32)
    assert np.array_equal(ref.mt19937(12345, 2000), raw)


def _stream(n, count, pts):
    """drawIndexSample / isSampleGood / computeModelCoefficients restated in numpy float32"""
    raw = np.random.RandomState(12345)._bit_generator.random_raw(count * 3 * 1000 + 10).astype(np.uint32)
    pos = 0
    sh = list(range(n))
    out = []
    for _ in range(count):
        found = None
        if n >= 3:
            for _check in range(1000):
                for i in range(3):
                    r = int(raw[pos]) >> 1
                    pos += 1
                    j = i + r % (n - i)
                    sh[i], sh[j] = sh[j], sh[i]
                p0, p1, p2 = (pts[sh[k], :3].astype(f32) for k in range(3))
                a, b = p1 - p0, p2 - p0
                with np.errstate(all="ignore"):
                    q = a / b
                if (q[0] != q[1]) or (q[2] != q[1]):
                    c = np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0], 0], f32)
                    z = (c[0] * c[0] + c[2] * c[2]) + (c[1] * c[1] + c[3] * c[3])
                    if z > 0:
                        c = c / np.sqrt(z)
                    dot = (c[0] * p0[0] + c[2] * p0[2]) + (c[1] * p0[1] + c[3] * f32(1))
                    c[3] = -dot
                    found = (tuple(sh[:3]), c)
                    break
        out.append(found)
        if found is None:
            break
    return out


def _scan(seed, n=400, plane=True):
    rng = np.random.default_rng(seed)
    pts = np.zeros((n, 8), f32)
    pts[:, 0] = rng.uniform(-10, 10, n)
    pts[:, 1] = rng.uniform(-10, 10, n)
    pts[:, 2] = (-1.8 + rng.normal(0, 0.02, n)) if plane else rng.uniform(-3, -1, n)
    pts[:, 3] = 1
    out = rng.random(n) < 0.3
    pts[out, 2] = rng.uniform(-3, -1, out.sum())
    return pts


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_sample_stream(ref, seed):
    pts = _scan(seed, 200)
    got = ref.hypotheses(pts, 50)
    want = _stream(200, 50, pts)
    for g, w in zip(got, want):
        assert g["ok"] == 1
        assert tuple(g["idx"]) == w[0]
        assert np.array_equal(g["c"].view(np.uint32), w[1].view(np.uint32))


def collinear(n=500):
    """points t (1, 2, 4) at dyadic t: every (p1 - p0) / (p2 - p0) has three equal components, so no sample is ever good.  (An
    axis-aligned line is no such cloud: its 0 / 0 components are NaN, which isSampleGood counts as good.)"""
    t = (-0.25 - np.arange(1, n + 1) * 2.0 ** -10).astype(f32)
    pts = np.zeros((n, 4), f32)
    pts[:, 0], pts[:, 1], pts[:, 2], pts[:, 3] = t, 2 * t, 4 * t, 1
    return pts


def test_no_sample_when_collinear_or_tiny(ref):
    line = collinear()
    assert ref.hypotheses(line, 2)["ok"][0] == 0
    assert ref.hypotheses(line[:2], 1)["ok"][0] == 0
    r = ref.detect(line, use_normal_filtering=0, floor_pts_thresh=100)
    assert r["n_filtered"] == 500 and r["reason"] == "NO_MODEL" and r["ransac_iterations"] == 0
    axis = line.copy()
    axis[:, 1] = axis[:, 0] = 0
    assert ref.hypotheses(axis, 1)["ok"][0] == 1


def test_clip_masks(ref):
    rng = np.random.default_rng(5)
    pts = np.zeros((2000, 4), f32)
    pts[:, :3] = rng.uniform(-4, 0, (2000, 3)).astype(f32)
    pts[:10, 2] = f32(-3.0)       # on the lower plane: kept (>=)
    pts[10:20, 2] = f32(-1.0)     # on the upper plane: >= -d_lo holds, so the negative clip drops it
    pts[20, 2] = np.nan
    pts[21, 0] = np.inf
    pts[22, 1] = -np.inf
    pts[23, 2] = np.inf
    pts[24, 2] = -np.inf
    r = ref.detect(pts, use_normal_filtering=0, floor_pts_thresh=10 ** 6)
    z = pts[:, 2]
    with np.errstate(invalid="ignore"):
        s = (f32(0) * pts[:, 0] + f32(0) * pts[:, 1]) + z
        want = (s >= f32(-3.0)) & ~(s >= f32(-1.0))
    assert np.array_equal(r["band_mask"], want)
    assert want[:10].all() and not want[10:25].any()
    assert r["reason"] == "TOO_FEW_FILTERED" and r["n_filtered"] == want.sum()


def test_eigen33_against_eigh(ref):
    rng = np.random.default_rng(7)
    worst = 0.0
    for _ in range(2000):
        P = rng.normal(size=(10, 3)) * rng.uniform(0.01, 3, 3)
        Cm = np.cov(P.T, bias=True).astype(f32)
        v = ref.eigen33(Cm)
        w, V = np.linalg.eigh(Cm.astype(np.float64))
        gap = (w[1] - w[0]) / max(w[2], 1e-12)
        if gap < 1e-3:
            continue
        worst = max(worst, 1 - abs(float(np.dot(v.astype(np.float64), V[:, 0]))))
    assert worst < 1e-3


def _normal_keep_numpy(band, thresh_deg):
    from scipy.spatial import cKDTree
    xyz = band[:, :3].astype(np.float64)
    k = min(10, len(xyz))
    _, idx = cKDTree(xyz).query(xyz, k=k)
    idx = np.asarray(idx).reshape(len(xyz), k)
    cos_t = math.cos(thresh_deg * math.pi / 180.0)
    zs, ok = np.empty(len(xyz)), np.empty(len(xyz), bool)
    for i in range(len(xyz)):
        P = xyz[idx[i]]
        w, V = np.linalg.eigh(np.cov(P.T, bias=True))
        zs[i] = abs(V[2, 0])
        # PCL forms cov = E[ab] - E[a]E[b] in float32: its noise is ~1e-6 of the raw second moments, so only neighbourhoods whose
        # two smallest eigenvalues are farther apart than that have a normal both computations must agree on
        ok[i] = w[1] - w[0] > 1e-5 * np.mean(np.sum(P * P, axis=1))
    return zs, cos_t, ok


def test_normal_filter_against_eigh(ref):
    """a 2-D dense patch of ground, a wall and a 30-degree ramp (a synthetic scan's neighbourhoods lie along its rings, where the
    float32 moments decide the normal)"""
    rng = np.random.default_rng(11)
    g = np.c_[rng.uniform(-5, 5, (3000, 2)), -1.8 + rng.normal(0, 0.003, 3000)]
    w = np.c_[np.full(1500, 4.0) + rng.normal(0, 0.003, 1500), rng.uniform(-5, 5, 1500), rng.uniform(-2.9, -1.1, 1500)]
    u = rng.uniform(0, 3, (1500, 2))
    ramp = np.c_[u[:, 0] - 6, u[:, 1], -2.9 + np.tan(np.radians(30)) * u[:, 0] * 0.5 + rng.normal(0, 0.003, 1500)]
    c = np.zeros((6000, 8), f32)
    c[:, :3] = np.r_[g, w, ramp]
    c[:, 3] = 1
    r = ref.detect(c, **LAUNCH["hdl"])
    band = c[r["band_mask"]]
    zs, cos_t, ok = _normal_keep_numpy(band, 20.0)
    away = ok & (np.abs(zs - cos_t) > 0.02)  # keep masks agree away from the threshold, on well-conditioned neighbourhoods
    assert away.mean() > 0.5
    assert np.array_equal(r["normal_keep"][away], (zs > cos_t)[away])


def _python_ransac(filt, hyps):
    xyz = filt[:, :3].astype(f32)
    n = len(xyz)
    it, best, k, best_h = 0, -(2 ** 31 - 1), 1.0, None
    logp, one = math.log(1 - 0.99), 1.0 / n
    for h in hyps:
        if not it < k:
            break
        if h is None:
            break
        c = h[1]
        d = (c[0] * xyz[:, 0] + c[2] * xyz[:, 2]) + (c[1] * xyz[:, 1] + c[3] * f32(1))
        cnt = int((np.abs(d).astype(np.float64) < 0.1).sum())
        if cnt > best:
            best, best_h = cnt, h
            p = 1.0 - math.pow(best * one, 3.0)
            p = min(1 - 2.220446049250313e-16, max(2.220446049250313e-16, p))
            k = logp / math.log(p)
        it += 1
        if it > 10000:
            break
    return it, best_h


@pytest.mark.parametrize("seed,plane", [(0, True), (1, True), (2, False)])
def test_ransac_loop_replayed_in_python(ref, seed, plane):
    pts = _scan(seed, 600, plane)
    r = ref.detect(pts, use_normal_filtering=0, floor_pts_thresh=0)
    filt = r["filtered"]
    it, best = _python_ransac(filt, _stream(len(filt), min(r["ransac_iterations"] + 1, 2000), filt))
    assert it == r["ransac_iterations"]
    assert best[0] == r["model_indices"]
    c = best[1]
    d = (c[0] * filt[:, 0] + c[2] * filt[:, 2]) + (c[1] * filt[:, 1] + c[3] * f32(1))
    assert np.array_equal(filt[np.abs(d).astype(np.float64) < 0.1], r["inliers"])


@pytest.mark.parametrize("sensor,frame", [("vlp16", 0), ("hdl32e", 2), ("kitti", 4)])
def test_known_plane_recovery(ref, synth, sensor, frame):
    """the synthetic ground is z = -1.8 in the sensor frame: the published plane is (0, 0, 1, 1.8) up to the noise"""
    c = synth.scan(sensor, frame=frame, stride=8)
    r = ref.detect(c, **LAUNCH["hdl"])
    assert r["detected"] and r["reason"] == "OK"
    assert r["coeffs"][2] > 0.999 and abs(r["coeffs"][3] - 1.8) < 0.05
    assert r["n_inliers"] > 0.8 * r["n_filtered"]


def test_tilted_sensor(ref, synth):
    """a sensor pitched by 10 deg, compensated by tilt_deg, still finds the ground; uncompensated, the band misses most of it"""
    c = synth.scan("vlp16", frame=1, stride=8, pitch=math.radians(10.0))
    r = ref.detect(c, **dict(LAUNCH["hdl"], tilt_deg=10.0))
    assert r["detected"]
    r0 = ref.detect(c, **dict(LAUNCH["hdl"], tilt_deg=-10.0))
    assert r0["n_filtered"] < r["n_filtered"]


def test_abi_struct_sizes(tmp_path):
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include "b200reg.h"\nint main(){printf("%zu %zu\\n", sizeof(b2r_floor_params), sizeof(b2r_floor_result));return 0;}\n')
    exe = tmp_path / "s"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(_capi.FloorParams), C.sizeof(_capi.FloorResult)] == [48, 72]
    assert HYP.itemsize == 32
