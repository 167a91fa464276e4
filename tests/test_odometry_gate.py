"""CPU-only: the odometry driver's gate (csrc/odometry_gate.cuh: the pose products, Eigen's matrix -> quaternion w, "reject this frame"
apps/scan_matching_odometry_nodelet.cpp:214-233 and "switch keyframe" :241-252), compiled by the host compiler alone
(tests/odo_gate_harness.cpp) and compared with the numpy float32 restatement of the reference's lines in tests/odometry_ref.py:
all four branches of the quaternion conversion, thresholds placed exactly on the compared quantities, the reported pose bit for
bit, and a seeded sweep of pose pairs for decision equality."""
import os
import subprocess
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import odometry_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
INF = float("inf")
P0 = dict(keyframe_delta_trans=INF, keyframe_delta_angle=INF, keyframe_delta_time=INF, transform_thresholding=1, max_acceptable_trans=INF,
          max_acceptable_angle=INF)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("odo_gate")
    exe = str(d / "odo_gate_harness")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++17", "-O2", "-Wall", "-ffp-contract=off", "-o", exe,
                           os.path.join(ROOT, "tests", "odo_gate_harness.cpp")])

    def run(cases):
        """cases: list of dict(kp, pt, tr, converged, stamp, kstamp, **params) -> list of result dicts"""
        rec = np.zeros((len(cases), 57))
        for i, c in enumerate(cases):
            p = dict(P0, **c.get("p", {}))
            rec[i, 0:16] = np.asarray(c.get("kp", np.eye(4)), f32).reshape(-1)
            rec[i, 16:32] = np.asarray(c.get("pt", np.eye(4)), f32).reshape(-1)
            rec[i, 32:48] = np.asarray(c["tr"], f32).reshape(-1)
            rec[i, 48:51] = [float(c.get("converged", True)), c.get("stamp", 0.0), c.get("kstamp", 0.0)]
            rec[i, 51:57] = [p["keyframe_delta_trans"], p["keyframe_delta_angle"], p["keyframe_delta_time"], float(p["transform_thresholding"]),
                             p["max_acceptable_trans"], p["max_acceptable_angle"]]
        fin, fout = str(d / "in.f64"), str(d / "out.f64")
        rec.tofile(fin)
        subprocess.check_call([exe, fin, fout])
        out = np.fromfile(fout).reshape(len(cases), 57)
        return [dict(decision=int(o[0]), odom=o[1:17].astype(f32).reshape(4, 4), dx=o[17], da=o[18], delta_trans=o[19], delta_angle=o[20],
                     w_delta=f32(o[21]), w_trans=f32(o[22]), too_large=bool(o[23]), wants_keyframe=bool(o[24]),
                     inv=o[25:41].astype(f32).reshape(4, 4), delta=o[41:57].astype(f32).reshape(4, 4)) for o in out]
    return run


def pose(R, t=(0, 0, 0)):
    T = np.eye(4, dtype=f32)
    T[:3, :3] = np.asarray(R, np.float64).astype(f32)
    T[:3, 3] = t
    return T


def bits(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


def same_bits(a, b):
    return np.array_equal(bits(a), bits(b))


def ulp32(x):
    return float(np.spacing(f32(abs(x))))


SKEW = np.array([1.0, 2.0, 3.0]) / np.sqrt(14.0)
AXES = {"x": np.array([1.0, 0, 0]), "y": np.array([0, 1.0, 0]), "z": np.array([0, 0, 1.0]), "skew": SKEW, "xy": np.array([1.0, 1.0, 0]) / np.sqrt(2.0),
        "-z": np.array([0, 0, -1.0])}


def rotation_cases():
    out = []
    for name, ax in AXES.items():
        for deg in (0.0, 1e-3, 5.0, 60.0, 119.0, 120.0, 121.0, 150.0, 179.0, 179.99, 180.0):
            out.append((f"{name}{deg}", pose(Rotation.from_rotvec(ax * np.deg2rad(deg)).as_matrix(), (0.3, -0.2, 0.1))))
    rng = np.random.default_rng(7)
    for k in range(40):  # slightly non-orthonormal float32 rotations, as an align returns them, at every angle
        R = Rotation.from_rotvec(rng.normal(size=3) / 1.2 * rng.uniform(0, np.pi)).as_matrix() + rng.normal(size=(3, 3)) * 1e-6
        out.append((f"noisy{k}", pose(R, rng.normal(size=3))))
    # half-turn about (1,1,0)/sqrt 2 with m00 == m11 exactly and an asymmetric disturbance: '>' keeps i = 0 on the tie, and the
    # two candidates for w differ
    T = pose([[0, 1, 5e-4], [1, 0, -1e-3], [-2e-4, 1e-3, -1]])
    out.append(("tie01", T))
    T = pose([[-1, 1e-3, 5e-4], [-1e-3, 0.25, 1], [2e-4, 1, 0.25]])  # m11 == m22 > m00: i = 1 on the tie
    out.append(("tie12", T))
    # a trace a few ulps above 3 (float32 rounding of a near-identity rotation): w one ulp above 1, acos -> NaN, every comparison false
    out.append(("w_above_1", pose(np.diag([f32(1) + 4 * np.spacing(f32(1))] * 3))))
    return out


def test_quaternion_w_takes_all_four_branches_and_matches_eigen(harness):
    cases = rotation_cases()
    res = harness([dict(tr=T) for _, T in cases])
    seen = set()
    for (name, T), r in zip(cases, res):
        seen.add(ref.quat_branch(T[:3, :3]))
        want = ref.quat_w(T)
        assert same_bits(r["w_trans"], want), (name, r["w_trans"], want)
        # prev_trans = I: the inverse is exactly I and delta == trans
        assert np.array_equal(r["delta"], T) and same_bits(r["w_delta"], want), name  # (up to the sign of a zero)
        if np.isfinite(ref.angle(T)):
            assert abs(r["delta_angle"] - float(ref.angle(T))) <= ulp32(r["delta_angle"]), name
            assert r["delta_angle"] == float(f32(r["delta_angle"])), name  # acosf widened, not a float64 acos
        else:
            assert np.isnan(r["delta_angle"]) and np.isnan(r["da"]), name
    assert seen == {"w", 0, 1, 2}
    by = dict(zip([n for n, _ in cases], res))
    # the branches the named cases are there for, and the values a wrong (j, k) order or a wrong diagonal pick would change
    for ax, br in (("x", 0), ("y", 1), ("z", 2)):
        for deg in (121.0, 150.0, 179.0):
            T = dict(cases)[f"{ax}{deg}"]
            assert ref.quat_branch(T[:3, :3]) == br
            assert abs(by[f"{ax}{deg}"]["delta_angle"] - np.deg2rad(deg) / 2) < 1e-5  # acos(w) is HALF the rotation angle
        assert ref.quat_branch(dict(cases)[f"{ax}119.0"][:3, :3]) == "w"
    # about -z the non-positive-trace branch returns a NEGATIVE w (the conversion does not normalise the sign): the angle compared
    # is pi - 75 degrees, above pi / 2, exactly as in the reference
    assert by["-z150.0"]["w_trans"] < 0 and abs(by["-z150.0"]["delta_angle"] - (np.pi - np.deg2rad(150.0) / 2)) < 1e-5
    assert abs(by["skew179.0"]["delta_angle"] - np.deg2rad(179.0) / 2) < 1e-5
    assert ref.quat_branch(dict(cases)["tie01"][:3, :3]) == 0 and ref.quat_branch(dict(cases)["tie12"][:3, :3]) == 1
    assert by["tie01"]["w_trans"] != 0 and by["tie12"]["w_trans"] != 0
    assert by["w_above_1"]["w_trans"] == f32(1) + np.spacing(f32(1))


def test_nan_angle_compares_false_everywhere(harness):
    T = dict(rotation_cases())["w_above_1"]
    tiny = dict(keyframe_delta_angle=0.0, max_acceptable_angle=0.0)
    r, = harness([dict(tr=T, p=tiny)])
    assert np.isnan(r["da"]) and np.isnan(r["delta_angle"])
    assert not r["too_large"] and not r["wants_keyframe"] and r["decision"] == ref.ACCEPTED
    assert ref.gate(dict(P0, **tiny), np.eye(4), np.eye(4), T, True, 0.0, 0.0)[0] == ref.ACCEPTED
    # the same thresholds do fire on an ordinary small rotation
    r, = harness([dict(tr=pose(Rotation.from_euler("z", 1.0, degrees=True).as_matrix()), p=tiny)])
    assert r["too_large"] and r["wants_keyframe"] and r["decision"] == ref.REJECTED


def test_norms_and_angles_have_the_reference_types(harness):
    """dx / delta_trans: float32 norms widened; da / delta_angle: acosf of the float32 w widened"""
    rng = np.random.default_rng(3)
    cases = []
    for _ in range(200):
        pt = pose(Rotation.from_rotvec(rng.normal(size=3) * 0.3).as_matrix(), rng.normal(size=3))
        tr = pose(Rotation.from_rotvec(rng.normal(size=3) * 0.3).as_matrix() + rng.normal(size=(3, 3)) * 1e-7, rng.normal(size=3) * 3)
        cases.append(dict(pt=pt, tr=tr))
    res = harness(cases)
    differs64 = 0
    for c, r in zip(cases, res):
        inv = ref.inverse_rigid(c["pt"])
        assert same_bits(r["inv"], inv)
        assert same_bits(r["delta"], ref.mul4(inv, c["tr"]))
        assert r["dx"] == float(ref.norm3(r["delta"])) and r["delta_trans"] == float(ref.norm3(c["tr"]))
        for key, m in (("da", r["delta"]), ("delta_angle", c["tr"])):
            assert r[key] == float(f32(r[key])) and abs(r[key] - float(ref.angle(m))) <= ulp32(r[key])
        t = c["tr"][:3, 3].astype(np.float64)
        differs64 += r["delta_trans"] != float(np.sqrt(t @ t))
        # the documented inverse is a good inverse: within a few float32 ulps of float64 linear algebra
        assert np.max(np.abs(r["inv"] - np.linalg.inv(c["pt"].astype(np.float64)))) < 1e-6
    assert differs64 > 100  # a float64 norm of the float32 entries is a different number most of the time


def test_thresholds_are_strict_on_the_exact_value(harness):
    rng = np.random.default_rng(11)
    cases, expect = [], []
    for _ in range(30):
        pt = pose(Rotation.from_rotvec(rng.normal(size=3) * 0.2).as_matrix(), rng.normal(size=3))
        tr = pose(Rotation.from_rotvec(rng.normal(size=3) * 0.4).as_matrix(), rng.normal(size=3))
        stamp, kstamp = 17.25 + rng.uniform(), 16.0 + rng.uniform()
        base, = harness([dict(pt=pt, tr=tr, stamp=stamp, kstamp=kstamp)])
        assert base["decision"] == ref.ACCEPTED and 0 < base["da"] < 1.6 and 0 < base["delta_angle"] < 1.6
        vals = dict(max_acceptable_trans=base["dx"], max_acceptable_angle=base["da"], keyframe_delta_trans=base["delta_trans"],
                    keyframe_delta_angle=base["delta_angle"], keyframe_delta_time=stamp - kstamp)
        for key, v in vals.items():
            fires = ref.REJECTED if key.startswith("max") else ref.KEYFRAME
            # on the value, one double below, one double above; and one FLOAT below / above (the compared quantity is a float32)
            for thr, want in ((v, ref.ACCEPTED), (np.nextafter(v, -INF), fires), (np.nextafter(v, INF), ref.ACCEPTED),
                              (float(np.nextafter(f32(v), f32(-INF))), fires), (float(np.nextafter(f32(v), f32(INF))), ref.ACCEPTED)):
                if key == "keyframe_delta_time" and thr != v and abs(thr - v) > 1e-12:
                    continue  # the time difference is a double: no float32 neighbours
                cases.append(dict(pt=pt, tr=tr, stamp=stamp, kstamp=kstamp, p={key: thr}))
                expect.append((key, thr, want))
    res = harness(cases)
    for c, r, (key, thr, want) in zip(cases, res, expect):
        assert r["decision"] == want, (key, thr)
        if key in ("max_acceptable_trans", "keyframe_delta_trans", "keyframe_delta_time"):  # norms and times equal the restatement bit for bit (the angles only to one float32 ulp)
            assert ref.gate(dict(P0, **c["p"]), np.eye(4), c["pt"], c["tr"], True, c["stamp"], c["kstamp"])[0] == want, (key, thr)
    # thresholding switched off: tiny limits reject nothing
    r, = harness([dict(tr=pose(np.eye(3), (5, 0, 0)), p=dict(transform_thresholding=0, max_acceptable_trans=1e-9, max_acceptable_angle=1e-9))])
    assert r["decision"] == ref.ACCEPTED and r["too_large"]


def test_reported_pose_is_bitwise_the_float32_product(harness):
    rng = np.random.default_rng(5)
    cases = []
    for k in range(300):
        kp = pose(Rotation.from_rotvec(rng.normal(size=3)).as_matrix() + rng.normal(size=(3, 3)) * 1e-6, rng.normal(size=3) * 50)
        pt = pose(Rotation.from_rotvec(rng.normal(size=3) * 0.2).as_matrix(), rng.normal(size=3))
        tr = pose(Rotation.from_rotvec(rng.normal(size=3) * 0.2).as_matrix(), rng.normal(size=3))
        p = [dict(), dict(max_acceptable_trans=0.0), dict(keyframe_delta_trans=0.0)][k % 3]
        cases.append(dict(kp=kp, pt=pt, tr=tr, converged=k % 5 != 0, p=p))
    res = harness(cases)
    decisions = set()
    fused_differs = 0
    for c, r in zip(cases, res):
        rejected = not c["converged"] or "max_acceptable_trans" in c["p"]
        want = ref.mul4(c["kp"], c["pt"] if rejected else c["tr"])  # :217 / :231 keyframe_pose * prev_trans, :221 keyframe_pose * trans
        assert r["decision"] == (ref.REJECTED if rejected else ref.KEYFRAME if "keyframe_delta_trans" in c["p"] else ref.ACCEPTED)
        assert same_bits(r["odom"], want)
        decisions.add(r["decision"])
        other = c["tr"] if rejected else c["pt"]
        assert not same_bits(r["odom"], ref.mul4(c["kp"], other))
        exact = (c["kp"].astype(np.float64) @ (c["pt"] if rejected else c["tr"]).astype(np.float64)).astype(f32)
        fused_differs += not same_bits(want, exact)
    assert decisions == {ref.REJECTED, ref.ACCEPTED, ref.KEYFRAME}
    assert fused_differs > 50  # the unfused left-to-right float32 sum is a different number from a wider or fused one often enough to see


def test_engine_host_code_is_compiled_without_contraction():
    """the products above are bit-exact only if the host compiler keeps a * b + c as two roundings: the engine's build passes the
    host compiler the same flag as the harness and the oracle"""
    from hdl_graph_slam_b200 import build
    assert "--compiler-options=-ffp-contract=off" in build.NVCC_FLAGS


def test_random_sweep_decisions_equal_the_restatement(harness):
    rng = np.random.default_rng(2024)
    n = 12000
    cases = []
    for k in range(n):
        scale = [0.02, 0.3, 1.5, 3.0][k % 4]
        pt = pose(Rotation.from_rotvec(rng.normal(size=3) * scale * 0.5).as_matrix(), rng.normal(size=3) * scale)
        tr = pose(Rotation.from_rotvec(rng.normal(size=3) * scale * 0.6).as_matrix() + rng.normal(size=(3, 3)) * 1e-7, rng.normal(size=3) * scale)
        kp = pose(Rotation.from_rotvec(rng.normal(size=3)).as_matrix(), rng.normal(size=3) * 20)
        p = dict(keyframe_delta_trans=rng.uniform(0.1, 3.0), keyframe_delta_angle=rng.uniform(0.05, 1.5), keyframe_delta_time=rng.uniform(0.1, 2.0),
                 transform_thresholding=int(rng.integers(0, 2)), max_acceptable_trans=rng.uniform(0.2, 4.0), max_acceptable_angle=rng.uniform(0.1, 1.5))
        cases.append(dict(kp=kp, pt=pt, tr=tr, converged=bool(rng.uniform() > 0.1), stamp=rng.uniform(0, 3), kstamp=rng.uniform(0, 1), p=p))
    res = harness(cases)
    PT, TR = np.stack([c["pt"] for c in cases]), np.stack([c["tr"] for c in cases])
    par = {k: np.array([c["p"][k] for c in cases]) for k in cases[0]["p"]}
    big, dx, da = ref.too_large(PT, TR, par["max_acceptable_trans"], par["max_acceptable_angle"])
    sw, dt, dang, _ = ref.wants_keyframe(TR, np.array([c["stamp"] for c in cases]), np.array([c["kstamp"] for c in cases]),
                                         par["keyframe_delta_trans"], par["keyframe_delta_angle"], par["keyframe_delta_time"])
    conv = np.array([c["converged"] for c in cases])
    want = np.where(~conv | (big & (par["transform_thresholding"] != 0)), ref.REJECTED, np.where(sw, ref.KEYFRAME, ref.ACCEPTED))
    got = np.array([r["decision"] for r in res])
    # an angle within one float32 ulp of its threshold may fall either way (acosf is not pinned to the last bit): none is that close here
    near = (np.abs(da - par["max_acceptable_angle"]) < 1e-6) | (np.abs(dang - par["keyframe_delta_angle"]) < 1e-6)
    assert near.sum() == 0
    assert np.array_equal(got, want)
    assert np.array_equal(np.array([r["dx"] for r in res]), dx) and np.array_equal(np.array([r["delta_trans"] for r in res]), dt)
    counts = np.bincount(got, minlength=3)
    assert counts.min() > 1000, counts
    # each criterion alone decides a fair share of the frames
    assert (big & conv & (par["transform_thresholding"] != 0)).sum() > 300 and (~big & sw).sum() > 300
