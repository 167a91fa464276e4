"""GPU: covariances of exactly axis-aligned neighbourhoods, where the eigenvalues tie and the PLANE normal is the column upstream's
JacobiSVD leaves last (e_z for lines along x and y, e_x for lines along z; tests/test_diagonal_normals.py states the rule).  The clouds
are separated segments on a 0.25 grid at power-of-two offsets (common.axis_lines), so FastGICP's demeaned moments and PCL's float32
raw moments are both exactly diagonal.  FAST_GICP and FAST_VGICP are compared with the oracle within 1e-8, GICP with the pcl GICP
reference within 1e-8, B200_VGICP_CUDA (whose float32 Jacobi picks its own column: ENGINE) with its reference bit for bit; then one
align per method on a scene that mixes such lines with a room, against the method's reference."""
import numpy as np
import pytest

import gicp_pcl_ref as gr
import hdl_graph_slam_b200 as pkg
import vgicp_cuda_ref as vc
import vgicp_ref as vr
from common import axis_lines, rot_err, trans_err
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

METHODS = ["FAST_GICP", "FAST_VGICP", "GICP", "B200_VGICP_CUDA"]


@pytest.fixture(scope="module")
def refs(tmp_path_factory):
    return dict(GICP=gr.Reference(tmp_path_factory.mktemp("gicp_pcl_ref")), FAST_VGICP=vr.Reference(tmp_path_factory.mktemp("vgicp_ref")),
                B200_VGICP_CUDA=vc.Reference(tmp_path_factory.mktemp("vgicp_cuda_ref")))


def handle(method, k=20):
    p = {"registration_method": method, "reg_correspondence_randomness": str(k)}
    if "VGICP" in method:
        p["reg_resolution"] = "1.0"
    return pkg.select_registration_method(p)


def plane(axis):
    n = np.eye(3)[axis]
    return np.eye(3) - (1.0 - 1e-3) * np.outer(n, n)


def line_axis(pts):
    """per point, the axis of its segment (segments are > 50 m apart and at least 24 points long)"""
    from scipy.spatial import cKDTree
    _, idx = cKDTree(pts[:, :3]).query(pts[:, :3], k=2)
    d = np.abs(pts[idx[:, 1], :3] - pts[:, :3])
    assert (np.count_nonzero(d, axis=1) == 1).all()
    return np.argmax(d, axis=1)


@pytest.mark.parametrize("k", [2, 3, 20])
@pytest.mark.parametrize("method", METHODS)
def test_axis_line_covariances(refs, method, k):
    pts = axis_lines(n_per_axis=40, seed=k)
    r = handle(method, k)
    r.setInputSource(pts)
    got = r.getCovariances(0, pts.shape[0])
    r.close()
    if method == "B200_VGICP_CUDA":
        assert np.array_equal(got, refs[method].covariances(pts, k))
        return
    want = refs["GICP"].covariances(pts, k) if method == "GICP" else orc.gicp_covariances(pts, k)
    assert np.max(np.abs(got - want)) <= 1e-8
    # and both are the JacobiSVD normal of each line: e_z along x and y, e_x along z
    along = line_axis(pts)
    rule = np.stack([plane(2 if a < 2 else 0) for a in along])
    assert np.max(np.abs(got - rule)) <= 1e-12 and np.max(np.abs(want - rule)) <= 1e-12


def mixed_scene():
    """axis lines plus a room 32 m below them; the source is the same scene seen from an exact dyadic translation (lines stay
    axis-aligned) with a second room sample"""
    lines = axis_lines(n_per_axis=40, seed=7)
    room_t = vr.room(12000, seed=70)
    room_s = vr.room(12000, seed=71)
    down = np.array([0.0, 0.0, -32.0, 0.0], np.float32)
    tgt = np.concatenate([lines, room_t + down])
    src = np.concatenate([lines, room_s + down])
    src[:, :3] -= np.array([0.25, -0.125, 0.0625], np.float32)
    return tgt, src


@pytest.mark.parametrize("method", METHODS)
def test_align_on_a_scene_with_axis_lines(refs, method):
    tgt, src = mixed_scene()
    r = handle(method)
    r.setInputTarget(tgt)
    r.setInputSource(src)
    scov, tcov = r.getCovariances(0, src.shape[0]), r.getCovariances(1, tgt.shape[0])
    guess = np.eye(4, dtype=np.float32)
    r.align(guess)
    T, conv, it = r.getFinalTransformation(), r.hasConverged(), r.nr_iterations
    if method == "FAST_GICP":  # the oracle builds its own covariances
        o = orc.gicp_align(src, tgt, guess)
        assert (conv, it) == (o["converged"], o["iterations"])
        assert trans_err(T, o["T"]) < 1e-6 and rot_err(T, o["T"]) < 1e-6
        assert np.array_equal(r.getCorrespondences(src.shape[0]), o["corr"])
    elif method == "GICP":
        assert np.max(np.abs(scov - refs[method].covariances(src))) <= 1e-8 and np.max(np.abs(tcov - refs[method].covariances(tgt))) <= 1e-8
        w = refs[method].align(src, tgt, guess, scov=scov, tcov=tcov)
        assert (conv, it) == (w["converged"], w["iterations"])
        gr.end_point_is_as_good(T, w["T"])
    else:
        if method == "FAST_VGICP":
            assert np.max(np.abs(scov - vr.covariances(src))) <= 1e-8 and np.max(np.abs(tcov - vr.covariances(tgt))) <= 1e-8
        else:
            assert np.array_equal(scov, refs[method].covariances(src)) and np.array_equal(tcov, refs[method].covariances(tgt))
        o = refs[method].map(tgt, 1.0, tcov).align(src, scov=scov)
        assert (conv, it) == (o["converged"], o["iterations"])
        assert np.max(np.abs(T.astype(np.float64) - o["T"])) <= 1e-6
    assert conv and np.max(np.abs(T[:3, 3] - [0.25, -0.125, 0.0625])) < 0.05
    want = orc.fitness(tgt, src, T, 2.5)[0]
    assert abs(r.getFitnessScore(2.5) - want) <= 1e-12 * want
    r.close()
