"""CPU-only: the PLANE normal of an exactly diagonal covariance (an axis-aligned line, or all neighbours one point), where the eigenvalues
tie and "the smallest eigenvector" is not unique.  Upstream's JacobiSVD does no rotation on a diagonal matrix and leaves last in U the
column its step-4 sort puts there (first maximum of the remaining |values| swapped in only when not in place, stop at a zero maximum).
The engine's closed form sym_min_eigvec3 (linalg.cuh compiled as host code by tests/diag_normal_harness.cu), the oracle's rule
(orc::diagonal_normal) and a numpy restatement (common.jacobisvd_diagonal_normal) must all return that column, the references'
covariances must be built on it, and every non-diagonal input must give the same bits as the solver before the rule."""
import os
import subprocess

import numpy as np
import pytest

import gicp_pcl_ref as gr
from common import axis_lines, jacobisvd_diagonal_normal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
EX, EY, EZ = np.eye(3)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("diag_normal") / "diag_normal_harness")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-w", "-Wno-deprecated-gpu-targets", "-ccbin", CXX, "-Xcompiler", "-ffp-contract=off",
                           "-o", exe, os.path.join(ROOT, "tests", "diag_normal_harness.cu")])
    return exe


def normals(harness, diagonals):
    """per diagonal: (engine, engine before the rule, oracle rule, oracle Jacobi alone), each a 3-vector"""
    text = "".join("%r %r %r\n" % tuple(float(x) for x in d) for d in diagonals)
    out = subprocess.run([harness, "table"], input=text, capture_output=True, text=True, check=True)
    rows = np.array([[float(x) for x in line.split()] for line in out.stdout.splitlines()])
    assert rows.shape == (len(diagonals), 12)
    return rows.reshape(-1, 4, 3)


def axis_of(v):
    """the axis a unit vector lies on, up to sign; None if it lies on none"""
    a = int(np.argmax(np.abs(v)))
    return a if abs(v[a]) == 1.0 and np.count_nonzero(v) == 1 else None


def test_axis_lines_table(harness):
    """one non-zero entry: the line along x and along y give e_z, the line along z gives e_x; the engine before this rule gave e_y for
    the z line, the oracle's ascending Jacobi alone gives e_y, e_x, e_x"""
    a = 0.3125
    got = normals(harness, [(a, 0, 0), (0, a, 0), (0, 0, a)])
    for (new, old, rule, jac), want, was, jacobi in zip(got, (2, 2, 0), (2, 2, 1), (1, 0, 0)):
        assert axis_of(new) == axis_of(rule) == want and np.array_equal(new, np.eye(3)[want])
        assert axis_of(old) == was and axis_of(jac) == jacobi


DIAGONALS = [
    # one non-zero entry on each axis, at several magnitudes
    (1.0, 0, 0), (0, 1.0, 0), (0, 0, 1.0), (1e-12, 0, 0), (0, 7e5, 0), (0, 0, 3e-7),
    # two equal non-zero entries larger than the third (zero or not), in every position
    (2.0, 2.0, 0), (2.0, 0, 2.0), (0, 2.0, 2.0), (2.0, 2.0, 0.5), (2.0, 0.5, 2.0), (0.5, 2.0, 2.0),
    # two equal non-zero entries smaller than the third
    (0.5, 0.5, 2.0), (0.5, 2.0, 0.5), (2.0, 0.5, 0.5),
    # all equal (a multiple of I) and the zero matrix
    (1.5, 1.5, 1.5), (1e-9, 1e-9, 1e-9), (0, 0, 0),
    # a tiny negative entry from cancellation: the sort compares |values|
    (0.25, -1e-17, 0), (-1e-17, 0.25, 0), (0, -1e-17, 0.25), (0, 0.25, -1e-17), (-1e-17, 0, 0), (0, 0, -1e-17), (-1e-17, -1e-17, 0.25),
    # three distinct values in every order (the normal is the unique smallest |value|)
    (1.0, 2.0, 3.0), (3.0, 2.0, 1.0), (2.0, 3.0, 1.0), (1.0, 3.0, 2.0),
]


def test_every_diagonal_pattern_follows_jacobisvd(harness):
    got = normals(harness, DIAGONALS)
    for d, (new, old, rule, jac) in zip(DIAGONALS, got):
        want = axis_of(jacobisvd_diagonal_normal(np.diag(d)))
        assert want is not None
        assert axis_of(new) == want and np.array_equal(new, np.eye(3)[want]), d
        assert axis_of(rule) == want, d


def test_jacobisvd_rule_restated():
    """the rule on hand-worked cases: the sort swaps on a STRICTLY larger first maximum and stops at a zero maximum"""
    n = lambda *d: jacobisvd_diagonal_normal(np.diag(d))  # noqa: E731
    assert np.array_equal(n(0, 0, 0), EZ) and np.array_equal(n(2, 2, 2), EZ)
    assert np.array_equal(n(5, 0, 0), EZ) and np.array_equal(n(0, 5, 0), EZ) and np.array_equal(n(0, 0, 5), EX)
    assert np.array_equal(n(1, 1, 4), EX)  # (4, 1, 1) after swapping columns 0 and 2: the old column 0 is last
    assert np.array_equal(n(4, 1, 1), EZ) and np.array_equal(n(1, 4, 1), EZ)
    assert np.array_equal(n(0.25, -1e-17, 0), EZ)  # |-1e-17| > 0: the y column is kept ahead of z
    assert jacobisvd_diagonal_normal(np.array([[1.0, 1e-300, 0], [1e-300, 1.0, 0], [0, 0, 1.0]])) is None


def test_non_diagonal_inputs_keep_their_bits(harness):
    """1e5 random rotated spectra, 3 in 5 with one or two off-diagonals exactly 0 (never all three): the solver returns bit for bit
    what it returned before the diagonal branch"""
    out = subprocess.run([harness, "random", "100000"], capture_output=True, text=True, check=True).stdout
    stats = dict(kv.split("=") for kv in out.split())
    assert int(stats["mismatch"]) == 0 and int(stats["with_zero_offdiagonal"]) > 50000


def plane(n):
    return np.eye(3) - (1.0 - 1e-3) * np.outer(n, n)


@pytest.mark.parametrize("k", [2, 3, 20])
def test_reference_covariances_on_axis_lines(oracle, tmp_path_factory, k):
    """the oracle's FastGICP covariances (demeaned moments) and the pcl GICP reference's (float32 raw moments, exact on these lines)
    are the PLANE matrices of the axis each point's line does NOT run along as JacobiSVD picks it: e_z for x and y lines, e_x for z"""
    pts = axis_lines(n_per_axis=12, seed=k)
    along = np.array([segment_axis(pts, i, k) for i in range(len(pts))])
    want = np.stack([plane(np.eye(3)[2 if a < 2 else 0]) for a in along])
    got = oracle.gicp_covariances(pts, k)
    assert np.max(np.abs(got - want)) <= 1e-15
    ref = gr.Reference(tmp_path_factory.mktemp("gicp_pcl_ref"))
    assert np.max(np.abs(ref.covariances(pts, k) - want)) <= 1e-15


def segment_axis(pts, i, k):
    """the axis of the segment point i lies on (its k nearest neighbours differ from it along that axis only)"""
    d = pts[:, :3] - pts[i, :3]
    near = np.argsort((d * d).sum(axis=1), kind="stable")[:max(k, 2)]
    spread = np.ptp(pts[near, :3], axis=0)
    assert np.count_nonzero(spread) == 1
    return int(np.flatnonzero(spread)[0])
