"""CPU-only: an INDEPENDENT second derivation of the two registration cost models, written straight from the published algorithms
with numpy float64 + scipy (cKDTree, expm, svd) — no code path shared with oracle/ or the engine — checked against the oracle.

The oracle (oracle/*.cpp) and the engine's host/device logic were written by the same hand from SURVEY.md Appendix A, so a wrong
recollection would pass every oracle-vs-engine test.  Here the same quantities are rebuilt a different way:
  * GICP (Segal et al. 2009 / fast_gicp): k-NN by scipy's cKDTree, covariance by np.cov, plane regularisation by np.linalg.svd,
    M_i = (C_B + R C_A R^T)^-1 by np.linalg.inv, H = sum J^T M J and b = sum J^T M e by einsum with J = d e / d(twist) obtained
    from the CLOSED FORM d(T p)/d(omega, v) = [-skew(T p) | I] (sign folded into e = mu_B - T mu_A), the LM step by
    np.linalg.solve and the pose update by scipy.linalg.expm of the 4x4 twist matrix (no hand-written se3_exp);
  * NDT (Magnusson 2009 / ndt_omp DIRECT7): voxel Gaussians by np.unique + np.cov, score as the plain sum of Gaussians over the
    centre cell and its 6 face neighbours, gradient by CENTRAL FINITE DIFFERENCES of that independent score.
What this cannot pin (no upstream sources in this image): implementation quirks such as tie-breaking and float32 rounding order;
those are covered by the bit-exact oracle-vs-engine tests."""
import numpy as np
import pytest
from scipy.spatial import cKDTree
from scipy.linalg import expm
from common import axis_lines, jacobisvd_diagonal_normal, perturb, relrel


def skew(v):
    z = np.zeros(len(v))
    return np.stack([np.stack([z, -v[:, 2], v[:, 1]], -1), np.stack([v[:, 2], z, -v[:, 0]], -1), np.stack([-v[:, 1], v[:, 0], z], -1)], -2)


def indep_covariances(pts, k=20):
    """fast_gicp calculate_covariances with PLANE regularisation, numpy/scipy only"""
    xyz = pts[:, :3].astype(np.float64)
    d, idx = cKDTree(xyz).query(xyz, k=k + 1)
    # points whose k-th and (k+1)-th neighbours are (nearly) equidistant have an ambiguous neighbour set: excluded from the comparison
    ambiguous = (d[:, k] - d[:, k - 1]) < 1e-6 * np.maximum(d[:, k], 1e-12)
    nb = xyz[idx[:, :k]]                                   # (n, k, 3)
    c = nb - nb.mean(axis=1, keepdims=True)
    cov = np.einsum("nki,nkj->nij", c, c) / k
    U, S, Vt = np.linalg.svd(cov)
    reg = np.einsum("nij,j,njk->nik", U, np.array([1.0, 1.0, 1e-3]), Vt)
    # an exactly diagonal covariance (an axis-aligned line) ties singular values, which LAPACK orders its own way: JacobiSVD's rule
    for i in np.flatnonzero((cov[:, 0, 1] == 0) & (cov[:, 0, 2] == 0) & (cov[:, 1, 2] == 0)):
        n = jacobisvd_diagonal_normal(cov[i])
        reg[i] = np.eye(3) - (1.0 - 1e-3) * np.outer(n, n)
    return reg, ambiguous


def indep_linearize(src, scov, tgt, tcov, T, max_dist):
    T = np.asarray(T, np.float64)
    Tf = T.astype(np.float32)
    q = (src[:, :3].astype(np.float32) @ Tf[:3, :3].T + Tf[:3, 3]).astype(np.float64)  # correspondences are searched with the float32 pose
    d, j = cKDTree(tgt[:, :3].astype(np.float64)).query(q, k=2)
    ambiguous = (d[:, 1] - d[:, 0]) < 1e-6 * np.maximum(d[:, 1], 1e-12)
    valid = d[:, 0] ** 2 < max_dist ** 2
    corr = np.where(valid, j[:, 0], -1)
    a = src[valid, :3].astype(np.float64)
    bpts = tgt[corr[valid], :3].astype(np.float64)
    R = T[:3, :3]
    ta = a @ R.T + T[:3, 3]
    e = bpts - ta
    M = np.linalg.inv(tcov[corr[valid]] + R @ scov[valid] @ R.T)
    # e(delta) = mu_B - exp(delta) T mu_A  =>  de/d(omega) = skew(T mu_A), de/dv = -I
    J = np.concatenate([skew(ta), -np.broadcast_to(np.eye(3), (len(ta), 3, 3))], axis=2)   # (n, 3, 6)
    H = np.einsum("nia,nij,njb->ab", J, M, J)
    b = np.einsum("nia,nij,nj->a", J, M, e)
    cost = np.einsum("ni,nij,nj->", e, M, e)
    return corr, ambiguous, H, b, cost


@pytest.fixture(scope="module")
def pair(synth):
    return synth.scan("vlp16_16k", frame=1, stride=8), synth.scan("vlp16_16k", frame=0, stride=8)


def test_gicp_covariances_independent(pair, oracle):
    src, _ = pair
    want, amb = indep_covariances(src, 20)
    got = oracle.gicp_covariances(src, 20)
    ok = ~amb
    assert ok.mean() > 0.99
    assert np.max(np.abs(got[ok] - want[ok])) < 1e-6  # the smallest singular vector of a near-isotropic patch is ill-conditioned: 1e-6, not 1e-9


def test_gicp_covariances_of_axis_lines_independent(oracle):
    """exactly diagonal covariances (common.axis_lines): the diagonal branch against the oracle, every point (the regularised matrix
    depends on the normal alone, so the tie-ambiguous neighbour sets do not matter here)"""
    p = axis_lines(n_per_axis=4, seed=2)
    want, _ = indep_covariances(p, 20)
    assert np.max(np.abs(oracle.gicp_covariances(p, 20) - want)) <= 1e-12


def test_gicp_linearize_and_one_lm_step_independent(pair, oracle):
    src, tgt = pair
    scov = oracle.gicp_covariances(src, 20)
    tcov = oracle.gicp_covariances(tgt, 20)
    for T0 in (np.eye(4), perturb(4, 0.3, 2.0)):
        T0 = np.asarray(T0, np.float32).astype(np.float64)
        corr, amb, H, b, cost = indep_linearize(src, scov, tgt, tcov, T0, 2.5)
        o = oracle.gicp_linearize(src, scov, tgt, tcov, T0, 2.5)
        differ = (corr != o["corr"]) & ~amb
        assert differ.sum() == 0, f"{differ.sum()} unambiguous correspondences differ"
        if (corr != o["corr"]).sum() == 0:  # no tie was resolved differently: the sums are over the same set
            assert relrel(H, o["H"]) < 1e-9 and relrel(b, o["b"]) < 1e-9 and abs(cost - o["err"]) <= 1e-9 * cost
        else:
            assert relrel(H, o["H"]) < 1e-4 and relrel(b, o["b"]) < 1e-4
        # one Levenberg-Marquardt step: lambda0 = 1e-9 max|diag H|, d = -(H + lambda I)^-1 b, x1 = expm(twist(d)) x0
        lam = 1e-9 * np.max(np.abs(np.diag(o["H"])))
        d = np.linalg.solve(o["H"] + lam * np.eye(6), -o["b"])
        tw = np.zeros((4, 4))
        tw[:3, :3] = skew(d[None, :3])[0]
        tw[:3, 3] = d[3:]
        x1 = expm(tw) @ T0
        r = oracle.gicp_align(src, tgt, T0.astype(np.float32), max_iterations=1, src_cov=scov, tgt_cov=tcov)
        assert r["iterations"] == 1
        assert np.max(np.abs(r["T64"] - x1)) < 1e-9, "se3_exp / step direction differs from expm of the twist"
        # and the accepted step lowers the cost evaluated independently at the new pose (rho > 0)
        _, _, _, _, cost1 = indep_linearize(src, scov, tgt, tcov, x1, 2.5)
        assert cost1 < cost


def euler_xyz(p):
    cx, sx, cy, sy, cz, sz = np.cos(p[3]), np.sin(p[3]), np.cos(p[4]), np.sin(p[4]), np.cos(p[5]), np.sin(p[5])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rx @ Ry @ Rz, np.asarray(p[:3], np.float64)


class IndepNdt:
    """pcl::VoxelGridCovariance + the DIRECT7 score of ndt_omp, numpy only"""

    def __init__(self, tgt, res, outlier_ratio=0.55):
        xyz = tgt[:, :3].astype(np.float64)
        ijk = np.floor(xyz / res).astype(np.int64)
        keys, inv, counts = np.unique(ijk, axis=0, return_inverse=True, return_counts=True)
        self.res, self.cells = res, {}
        order = np.argsort(inv.ravel(), kind="stable")
        starts = np.concatenate([[0], np.cumsum(counts)])
        for c in range(len(keys)):
            n = counts[c]
            if n < 6:
                continue
            p = xyz[order[starts[c]: starts[c + 1]]]
            cov = np.cov(p.T, bias=True) * (n - 1.0) / n       # PCL: single-pass population covariance, then (n-1)/n
            w, V = np.linalg.eigh(cov)
            if w[0] < 0 or w[1] < 0 or w[2] <= 0:
                continue
            lo = 0.01 * w[2]
            if w[0] < lo:
                w = np.maximum(w, lo)
                cov = (V * w) @ V.T
            self.cells[tuple(keys[c])] = (p.mean(axis=0), np.linalg.inv(cov))
        c1, c2 = 10.0 * (1 - outlier_ratio), outlier_ratio / res ** 3
        d3 = -np.log(c2)
        self.d1 = -np.log(c1 + c2) - d3
        self.d2 = -2 * np.log((-np.log(c1 * np.exp(-0.5) + c2) - d3) / self.d1)

    def cells_of(self, src, p):
        R, t = euler_xyz(p)
        return np.floor((src[:, :3].astype(np.float64) @ R.T + t) / self.res).astype(np.int64)

    def score(self, src, p, base=None):
        """base: cell assignment to use (the analytic gradient differentiates the score with the neighbourhood held fixed; a finite
        difference that lets points hop between cells would differentiate a discontinuous function)"""
        R, t = euler_xyz(p)
        x = src[:, :3].astype(np.float64) @ R.T + t
        if base is None:
            base = np.floor(x / self.res).astype(np.int64)
        total, pairs = 0.0, 0
        for off in ((0, 0, 0), (1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)):
            for i, key in enumerate(map(tuple, base + np.array(off))):
                cell = self.cells.get(key)
                if cell is None:
                    continue
                q = x[i] - cell[0]
                total += -self.d1 * np.exp(-0.5 * self.d2 * q @ cell[1] @ q)
                pairs += 1
        return total, pairs


def test_ndt_score_and_gradient_independent(synth, oracle):
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)
    src = synth.scan("vlp16_16k", frame=1, stride=8)[::4]   # 4096 points: the independent score is a Python loop
    m = oracle.NdtMap(tgt, 1.0)
    ind = IndepNdt(tgt, 1.0)
    dump = m.dump()
    assert int((dump["npts"] >= 6).sum()) == len(ind.cells)  # same set of valid voxels (n >= 6, positive definite)
    for p in (np.zeros(6), np.array([0.2, -0.1, 0.05, 0.01, -0.02, 0.03])):
        o = m.derivatives(src, p)
        s, pairs = ind.score(src, p)
        # ndt_omp reports score = sum of +d1... sign conventions: compare magnitudes of the Gaussian sum and the pair count exactly
        assert pairs == o["n_pairs"]
        assert abs(abs(s) - abs(o["score"])) <= 2e-5 * abs(s)   # per-pair math is float32 in ndt_omp / the oracle
        # gradient of the (sign-consistent) score by central differences
        sign = 1.0 if np.sign(s) == np.sign(o["score"]) else -1.0
        g = np.zeros(6)
        base = ind.cells_of(src, p)
        for k in range(6):
            h = 1e-4
            pp, pm = p.copy(), p.copy()
            pp[k] += h
            pm[k] -= h
            g[k] = sign * (ind.score(src, pp, base)[0] - ind.score(src, pm, base)[0]) / (2 * h)
        # ndt_omp's score_gradient is the gradient of -score_reported... accept either orientation, but it must be ONE orientation
        rel_pos = np.max(np.abs(g - o["g"])) / np.max(np.abs(g))
        rel_neg = np.max(np.abs(g + o["g"])) / np.max(np.abs(g))
        assert min(rel_pos, rel_neg) < 2e-3, (rel_pos, rel_neg)


def _rot_derivs(a):
    """R(a) about one axis and its first and second derivatives, for the x, y, z factors of R = Rx Ry Rz"""
    c, s = np.cos(a), np.sin(a)
    R = np.array([[c, -s], [s, c]])
    dR = np.array([[-s, -c], [c, -s]])
    return R, dR, -R


def _euler_factor(axis, a, order):
    M = np.zeros((3, 3))
    keep = [i for i in range(3) if i != axis]
    blk = _rot_derivs(a)[order]
    if axis == 1:  # Ry = [[c, 0, s], [0, 1, 0], [-s, 0, c]]: the 2x2 block acts on (z, x)
        blk = blk.T
    M[np.ix_(keep, keep)] = blk
    if order == 0:
        M[axis, axis] = 1.0
    return M


def indep_ndt_hessian(ind, src, p, cells_mask):
    """ndt_omp computeHessian restated from the definition: the Hessian in p of sum over (point, cell) of -d1 exp(-d2/2 q^T C q),
    q = R(p) x + t - mean, with dq/dp and d2q/dp2 from the derivatives of R = Rx Ry Rz (numpy float64; the (point, cell) pairs are
    the ones the oracle visited)"""
    x = src[:, :3].astype(np.float64)
    R, t = euler_xyz(p)
    F = [[_euler_factor(ax, p[3 + ax], o) for o in range(3)] for ax in range(3)]
    def dR(orders):  # noqa: E306
        return F[0][orders[0]] @ F[1][orders[1]] @ F[2][orders[2]]
    d1R = [dR([1 if k == a else 0 for k in range(3)]) for a in range(3)]
    d2R = [[dR([(a == k) + (b == k) for k in range(3)]) for b in range(3)] for a in range(3)]
    xt = x @ R.T + t
    base = np.floor(xt / ind.res).astype(np.int64)  # only used with the oracle's accepted offsets below
    H = np.zeros((6, 6))
    offs = ((0, 0, 0), (1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1))
    for i in range(x.shape[0]):
        if not cells_mask[i]:
            continue
        J = np.zeros((3, 6))
        J[:, :3] = np.eye(3)
        for a in range(3):
            J[:, 3 + a] = d1R[a] @ x[i]
        Hx = [[d2R[a][b] @ x[i] for b in range(3)] for a in range(3)]
        for c, off in enumerate(offs):
            if not (cells_mask[i] >> c) & 1:
                continue
            mean, C = ind.cells[tuple(base[i] + np.array(off))]
            q = xt[i] - mean
            e = np.exp(-0.5 * ind.d2 * q @ C @ q)
            qCJ = q @ C @ J
            sec = np.zeros((6, 6))
            for a in range(3):
                for b in range(3):
                    sec[3 + a, 3 + b] = q @ C @ Hx[a][b]
            H += ind.d1 * ind.d2 * e * (-ind.d2 * np.outer(qCJ, qCJ) + J.T @ C @ J + sec)
    return H


def test_ndt_hessian_pass_independent(synth, oracle):
    """the oracle's float64 Hessian pass (what k_ndt_hessian must reproduce) against the Hessian of the NDT score derived from its
    definition with numpy, on the same (point, cell) pairs"""
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)
    src = synth.scan("vlp16_16k", frame=1, stride=8)[::8]
    m = oracle.NdtMap(tgt, 1.0)
    ind = IndepNdt(tgt, 1.0)
    for p in (np.array([0.1, -0.05, 0.02, 0.0, 0.0, 0.0]), np.array([0.2, -0.1, 0.05, 0.01, -0.02, 0.03])):
        # the oracle picks cells by the float32 transform: keep the points that are not within 1e-4 of a cell face
        R, t = euler_xyz(p)
        xt = src[:, :3].astype(np.float64) @ R.T + t
        same = np.ones(src.shape[0], bool)
        for d in range(3):
            lo = np.floor(xt[:, d])
            same &= (np.abs(xt[:, d] - lo) > 1e-4) & (np.abs(xt[:, d] - lo - 1) > 1e-4)
        sub = src[same]
        o = m.hessian_at(sub, p)
        cells = m.derivatives(sub, p)["cells"]
        assert int(sum(bin(int(c)).count("1") for c in cells)) > 1000
        h = indep_ndt_hessian(ind, sub, p, cells)
        # the oracle transforms the point in float32 (~1e-6 m at these ranges): agreement to ~2e-5, a wrong term is off by O(1)
        assert relrel(o, h) < 1e-4, relrel(o, h)
