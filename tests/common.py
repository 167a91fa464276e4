"""shared helpers for the parity tests"""
import numpy as np


def rot_err(Ta, Tb):
    R = Ta[:3, :3].astype(np.float64).T @ Tb[:3, :3].astype(np.float64)
    # sin(angle) from the skew part: well conditioned near zero (arccos of the trace is not)
    v = 0.5 * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    s = float(np.linalg.norm(v))
    c = float(np.clip((np.trace(R) - 1) / 2, -1, 1))
    return float(np.arctan2(s, c)) if s > 1e-3 else s


def trans_err(Ta, Tb):
    return float(np.linalg.norm(Ta[:3, 3].astype(np.float64) - Tb[:3, 3].astype(np.float64)))


def perturb(seed, dt=0.3, dr_deg=2.0):
    rng = np.random.default_rng(seed)
    t = rng.uniform(-dt, dt, 3)
    a = np.deg2rad(rng.uniform(-dr_deg, dr_deg, 3))
    cx, sx, cy, sy, cz, sz = np.cos(a[0]), np.sin(a[0]), np.cos(a[1]), np.sin(a[1]), np.cos(a[2]), np.sin(a[2])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    T = np.eye(4)
    T[:3, :3] = Rz @ Ry @ Rx
    T[:3, 3] = t
    return T


VOXEL_KINDS = ("generic", "plane_z", "plane_diag", "line_x", "line_diag", "identical", "clamp_one_below", "clamp_one_above",
               "clamp_two", "clamp_none")


def voxel_points(kind, n, cell, res, rng, offset=(0.0, 0.0, 0.0)):
    """n float32 points (x y z 1) inside the NDT cell `cell` (integer ijk) of size `res`, shaped so the voxel's covariance is
    degenerate or sits at the eigenvalue clamp.  Coordinates are multiples of res/64 away from the cell faces, so they are exact
    in float32 (also after `offset`, a multiple of res/64) and exact planes / lines stay exact:
      plane_z (z = const), plane_diag (x - y = const), line_x (y, z const), line_diag (x = y = z up to the cell origin),
      identical (n copies of one point), clamp_*: 3 orthogonal point pairs whose eigenvalue ratios are 1 % -+ 1e-4 of the largest
      (one_below: the smallest is clamped, one_above: not, two: both smaller ones clamped, none: all above 1 %)."""
    o = (np.asarray(cell, np.float64) + 0.5) * res + np.asarray(offset, np.float64)  # cell centre
    q = res / 64.0
    u = lambda m: rng.integers(-20, 21, m) * q  # noqa: E731  grid offsets within +-0.31 res of the centre
    p = np.zeros((n, 3))
    if kind == "generic":
        p = np.c_[u(n), u(n), u(n)]
    elif kind == "plane_z":
        p = np.c_[u(n), u(n), np.full(n, 3 * q)]
    elif kind == "plane_diag":
        a = u(n)
        p = np.c_[a, a - 2 * q, u(n)]
    elif kind == "line_x":
        p = np.c_[u(n), np.full(n, -q), np.full(n, 5 * q)]
    elif kind == "line_diag":
        a = u(n)
        p = np.c_[a, a, a]
    elif kind == "identical":
        p = np.tile([[q, -2 * q, 3 * q]], (n, 1))
    else:
        r2 = {"clamp_one_below": (0.25, 0.0099), "clamp_one_above": (0.25, 0.0101), "clamp_two": (0.0099, 0.0098),
              "clamp_none": (0.25, 0.02)}[kind]
        a = 0.3 * res
        ax = [a, a * np.sqrt(r2[0]), a * np.sqrt(r2[1])]
        base = [np.eye(3)[d] * s * ax[d] for d in range(3) for s in (1.0, -1.0)]
        p = np.array([base[i % 6] for i in range(n)])
        if n % 6:  # extra points at the centre keep the mean and the axes
            p[6:] = 0.0
    pts = (o + p).astype(np.float32)
    return np.c_[pts, np.ones(n, np.float32)]


def relrel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def jacobisvd_diagonal_normal(C):
    """The PLANE normal of an exactly diagonal 3x3 C, whose tied eigenvalues leave the smallest eigenvector undefined: the column
    Eigen's JacobiSVD leaves last in U.  It does no rotation on a diagonal matrix; its step-4 sort swaps the FIRST maximum of the
    remaining |values| into place when it is not already there and stops at a zero maximum.  None for a matrix that is not diagonal."""
    C = np.asarray(C, np.float64)
    if C[0, 1] != 0.0 or C[0, 2] != 0.0 or C[1, 2] != 0.0:
        return None
    s = list(np.abs(np.diag(C)))
    col = [0, 1, 2]
    for i in range(3):
        pos = i + int(np.argmax(s[i:]))  # argmax returns the first maximum
        if s[pos] == 0.0:
            break
        s[i], s[pos] = s[pos], s[i]
        col[i], col[pos] = col[pos], col[i]
    return np.eye(3)[col[2]]


def axis_lines(n_per_axis=40, seed=0, length=(24, 40)):
    """(n, 4) float32 records: separated straight segments along x, y and z, points on a 0.25 grid, every coordinate off the
    segment's axis 0 or a power of two (so PCL's float32 raw moments are exact and the off-diagonals cancel to exactly 0) and
    every segment more than 50 m from any other (so the k nearest neighbours of each point, k < length[0], lie on its own
    segment).  The first segment of each axis lies on the axis itself.  Each neighbourhood's covariance is exactly diagonal."""
    rng = np.random.default_rng(seed)
    vals = np.array([0.0, 64.0, -64.0, 128.0, -128.0, 256.0, -256.0, 512.0])
    on_axis = [tuple(float(128 * axis) if a == axis else 0.0 for a in range(3)) for axis in range(3)]
    used = set(on_axis)
    segs = []
    for axis in range(3):
        for s in range(n_per_axis):
            c = on_axis[axis]
            while s > 0:
                c = tuple(float(v) for v in rng.choice(vals, 3))
                if c not in used:
                    used.add(c)
                    break
            m = int(rng.integers(length[0], length[1] + 1))
            p = np.tile(np.asarray(c), (m, 1))
            p[:, axis] += 0.25 * np.arange(m) - 4.0
            segs.append(p)
    p = np.concatenate(segs)
    p = p[rng.permutation(len(p))]
    return np.c_[p, np.ones(len(p))].astype(np.float32)
