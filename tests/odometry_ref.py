"""Test-side restatement, in numpy float32, of the pose arithmetic and control flow of ScanMatchingOdometryNodelet::matching
(apps/scan_matching_odometry_nodelet.cpp:165-262), written from the reference's lines and independent of csrc/odometry_gate.cuh.

All functions take stacks of row-major 4x4 float32 matrices, shape (n, 4, 4), and work element-wise in float32 (numpy rounds every
float32 array operation once: products and sums are never fused).  `Replay` is the whole matching() walk for one sequence, with
the align supplied by the caller (the oracle)."""
import numpy as np

f32 = np.float32
REJECTED, ACCEPTED, KEYFRAME = 0, 1, 2


def mul4(a, b):
    """Eigen Matrix4f * Matrix4f: every entry the left-to-right dot product ((a0 b0 + a1 b1) + a2 b2) + a3 b3 in float32"""
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    o = np.empty(np.broadcast_shapes(a.shape, b.shape), f32)
    for r in range(4):
        for c in range(4):
            s = a[..., r, 0] * b[..., 0, c]
            s = s + a[..., r, 1] * b[..., 1, c]
            s = s + a[..., r, 2] * b[..., 2, c]
            s = s + a[..., r, 3] * b[..., 3, c]
            o[..., r, c] = s
    return o


def quat_w(m):
    """w of Eigen::Quaternionf(R) (Eigen/src/Geometry/Quaternion.h, quaternionbase_assign_impl<Other, 3, 3>): all four branches"""
    m = np.asarray(m, f32)
    out = np.empty(m.shape[:-2], f32)
    it = np.nditer(out, flags=["multi_index"], op_flags=["writeonly"])
    for cell in it:
        R = m[it.multi_index]
        t = f32(f32(R[0, 0] + R[1, 1]) + R[2, 2])
        if t > f32(0):
            cell[...] = f32(0.5) * np.sqrt(f32(t + f32(1)))
            continue
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j = (i + 1) % 3
        k = (j + 1) % 3
        t = np.sqrt(f32(f32(f32(R[i, i] - R[j, j]) - R[k, k]) + f32(1)))
        t = f32(0.5) / t
        cell[...] = f32(R[k, j] - R[j, k]) * t
    return out


def quat_branch(R):
    """which branch of the conversion a matrix takes: 'w' (trace > 0) or the index of the largest diagonal entry"""
    R = np.asarray(R, f32)
    if f32(f32(R[0, 0] + R[1, 1]) + R[2, 2]) > 0:
        return "w"
    i = 0
    if R[1, 1] > R[0, 0]:
        i = 1
    if R[2, 2] > R[i, i]:
        i = 2
    return i


def norm3(m):
    """`double d = m.block<3, 1>(0, 3).norm()`: a float32 norm, widened afterwards"""
    m = np.asarray(m, f32)
    x, y, z = m[..., 0, 3], m[..., 1, 3], m[..., 2, 3]
    return np.sqrt((x * x + y * y) + z * z).astype(np.float64)


def angle(m):
    """`double a = std::acos(Quaternionf(R).w())`: the float overload, widened afterwards.  Computed here as the float64 arc cosine
    rounded to float32, i.e. the correctly rounded acosf; a libm's acosf may differ from it by one float32 ulp."""
    with np.errstate(invalid="ignore"):
        return np.arccos(quat_w(m).astype(np.float64)).astype(f32).astype(np.float64)


def inverse_rigid(m):
    """prev_trans.inverse() as the engine documents it (DESIGN.md §2): the 3x3 block inverted by cofactors in float64, -A^-1 t in
    float64, every entry rounded to float32 once, last row 0 0 0 1"""
    m = np.asarray(m, f32).astype(np.float64)
    a = m[..., :3, :3].reshape(m.shape[:-2] + (9,))
    A = [a[..., i] for i in range(9)]
    c00 = A[4] * A[8] - A[5] * A[7]
    c01 = A[5] * A[6] - A[3] * A[8]
    c02 = A[3] * A[7] - A[4] * A[6]
    with np.errstate(all="ignore"):
        idet = 1.0 / ((A[0] * c00 + A[1] * c01) + A[2] * c02)
        Ai = [c00 * idet, (A[2] * A[7] - A[1] * A[8]) * idet, (A[1] * A[5] - A[2] * A[4]) * idet,
              c01 * idet, (A[0] * A[8] - A[2] * A[6]) * idet, (A[2] * A[3] - A[0] * A[5]) * idet,
              c02 * idet, (A[1] * A[6] - A[0] * A[7]) * idet, (A[0] * A[4] - A[1] * A[3]) * idet]
        o = np.zeros(m.shape, f32)
        for r in range(3):
            for c in range(3):
                o[..., r, c] = Ai[r * 3 + c]
            o[..., r, 3] = -((Ai[r * 3] * m[..., 0, 3] + Ai[r * 3 + 1] * m[..., 1, 3]) + Ai[r * 3 + 2] * m[..., 2, 3])
    o[..., 3, 3] = 1
    return o


def too_large(prev_trans, trans, max_acceptable_trans, max_acceptable_angle):
    """:224-228 -> (reject, dx, da)"""
    delta = mul4(inverse_rigid(prev_trans), trans)
    dx, da = norm3(delta), angle(delta)
    return (dx > max_acceptable_trans) | (da > max_acceptable_angle), dx, da


def wants_keyframe(trans, stamp, keyframe_stamp, keyframe_delta_trans, keyframe_delta_angle, keyframe_delta_time):
    """:241-244 -> (switch, delta_trans, delta_angle, delta_time)"""
    dt, da = norm3(trans), angle(trans)
    dtime = np.asarray(stamp, np.float64) - np.asarray(keyframe_stamp, np.float64)
    return (dt > keyframe_delta_trans) | (da > keyframe_delta_angle) | (dtime > keyframe_delta_time), dt, da, dtime


def gate(p, keyframe_pose, prev_trans, trans, converged, stamp, keyframe_stamp):
    """:214-252 for ONE frame -> (decision, odom)"""
    keyframe_pose, prev_trans, trans = (np.asarray(x, f32) for x in (keyframe_pose, prev_trans, trans))
    if not converged:
        return REJECTED, mul4(keyframe_pose, prev_trans)
    if p.get("transform_thresholding", False) and bool(too_large(prev_trans, trans, p["max_acceptable_trans"], p["max_acceptable_angle"])[0]):
        return REJECTED, mul4(keyframe_pose, prev_trans)
    odom = mul4(keyframe_pose, trans)
    sw = bool(wants_keyframe(trans, stamp, keyframe_stamp, p["keyframe_delta_trans"], p["keyframe_delta_angle"], p["keyframe_delta_time"])[0])
    return (KEYFRAME if sw else ACCEPTED), odom


class Replay:
    """matching() (:165-262) with every branch: the first frame, the guess prev_trans * msf_delta, the not-converged and the
    thresholding rejections (which leave prev_trans, prev_time and the keyframe alone), the three keyframe criteria.
    align(cloud, keyframe, guess) -> dict(T, converged, iterations) is the caller's (the oracle's)."""

    def __init__(self, align, **params):
        self.align = align
        self.p = dict(keyframe_delta_trans=0.25, keyframe_delta_angle=0.15, keyframe_delta_time=1.0, transform_thresholding=False,
                      max_acceptable_trans=1.0, max_acceptable_angle=1.0)
        self.p.update({k: v for k, v in params.items() if k in self.p})
        self.keyframe = None
        self.log = []  # per frame: dict(decision, dx, da, delta_trans, delta_angle, delta_time, by_trans, by_angle, by_time, ...)

    def matching(self, stamp, cloud, msf_delta=None):
        I = np.eye(4, dtype=f32)
        if self.keyframe is None:  # :166-174
            self.prev_trans, self.keyframe_pose, self.keyframe_stamp, self.keyframe = I.copy(), I.copy(), stamp, cloud
            self.log.append(dict(decision=KEYFRAME, first=True))
            return dict(odom=I, trans=I, converged=False, iterations=0, keyframe_updated=True, frame_rejected=False, keyframe=cloud)
        guess = mul4(self.prev_trans, I if msf_delta is None else np.asarray(msf_delta, f32))  # :210
        target = self.keyframe
        o = self.align(cloud, target, guess)
        trans = np.asarray(o["T"], f32)
        d, odom = gate(self.p, self.keyframe_pose, self.prev_trans, trans, o["converged"], stamp, self.keyframe_stamp)
        rec = dict(decision=d, first=False, converged=o["converged"], guess=guess)
        if o["converged"]:
            _, rec["dx"], rec["da"] = (float(x) for x in too_large(self.prev_trans, trans, np.inf, np.inf))
            _, dt, da, dtime = wants_keyframe(trans, stamp, self.keyframe_stamp, np.inf, np.inf, np.inf)
            rec.update(delta_trans=float(dt), delta_angle=float(da), delta_time=float(dtime), by_trans=bool(dt > self.p["keyframe_delta_trans"]),
                       by_angle=bool(da > self.p["keyframe_delta_angle"]), by_time=bool(dtime > self.p["keyframe_delta_time"]))
        self.log.append(rec)
        if d != REJECTED:
            self.prev_trans = trans  # :235-236
            if d == KEYFRAME:  # :245-251
                self.keyframe, self.keyframe_pose, self.keyframe_stamp, self.prev_trans = cloud, odom, stamp, I.copy()
        return dict(odom=odom, trans=trans, converged=o["converged"], iterations=o["iterations"], keyframe_updated=d == KEYFRAME,
                    frame_rejected=d == REJECTED, keyframe=target)
