"""numpy restatement of the map-consistency check of GetNewObservations (src/LocalMapping_util.cc:104-147), the check
dspgn_keyframe_batch_gated runs on the device (dsp_slam_b200/csrc/dspgn_solve.cuh: gate_decide).

A tracked detection's pose-only estimate Zco is compared with the pose the map predicts, Tco = Tcw * Two:
  dist2D  x/z translation difference, fp32 (Eigen::Vector2f::norm);
  e       log(Tco^-1 * Zco) with both poses as g2o SE3Quat (unit quaternion with w >= 0, translation), fp64.
Kept when dist2D < 1 and |e| < 1.5.  Test infrastructure only.
"""
import numpy as np

KEPT, REJECTED = 1, 2


def quat_from_matrix(R):
    """Unit quaternion (w, x, y, z), w >= 0, of a 3x3 rotation (fp64): the trace form when the trace is positive, else
    the form pivoted on the largest diagonal entry; then sign and norm as SE3Quat's constructor normalises them."""
    m = np.asarray(R, dtype=np.float64)
    v = np.zeros(4)                                   # x, y, z, w
    tr = m[0, 0] + m[1, 1] + m[2, 2]
    if tr > 0.0:
        s = np.sqrt(tr + 1.0)
        h = 0.5 / s
        v[3] = 0.5 * s
        v[0] = (m[2, 1] - m[1, 2]) * h
        v[1] = (m[0, 2] - m[2, 0]) * h
        v[2] = (m[1, 0] - m[0, 1]) * h
    else:
        i = 0
        if m[1, 1] > m[0, 0]:
            i = 1
        if m[2, 2] > m[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(m[i, i] - m[j, j] - m[k, k] + 1.0)
        h = 0.5 / s
        v[i] = 0.5 * s
        v[3] = (m[k, j] - m[j, k]) * h
        v[j] = (m[j, i] + m[i, j]) * h
        v[k] = (m[k, i] + m[i, k]) * h
    return normalise(np.array([v[3], v[0], v[1], v[2]]))


def normalise(q):
    q = np.array(q, dtype=np.float64)
    if q[0] < 0.0:
        q = -q
    return q / np.sqrt(np.sum(q * q))


def qmul(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return np.array([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw])


def rot(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


class SE3Quat:
    """(q, t): x -> R(q) x + t."""

    def __init__(self, q, t):
        self.q = normalise(q)
        self.t = np.asarray(t, dtype=np.float64).reshape(3)

    @classmethod
    def from_matrix(cls, T):
        T = np.asarray(T)
        return cls(quat_from_matrix(T[:3, :3].astype(np.float64)), T[:3, 3].astype(np.float64))

    def inverse(self):
        qi = self.q * np.array([1.0, -1.0, -1.0, -1.0])
        return SE3Quat(qi, rot(qi) @ -self.t)

    def __mul__(self, o):
        return SE3Quat(qmul(self.q, o.q), self.t + rot(self.q) @ o.t)

    def log(self):
        """(omega, upsilon): omega the rotation vector, upsilon = V^-1 t (se3quat.h's two branches, d > 0.99999 and acos)."""
        R = rot(self.q)
        d = 0.5 * (np.trace(R) - 1.0)
        dR = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
        with np.errstate(invalid="ignore", divide="ignore"):
            if d > 0.99999:
                w = 0.5 * dR
                c2 = 1.0 / 12.0
            else:
                th = np.arccos(d)
                w = th / (2.0 * np.sqrt(1.0 - d * d)) * dR
                c2 = (1.0 - th / (2.0 * np.tan(th / 2.0))) / (th * th)
            W = skew(w)
            Vinv = np.eye(3) - 0.5 * W + c2 * (W @ W)
        return np.concatenate([w, Vinv @ self.t])

    @staticmethod
    def exp(xi):
        """SE(3) exponential of (omega, upsilon), the inverse of log (closed form, fp64)."""
        w, u = np.asarray(xi[:3], np.float64), np.asarray(xi[3:], np.float64)
        th = np.linalg.norm(w)
        W = skew(w)
        if th < 1e-12:
            R, V = np.eye(3) + W, np.eye(3) + 0.5 * W
        else:
            R = np.eye(3) + np.sin(th) / th * W + (1 - np.cos(th)) / th ** 2 * (W @ W)
            V = np.eye(3) + (1 - np.cos(th)) / th ** 2 * W + (th - np.sin(th)) / th ** 3 * (W @ W)
        return SE3Quat(quat_from_matrix(R), V @ u)


def skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def gate_values(Z, M):
    """(dist2D (fp32), |e| (fp64)) of the estimate Z against the map's prediction M (4x4 float32 matrices)."""
    Z = np.asarray(Z, dtype=np.float32)
    M = np.asarray(M, dtype=np.float32)
    d3 = Z[:3, 3] - M[:3, 3]
    dist2d = np.sqrt(np.float32(d3[0] * d3[0]) + np.float32(d3[2] * d3[2]), dtype=np.float32)
    e = (SE3Quat.from_matrix(M).inverse() * SE3Quat.from_matrix(Z)).log()
    return np.float32(dist2d), float(np.sqrt(np.sum(e * e)))


def gate(Z, M):
    """KEPT (1) when dist2D < 1 and |e| < 1.5, else REJECTED (2); a NaN fails."""
    dist2d, e = gate_values(Z, M)
    return KEPT if (dist2d < 1.0 and e < 1.5) else REJECTED
