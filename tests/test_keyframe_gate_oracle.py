"""The numpy restatement of GetNewObservations' map-consistency check (oracle/gate_check.py), pinned by properties:
g2o cannot be built here, so the SE3Quat maths is held against scipy's rotation vectors, log(exp(xi)) = xi on both
branches of log and near pi, and hand-worked cases on each side of both thresholds.  CPU only."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle import gate_check as G


def _T(R, t):
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = R
    T[:3, 3] = t
    return T


def test_quaternion_of_a_matrix_is_unit_with_nonnegative_w_and_round_trips():
    rng = np.random.default_rng(0)
    for R in list(Rotation.random(200, random_state=1).as_matrix()) + [np.diag([1.0, -1.0, -1.0]), np.diag([-1.0, 1.0, -1.0]),
                                                                       np.diag([-1.0, -1.0, 1.0]), np.eye(3)]:
        q = G.quat_from_matrix(R)
        assert abs(np.linalg.norm(q) - 1.0) < 1e-12 and q[0] >= 0.0
        np.testing.assert_allclose(G.rot(q), R, atol=1e-12)
    # a float matrix that is only nearly orthonormal still gives a unit quaternion
    R = (Rotation.from_rotvec(rng.normal(size=3)).as_matrix() * 1.001).astype(np.float32)
    assert abs(np.linalg.norm(G.quat_from_matrix(R)) - 1.0) < 1e-12


def test_log_rotation_part_matches_scipy_rotvec():
    rng = np.random.default_rng(2)
    for k in range(300):
        w = rng.normal(size=3)
        w *= rng.uniform(1e-4, 3.1) / np.linalg.norm(w)
        R = Rotation.from_rotvec(w)
        X = G.SE3Quat(G.quat_from_matrix(R.as_matrix()), rng.normal(size=3))
        np.testing.assert_allclose(X.log()[:3], R.as_rotvec(), atol=1e-8, err_msg=str(k))


@pytest.mark.parametrize("angle", [1e-7, 1e-4, 3e-3, 0.0044, 0.0045, 0.5, 2.0, np.pi - 1e-2, np.pi - 1e-4])
def test_log_inverts_exp_on_both_branches_and_near_pi(angle):
    rng = np.random.default_rng(int(angle * 1e6) % 1000)
    for _ in range(20):
        w = rng.normal(size=3)
        w *= angle / np.linalg.norm(w)
        xi = np.concatenate([w, rng.normal(size=3)])
        X = G.SE3Quat.exp(xi)
        d = 0.5 * (np.trace(G.rot(X.q)) - 1.0)
        branch_small = d > 0.99999
        assert branch_small == (angle < 0.00447), (angle, d)           # cos(a) = 0.99999 at a = 0.004472
        tol = 1e-6 if angle < np.pi - 1e-3 else 1e-4                    # near pi the rotation axis is ill-conditioned
        np.testing.assert_allclose(X.log(), xi, atol=tol, rtol=1e-6)


def test_inverse_and_product_are_group_operations():
    rng = np.random.default_rng(3)
    for _ in range(50):
        A = G.SE3Quat.exp(rng.normal(size=6))
        B = G.SE3Quat.exp(rng.normal(size=6))
        I = A.inverse() * A
        np.testing.assert_allclose(I.log(), np.zeros(6), atol=1e-9)
        AB = A * B
        x = rng.normal(size=3)
        np.testing.assert_allclose(G.rot(AB.q) @ x + AB.t, G.rot(A.q) @ (G.rot(B.q) @ x + B.t) + A.t, atol=1e-9)


def _map_pose():
    return _T(Rotation.from_euler("xyz", [0.1, -0.7, 0.05]).as_matrix(), [2.0, 0.5, 12.0])


def test_hand_worked_translation_threshold():
    M = _map_pose()
    for dx, dz, want in [(0.6, 0.79, G.KEPT), (0.6, 0.81, G.REJECTED), (0.0, 0.999, G.KEPT), (1.001, 0.0, G.REJECTED),
                         (0.0, 0.0, G.KEPT)]:
        Z = M.copy()
        Z[0, 3] += np.float32(dx); Z[2, 3] += np.float32(dz)
        dist2d, e = G.gate_values(Z, M)
        assert abs(dist2d - np.hypot(dx, dz)) < 1e-5
        assert e < 1.5                                                   # same rotation; |e| = |R_m^T dt| = |dt| < 1.3
        assert G.gate(Z, M) == want, (dx, dz, dist2d, e)
    # y alone does not count towards dist2D but does towards |e|
    Z = M.copy(); Z[1, 3] += np.float32(1.4)
    assert G.gate_values(Z, M)[0] == 0.0 and G.gate(Z, M) == G.KEPT
    Z = M.copy(); Z[1, 3] += np.float32(1.6)
    assert G.gate(Z, M) == G.REJECTED


def test_hand_worked_rotation_threshold():
    M = _map_pose()
    for angle, want in [(1.49, G.KEPT), (1.51, G.REJECTED), (3.0, G.REJECTED)]:
        # rotate about the object's own origin: t unchanged relative -> |e| = |omega| exactly (upsilon = 0)
        Rz = Rotation.from_rotvec([0.0, angle, 0.0]).as_matrix()
        Z = _T(M[:3, :3].astype(np.float64) @ Rz, M[:3, 3])
        dist2d, e = G.gate_values(Z, M)
        assert dist2d == 0.0 and abs(e - angle) < 1e-5, (angle, e)
        assert G.gate(Z, M) == want
    # rotation and translation each under their threshold, their combination over it
    Rz = Rotation.from_rotvec([0.0, 1.2, 0.0]).as_matrix()
    Z = _T(M[:3, :3].astype(np.float64) @ Rz, M[:3, 3] + M[:3, 1] * 1.0)
    assert G.gate_values(Z, M)[1] > 1.5 and G.gate(Z, M) == G.REJECTED


def test_nan_pose_is_rejected():
    M = _map_pose()
    Z = M.copy(); Z[0, 0] = np.nan
    assert G.gate(Z, M) == G.REJECTED
