"""fp64 numpy restatement of dspgn_pose_information (dsp_slam_b200/csrc/dspgn_solve.cuh: k_pose_information, DESIGN.md
section 4.13): the pose information of a record from the normal matrix H of the iteration its pose came from.

  undamped     H without the solve's damping: joint -1 on the pose diagonal and -s_damp on scale, pose-only -1e-2 I.
  marginal     the Schur complement of H onto the six pose coordinates [rho | phi] (scale and code eliminated).
  edge_map     the 6x6 matrix A with delta = A e: the solver's left perturbation delta of T_obj_cam caused by the
               perturbation Z exp(e) of the edge's measurement Z, e = [omega | upsilon], at scale s.
  information  A^T M A (not symmetrised), or None when the marginal system is not positive definite.
Test infrastructure only.
"""
import numpy as np


def undamped(H, s_damp=None):
    """H (P x P) of a joint solve (s_damp given) or a pose-only solve (s_damp None) without its damping, fp64.  Its upper
    triangle, mirrored: the solver keeps only that triangle (an fp32 J^T J need not be symmetric to the last bit)."""
    H = np.triu(np.asarray(H, dtype=np.float64))
    H = H + np.triu(H, 1).T
    if s_damp is None:
        H[np.arange(6), np.arange(6)] -= 1e-2
    else:
        H[np.arange(7), np.arange(7)] -= 1.0
        H[6, 6] -= float(s_damp)
    return H


def marginal(H):
    """Schur complement onto rows / columns 0..5, or None when the eliminated block or the result is not positive
    definite."""
    H = np.asarray(H, np.float64)
    A, B, C = H[:6, :6], H[:6, 6:], H[6:, 6:]
    if C.shape[0]:
        try:
            np.linalg.cholesky(C)
        except np.linalg.LinAlgError:
            return None
        A = A - B @ np.linalg.solve(C, B.T)
    try:
        np.linalg.cholesky(A)          # reads one triangle: symmetry is the caller's to check
    except np.linalg.LinAlgError:
        return None
    return A


def edge_map(s):
    """delta = [rho | phi] of T_oc' = exp(delta) T_oc for T_co' = Z exp(e) S, S = diag(s, s, s, 1):
    exp(delta) = S^-1 exp(-e) S, so rho = -upsilon / s and phi = -omega."""
    A = np.zeros((6, 6))
    A[0:3, 3:6] = -np.eye(3) / s
    A[3:6, 0:3] = -np.eye(3)
    return A


def record_scale(T, pose_scale=None):
    """s of a record: the pose-only call's scale argument, else cbrt(det R) of the record's Sim(3) pose."""
    if pose_scale is not None:
        return float(pose_scale)
    return float(np.cbrt(np.linalg.det(np.asarray(T, np.float64)[:3, :3])))


def measurement(T, s):
    """Z: the record's pose with its scale divided out of the rotation (SetPoseMeasurementSim3 / SE3)."""
    Z = np.array(T, dtype=np.float64)
    Z[:3, :3] /= s
    Z[3] = (0, 0, 0, 1)
    return Z


def information(H_undamped, s):
    """The record's 6x6 information in the edge's tangent space, or None (not positive definite)."""
    M = marginal(H_undamped)
    if M is None:
        return None
    A = edge_map(s)
    return A.T @ M @ A
