"""The pose information of a record (dspgn_pose_information) restated in fp64 numpy (tests/pose_info_model.py) and held to
the reference's own normal matrices: for every golden with per-iteration systems, Lambda from the last H_iters with its
damping removed, about the measurement DSP-SLAM builds from the run's final pose.

  symmetry                 Lambda = Lambda^T to rounding (the restatement does not symmetrise);
  positive definiteness    every run the reference finished good;
  the tangent-space map    by finite differences: for random e (|e| = 1e-4) the measurement is perturbed to Z exp(e),
                           the solver's own perturbation delta of T_obj_cam between the two poses is recovered with the
                           SE(3) log map of oracle/gate_check.py, and 1/2 e^T Lambda e must equal the marginal quadratic
                           model 1/2 delta^T M delta of H to 1e-3.  The map itself is not used to compute delta.
"""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import pose_info_model as PI  # noqa: E402
from oracle.gate_check import SE3Quat, rot  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")
CFG = os.path.join(os.path.dirname(HERE), "dsp_slam_b200", "configs")

# golden, scale_damping of the config it was made with (None: pose-only)
JOINT = ["recon_cfg1", "recon_kitti250", "recon_cfg3_b8", "recon_hyper", "recon_wide"]


def s_damp_of(name):
    d = np.load(os.path.join(GOLDEN, name + ".npz"))
    if "hyper_json" in d.files:
        return float(json.loads(bytes(d["hyper_json"]).decode())["joint_optim"]["scale_damping"])
    cfg = "config_redwood_01053.json" if "cfg3" in name else "config_kitti.json"
    return float(json.load(open(os.path.join(CFG, cfg)))["optimizer"]["joint_optim"]["scale_damping"])


def cases():
    """(label, undamped H of the last iteration, record pose, pose-only scale or None, run good)"""
    out = []
    for name in JOINT:
        d = np.load(os.path.join(GOLDEN, name + ".npz"))
        sd = s_damp_of(name)
        stacked = d["H_iters"].ndim == 4
        for i in range(d["H_iters"].shape[0] if stacked else 1):
            g = (lambda k: d[k][i]) if stacked else (lambda k: d[k])
            out.append((f"{name}[{i}]", PI.undamped(g("H_iters")[-1], sd), g("t_cam_obj"), None, bool(g("is_good"))))
    d = np.load(os.path.join(GOLDEN, "pose_only_cut.npz"))
    out.append(("pose_only_cut", PI.undamped(d["H_iters"][-1]), d["t_cam_obj"], float(d["in_scale"]), True))
    return out


CASES = cases()


def se3_matrix(q):
    T = np.eye(4)
    T[:3, :3] = rot(q.q)
    T[:3, 3] = q.t
    return T


def solver_delta(Z, e, s):
    """delta = [rho | phi] with exp(delta) T_oc = T_oc' for the solver poses T_co = Z S and T_co' = Z exp(e) S, from the
    two poses and the SE(3) log map (SE3Quat.log orders (omega, upsilon))."""
    S = np.diag([s, s, s, 1.0])
    T_oc = np.linalg.inv(Z @ S)
    T_oc2 = np.linalg.inv(Z @ se3_matrix(SE3Quat.exp(e)) @ S)
    D = T_oc2 @ np.linalg.inv(T_oc)
    w_u = SE3Quat.from_matrix(D).log()
    return np.concatenate([w_u[3:], w_u[:3]])


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_symmetric_and_positive_definite(case):
    label, H, T, pose_scale, good = case
    s = PI.record_scale(T, pose_scale)
    L = PI.information(H, s)
    if not good:
        pytest.skip(f"{label}: the reference's run failed")
    assert L is not None, label
    # the Schur complement and the map keep the symmetry of H (to rounding; nothing symmetrises the result)
    assert np.abs(L - L.T).max() <= 1e-12 * np.abs(L).max(), (label, np.abs(L - L.T).max())
    assert np.all(np.linalg.eigvalsh(L) > 0), label


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_tangent_space_map_by_finite_differences(case):
    label, H, T, pose_scale, good = case
    if not good:
        pytest.skip(f"{label}: the reference's run failed")
    s = PI.record_scale(T, pose_scale)
    Z = PI.measurement(T, s)
    M = PI.marginal(H)
    L = PI.information(H, s)
    rng = np.random.default_rng(4013)
    worst, unmapped = 0.0, 0.0
    for _ in range(32):
        e = rng.standard_normal(6)
        e *= 1e-4 / np.linalg.norm(e)
        d = solver_delta(Z, e, s)
        q_edge, q_model = 0.5 * e @ L @ e, 0.5 * d @ M @ d
        worst = max(worst, abs(q_edge - q_model) / q_model)
        unmapped = max(unmapped, abs(0.5 * e @ M @ e - q_model) / q_model)
    print(f"\n[pose information] {label}: s = {s:.4f}, max rel. quadratic-form error {worst:.1e} (without the map: {unmapped:.1e})")
    assert worst < 1e-3, (label, worst)
    assert unmapped > 1e-2, (label, unmapped)     # the check can tell a wrong map from the right one
