"""The reference's state at every Gauss-Newton iteration (tests/golden/states_*.npz, pose_only_cut.npz, written by
`make_golden.py --states`) and what the teacher-forced tests need to start one step from each of them.

Two correct fp32 trajectories of this iteration separate exponentially (DESIGN.md section 2), so a trajectory cannot be
held to the reference tightly after a few iterations.  One step from the reference's own state at iteration k can:
that is what these fixtures pin.
"""
import copy
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# states file, whole-run golden, decoder, config, iterations, with_code, sdf_only
STATE_RUNS = [
    ("states_cfg1", "recon_cfg1", "cars", "kitti", 5, False, False),
    ("states_kitti250", "recon_kitti250", "cars", "kitti", 10, False, False),
    ("states_cfg2full", "recon_cfg2full", "cars", "kitti", 10, False, False),
    ("states_cfg3", "recon_cfg3", "chairs", "redwood", 10, True, False),
    ("states_cfg3_b8", "recon_cfg3_b8", "chairs", "redwood", 10, True, False),
    ("states_sdf_only", "recon_sdf_only", "cars", "kitti", 10, False, True),
    ("states_hyper", "recon_hyper", "cars", "hyper", 6, False, False),
]

POSE_CUT_ITERS = 8          # pose_only_cut.npz: estimate_pose_cam_obj with pose_only_optim.num_iterations = 8
POSE_CUT_AT = 4             # optimizer.py:76-78: the inlier cut after iteration index 4


def load(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def hyper_cfg(cfg_kitti, d):
    """The config of recon_hyper.npz: the KITTI config with every value its hyper_json moves."""
    hyper = json.loads(bytes(d["hyper_json"]).decode())
    cfg = copy.deepcopy(cfg_kitti)
    cfg["optimizer"]["num_depth_samples"] = hyper["num_depth_samples"]
    cfg["optimizer"]["cut_off_threshold"] = hyper["cut_off_threshold"]
    cfg["optimizer"]["joint_optim"].update(hyper["joint_optim"])
    return cfg


def run_cfg(cfgname, iters, cfg_kitti, cfg_redwood, d):
    """The config dict a whole-run golden was made with."""
    if cfgname == "hyper":
        cfg = hyper_cfg(cfg_kitti, d)
    else:
        cfg = copy.deepcopy(cfg_kitti if cfgname == "kitti" else cfg_redwood)
    cfg["optimizer"]["joint_optim"]["num_iterations"] = iters
    return cfg


def joint_states(run, cfg_kitti, cfg_redwood):
    """Every iteration k of one STATE_RUNS entry as a list of dicts: the reference's state (Toc = t_obj_cam, z), the
    run's inputs, and what the reference computed from that state (H, b, dx, V, m, sdf_loss, render_loss,
    and Toc_next / z_next after its update).  Also returns the config dict."""
    sname, gname, dec, cfgname, iters, with_code, sdf_only = run
    s, d = load(sname), load(gname)
    cfg = run_cfg(cfgname, iters, cfg_kitti, cfg_redwood, d)
    stacked = d["in_pts"].ndim == 3
    out = []
    for i in range(d["in_pts"].shape[0] if stacked else 1):
        g = (lambda k: d[k][i]) if stacked else (lambda k: d[k])
        h = (lambda k: s[k][i]) if stacked else (lambda k: s[k])
        for k in range(iters):
            st = dict(run=sname, obj=i, k=k, Toc=h("Toc_iters")[k], z=h("z_iters")[k],
                      Toc_next=h("Toc_iters")[k + 1], z_next=h("z_iters")[k + 1],
                      pts=g("in_pts"), H=g("H_iters")[k], b=g("b_iters")[k], dx=g("dx_iters")[k],
                      sdf_loss=float(h("sdf_loss_iters")[k]), render_loss=float(h("render_loss_iters")[k]))
            if not sdf_only:
                st.update(rays=g("in_rays"), depth=g("in_depth"), V=int(g("V_iters")[k]), m=int(g("m_iters")[k]))
            out.append(st)
    return out, cfg


def pose_states():
    """Every iteration k of pose_only_cut.npz: the state, the points the reference used (inliers only after the cut),
    the 6x6 system and the loss."""
    d = load("pose_only_cut")
    out = []
    for k in range(POSE_CUT_ITERS):
        pts = d["in_pts"] if k <= POSE_CUT_AT else d["in_pts"][d["inlier_mask"]]
        out.append(dict(run="pose_only_cut", obj=0, k=k, Toc=d["Toc_iters"][k], Toc_next=d["Toc_iters"][k + 1],
                        z=d["in_code"], pts=pts, scale=float(d["in_scale"]), H=d["H_iters"][k], b=d["b_iters"][k],
                        dx=d["dx_iters"][k], sdf_loss=float(d["sdf_loss_iters"][k])))
    return out


def upload_pose(Toc, scale=None):
    """The t_cam_obj a library call starts from to be at state Toc: inverted in float64, rounded to fp32.  With a scale
    (pose-only objects) the SE(3) part, scale divided out, as estimate_pose_cam_obj takes it (optimizer.py:45-55)."""
    T = np.linalg.inv(np.asarray(Toc, np.float64))
    if scale is not None:
        T[:3, :3] /= scale
    return T.astype(np.float32)


def rot_allowance(k4, t_obj_cam):
    """Absolute rounding of the rotation prior's entries of H and b (loss.py:155-178, optimizer.py:174-179).
    r = 1 - (R_co e_y).n_g is a difference of numbers near 1, so each fp32 evaluation of it carries about one ulp of 1
    (2^-23: measured between the oracle and the reference as |db| = k4 |J_rot| 2^-23, e.g. 4.1e-2 in b at cfg1 state 1,
    where |J_rot| = 3.5e-2 and |b| = 259).  The entries k4 J r of b and k4 J J^T of H move by k4 |J_rot| times that, and
    |J_rot| = sin(tilt) = sqrt(2 r) up to the same rounding.  Allowed: twice the measured rounding, 2^-22.  Where the
    object is upright (r = 0) the allowance is k4 2^-44, nothing; near the reference's gate r < 1e-7 (loss.py:171) it
    also covers the prior switching on in one evaluation and off in the other (k4 |J| r = 4.5e-4 against 1.1e-3)."""
    T = np.linalg.inv(np.asarray(t_obj_cam, np.float64))
    R = T[:3, :3] / np.cbrt(np.linalg.det(T[:3, :3]))
    j = np.sqrt(2.0 * max(1.0 + R[1, 1], 0.0)) + 2.0 ** -22
    return float(k4) * j * 2.0 ** -22


def library_state(Toc, scale=None):
    """The t_obj_cam the library holds after an upload of upload_pose(Toc, scale): the fp32 pose re-scaled and re-inverted
    in fp32 (one-ulp perturbations of Toc)."""
    T = upload_pose(Toc, scale)
    if scale is not None:
        T[:3, :3] *= np.float32(scale)
    return np.linalg.inv(T).astype(np.float32)


def pose_iteration(oracle, dw, Toc, z, pts):
    """One iteration of estimate_pose_cam_obj's loop body (optimizer.py:59-74) with the oracle's terms: H, b, dx, |res|."""
    J, res = oracle.sdf_term(dw, np.asarray(pts, np.float32), np.asarray(Toc, np.float32), z, pose_dim=6)
    J = J[:, :6]
    n = np.float32(J.shape[0])
    H = ((J.T @ J) / n + np.float32(1e-2) * np.eye(6, dtype=np.float32)).astype(np.float32)
    b = (-(J.T @ res) / n).astype(np.float32)
    dx = (np.linalg.inv(H).astype(np.float32) @ b).astype(np.float32)
    return dict(H=H, b=b, dx=dx, J=J, res=res)


def system_errors(H, b, dx, ref, k4):
    """(|dH|, |db|) relative to max |H|, max |b|, with the rotation-prior allowance taken off the prior's rows and
    columns 3..5, and |ddx| relative to max(1, |dx|)."""
    a = rot_allowance(k4, ref["Toc"])
    dH = np.abs(H - ref["H"]); db = np.abs(b - ref["b"])
    dH[3:6, :7] = np.maximum(dH[3:6, :7] - a, 0); dH[:7, 3:6] = np.maximum(dH[:7, 3:6] - a, 0)
    db[3:6] = np.maximum(db[3:6] - a, 0)
    eH = float(dH.max() / np.abs(ref["H"]).max())
    eb = float(db.max() / np.abs(ref["b"]).max())
    edx = float(np.abs(dx - ref["dx"]).max()) / max(1.0, float(np.abs(ref["dx"]).max()))
    return eH, eb, edx


def dx_tol(k4, ref, tol):
    """The single-step dx tolerance; where the rotation prior is on, 5e-4 max(1, |dx|) as in
    test_single_step_sdf_only_tilted_prior (the fp32 explicit inverse of a system with k4 = 1e7 entries)."""
    T = np.linalg.inv(np.asarray(ref["Toc"], np.float64))
    R = T[:3, :3] / np.cbrt(np.linalg.det(T[:3, :3]))
    return 5e-4 if float(k4) * (1.0 + R[1, 1]) > 1e-3 else tol


def flip_ok(dV, dm, V, m):
    """Boundary flips of the render row sets that two correct fp32 evaluations of one state can show."""
    return abs(dm) <= max(3, int(0.01 * m)) and abs(dV) <= max(2, int(2e-4 * V))
