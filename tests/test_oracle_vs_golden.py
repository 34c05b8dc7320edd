"""Pins the CPU oracle (oracle/dsp_oracle.py) against outputs of the UNMODIFIED reference
(tests/golden/*.npz, produced by tests/golden/make_golden.py on PyTorch-CPU).

Tolerances.  Single stages at a fixed state: fp32 re-association only (1e-6 .. 1e-5 relative).
Whole GN runs: the loop amplifies fp32 rounding through discrete decisions (ReLU masks, |x|<1,
|sdf|<th, de_do>1e-2; SURVEY.md Appendix B.3) -- two correct fp32 implementations differ by
~1e-3 (SDF only) to ~1e-2 (render term, few rays) in the final pose after 10 iterations, so the
end-to-end bounds below are that noise floor, while iteration 0 of every run is held to 1e-4.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import teacher_states as TS  # noqa: E402


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def test_weight_norm_fold(oracle_decoders, stages):
    dw = oracle_decoders["cars"]
    assert dw.num_linear == 9 and dw.latent_in == (4,)
    assert [w.shape for w in dw.W] == [(256, 67), (256, 256), (256, 256), (189, 256), (256, 256),
                                       (256, 256), (256, 256), (256, 256), (1, 256)]
    for k in range(9):
        np.testing.assert_allclose(dw.W[k], stages[f"cars_W{k}"], rtol=0, atol=2e-7)


def test_decoder_forward_and_input_grad(oracle, oracle_decoders, stages):
    dw = oracle_decoders["cars"]
    y = oracle.decoder_forward(dw, stages["dec_in"])
    np.testing.assert_allclose(y, stages["dec_y"], rtol=0, atol=2e-7)
    y2, g = oracle.decoder_value_and_input_grad(dw, stages["dec_in"])
    np.testing.assert_allclose(y2, stages["jac_y"], rtol=0, atol=2e-7)
    assert rel(g, stages["jac_g"]) < 2e-6


def test_input_grad_matches_finite_differences(oracle, oracle_decoders, stages):
    dw = oracle_decoders["cars"]
    x = stages["dec_in"][:4].astype(np.float64)
    _, g = oracle.decoder_value_and_input_grad(dw, x.astype(np.float32))
    W = [w.astype(np.float64) for w in dw.W]; B = [b.astype(np.float64) for b in dw.b]

    def f(v):
        h = v
        for k in range(9):
            if k == 4:
                h = np.concatenate([h, v])
            h = W[k] @ h + B[k]
            if k < 8:
                h = np.maximum(h, 0)
        return np.tanh(h[0])
    for r in range(4):
        for c in (0, 10, 63, 64, 65, 66):
            e = np.zeros(67); e[c] = 1e-5
            fd = (f(x[r] + e) - f(x[r] - e)) / 2e-5
            assert abs(fd - g[r, c]) < 2e-4 * max(1.0, abs(fd)), (r, c, fd, g[r, c])


def test_sdf_term(oracle, oracle_decoders, stages):
    J, res = oracle.sdf_term(oracle_decoders["cars"], stages["sdf_pts"], stages["sdf_t_obj_cam"], stages["sdf_z"])
    assert rel(J, stages["sdf_J"]) < 2e-6
    np.testing.assert_allclose(res, stages["sdf_res"], rtol=0, atol=1e-6)


def test_render_term(oracle, oracle_decoders, stages):
    r = oracle.render_term(oracle_decoders["cars"], stages["rnd_rays"], stages["rnd_depth_obs"],
                           stages["sdf_t_obj_cam"], stages["rnd_depths"], stages["sdf_z"], 0.01)
    assert r is not None
    J, res, ctr = r
    assert J.shape == stages["rnd_J"].shape          # same band rows kept, same order
    assert rel(J, stages["rnd_J"]) < 2e-5
    np.testing.assert_allclose(res, stages["rnd_res"], rtol=0, atol=1e-5)


def test_rotation_prior(oracle, stages):
    for nm in ("up", "tilt"):
        J, r = oracle.rotation_prior(stages[f"rot_{nm}_T"])
        np.testing.assert_allclose(J, stages[f"rot_{nm}_J"], rtol=0, atol=1e-7)
        assert abs(float(r) - float(stages[f"rot_{nm}_r"])) < 1e-7
    assert float(stages["rot_tilt_r"]) > 1e-4 and float(stages["rot_up_r"]) == 0.0


def test_exponential_maps(oracle, stages):
    for i, x in enumerate(stages["exp_x"]):
        np.testing.assert_allclose(oracle.exp_sim3(x), stages["exp_sim3"][i], rtol=0, atol=3e-6)
        np.testing.assert_allclose(oracle.exp_se3(x[:6]), stages["exp_se3"][i], rtol=0, atol=1e-6)
    np.testing.assert_array_equal(oracle.exp_sim3(np.zeros(7, np.float32)), np.eye(4, dtype=np.float32))
    # quirk loss_utils.py:223: c = 0 for a negative scale step with rotation
    T = oracle.exp_sim3(stages["exp_x"][1])
    np.testing.assert_allclose(T, stages["exp_sim3"][1], rtol=0, atol=1e-6)


def test_huber_and_linspace(oracle, stages):
    rr, loss, _ = oracle.robust_residual(stages["hub_r"], 0.025)
    np.testing.assert_array_equal(rr, stages["hub_rr"])
    assert abs(float(loss) - float(stages["hub_loss"])) < 1e-9
    assert rr[-3] == 0.0                                           # |r| == 0 -> weight 0
    lin = oracle.linspace_f32(stages["lin_ab"][0], stages["lin_ab"][1], 50)
    np.testing.assert_array_equal(lin, stages["lin_out"])


RUNS = [  # file, decoder, config, iters, with_code, sdf_only, tol_T, tol_code
    ("recon_cfg1", "cars", "kitti", 5, False, False, 5e-4, 2e-4),
    ("recon_kitti250", "cars", "kitti", 10, False, False, 3e-2, 1.5e-2),
    ("recon_cfg3", "chairs", "redwood", 10, True, False, 3e-2, 1e-2),
    ("recon_sdf_only", "cars", "kitti", 10, False, True, 3e-3, 1e-3),
]


@pytest.mark.parametrize("name,dec,cfgname,iters,with_code,sdf_only,tol_T,tol_code", RUNS)
def test_whole_runs(oracle, oracle_decoders, cfg_kitti, cfg_redwood, golden_dir, name, dec, cfgname, iters,
                    with_code, sdf_only, tol_T, tol_code):
    d = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg = oracle.GNConfig.from_json_dict(cfg_kitti if cfgname == "kitti" else cfg_redwood)
    cfg.num_iterations = iters
    trace = []
    out = oracle.reconstruct_object(oracle_decoders[dec], cfg, d["in_t_cam_obj"], d["in_pts"], d["in_rays"],
                                    d["in_depth"], code=d["in_code"] if with_code else None,
                                    sdf_only=sdf_only, trace=trace)
    assert out["is_good"] and bool(d["is_good"])
    # iteration 0 (identical state): tight
    assert rel(trace[0]["H"], d["H_iters"][0]) < 5e-5
    assert rel(trace[0]["b"], d["b_iters"][0]) < 5e-5
    assert np.abs(trace[0]["dx"] - d["dx_iters"][0]).max() < 1e-4
    # end to end: noise floor of the iteration (see module docstring)
    assert np.abs(out["t_cam_obj"] - d["t_cam_obj"]).max() < tol_T
    assert np.abs(out["code"] - d["code"]).max() < tol_code
    assert abs(float(out["loss"]) - float(d["loss"])) < 0.05 * abs(float(d["loss"])) + 1e-5


def test_full_size_and_batched_goldens(oracle, oracle_decoders, cfg_kitti, cfg_redwood, golden_dir):
    """The oracle against the reference at FULL size (config 2 with the render term: 2048 pts + 2248 rays, V ~ 1e5, band
    rows in the thousands) and on config 3's batch of 8: the render counters V and m of every iteration until the
    trajectories separate, iteration 0 tightly, the end state to the measured noise floor."""
    d = np.load(os.path.join(golden_dir, "recon_cfg2full.npz"))
    cfg = oracle.GNConfig.from_json_dict(cfg_kitti)
    tr = []
    out = oracle.reconstruct_object(oracle_decoders["cars"], cfg, d["in_t_cam_obj"], d["in_pts"], d["in_rays"], d["in_depth"], trace=tr)
    assert out["is_good"]
    # 112,400 samples: one |x| < 1 boundary decision flips between two fp32 evaluations of x_o (not a band sample)
    assert abs(tr[0]["V"] - int(d["V_iters"][0])) <= 2 and tr[0]["m"] == int(d["m_iters"][0])
    # fp32 summation over 3814 + 2048 rows in a different order than torch.bmm().sum(0): 7e-5
    assert rel(tr[0]["H"], d["H_iters"][0]) < 2e-4 and rel(tr[0]["b"], d["b_iters"][0]) < 2e-4
    for k in range(10):                                     # thousands of band rows: single flips only
        assert abs(tr[k]["V"] - int(d["V_iters"][k])) <= 20 and abs(tr[k]["m"] - int(d["m_iters"][k])) <= 0.01 * d["m_iters"][k] + 3
    assert np.abs(out["t_cam_obj"] - d["t_cam_obj"]).max() < 5e-3 and np.abs(out["code"] - d["code"]).max() < 2e-3   # SURVEY B.3
    d = np.load(os.path.join(golden_dir, "recon_cfg3_b8.npz"))
    cfg = oracle.GNConfig.from_json_dict(cfg_redwood)
    cfg.num_iterations = 10
    errs = []
    for i in range(8):
        tr = []
        out = oracle.reconstruct_object(oracle_decoders["chairs"], cfg, d["in_t_cam_obj"][i], d["in_pts"][i], d["in_rays"][i],
                                        d["in_depth"][i], code=d["in_code"][i], trace=tr)
        assert out["is_good"] and bool(d["is_good"][i])
        assert tr[0]["V"] == int(d["V_iters"][i, 0]) and tr[0]["m"] == int(d["m_iters"][i, 0])
        assert rel(tr[0]["H"], d["H_iters"][i, 0]) < 5e-5 and np.abs(tr[0]["dx"] - d["dx_iters"][i, 0]).max() < 1e-4
        assert rel(tr[1]["H"], d["H_iters"][i, 1]) < 2e-2 and tr[1]["V"] == int(d["V_iters"][i, 1])
        errs.append(float(np.abs(out["t_cam_obj"] - d["t_cam_obj"][i]).max()))
    # ~100 band rows per object: chaotic; 7 of 8 objects stay within 3e-2 of the reference, one separates (0.59)
    assert sorted(errs)[6] < 3e-2 and np.median(errs) < 1e-2, errs


def test_soft_failure_too_few_samples(oracle, oracle_decoders, cfg_kitti, golden_dir):
    d = np.load(os.path.join(golden_dir, "recon_fail_few.npz"))
    assert not bool(d["is_good"])
    cfg = oracle.GNConfig.from_json_dict(cfg_kitti)
    out = oracle.reconstruct_object(oracle_decoders["cars"], cfg, d["in_t_cam_obj"], d["in_pts"], d["in_rays"], d["in_depth"])
    assert not out["is_good"] and out["status"] == oracle.ST_RENDER_FEW
    assert out["t_cam_obj"] is None and out["code"] is None and float(out["loss"]) == float(d["loss"]) == 0.0


def test_pose_only(oracle, oracle_decoders, cfg_kitti, golden_dir):
    d = np.load(os.path.join(golden_dir, "pose_only.npz"))
    cfg = oracle.GNConfig.from_json_dict(cfg_kitti)
    T = oracle.estimate_pose_cam_obj(oracle_decoders["cars"], cfg, d["in_t_co_se3"], float(d["in_scale"]), d["in_pts"], d["in_code"])
    np.testing.assert_allclose(T, d["t_cam_obj"], rtol=0, atol=2e-5)


def test_decode_sdf_on_reference_voxel_grid(oracle, oracle_decoders, golden_dir):
    v = np.load(os.path.join(golden_dir, "voxel.npz"))
    s = oracle.decode_sdf(oracle_decoders["cars"], v["z"], v["vox8"])
    np.testing.assert_allclose(s, v["vox8_sdf"], rtol=0, atol=2e-7)


def test_decoder_variants_vs_reference(oracle, golden_dir):
    """LayerNorm + xyz_in_all + use_tanh + two latent_in layers (deep_sdf_decoder.py:41-47,58-63,87-102): the oracle's
    forward, input Jacobian and SDF-term rows against the reference's (tests/golden/variant.npz)."""
    dw = oracle.DecoderWeights.from_npz(os.path.join(golden_dir, "decoder_variant.npz"))
    st = np.load(os.path.join(golden_dir, "variant.npz"))
    assert dw.xyz_in_all and dw.use_tanh and dw.latent_in == (2, 4) and sum(x is not None for x in dw.ln) == 5
    y, g = oracle.decoder_value_and_input_grad(dw, st["dec_in"])
    np.testing.assert_allclose(y, st["dec_y"], rtol=0, atol=2e-6)
    np.testing.assert_allclose(y, st["jac_y"], rtol=0, atol=2e-6)
    np.testing.assert_allclose(g, st["jac_g"], rtol=0, atol=5e-6)
    J, res = oracle.sdf_term(dw, st["sdf_pts"], oracle.inv4(st["sdf_t_cam_obj"]), st["sdf_z"])
    assert rel(J, st["sdf_J"]) < 1e-5 and np.abs(res - st["sdf_res"]).max() < 3e-6


@pytest.mark.parametrize("run", [r[0] for r in TS.STATE_RUNS])
def test_teacher_forced_states_vs_reference(oracle, oracle_decoders, cfg_kitti, cfg_redwood, run):
    """One oracle GN iteration from the reference's OWN state at every iteration k of every whole-run golden
    (tests/golden/states_*.npz) against the reference's iteration k: H, b, dx, the render counters V, m and both losses to
    the iteration-0 tolerances.  Also validates the fixtures: state k+1 is the reference's update exp_sim3(lr dx_k) state k.
    States where V or m differ by boundary flips are held to 3x those tolerances, except that at most 10 % of a run's states
    may exceed even that: one band row of ~100 is a different system (cfg3_b8 object 1, state 6: H moves by 5e-2).
    In the rotation prior's rows the comparison allows the prior's own fp32 rounding (rot_allowance)."""
    spec = next(r for r in TS.STATE_RUNS if r[0] == run)
    states, cfg = TS.joint_states(spec, cfg_kitti, cfg_redwood)
    ocfg = oracle.GNConfig.from_json_dict(cfg)
    dw, sdf_only = oracle_decoders[spec[2]], spec[6]
    tol = 2e-4                # as iteration 0 of cfg2full (test_full_size_and_batched_goldens); measured up to 1.8e-4 (sdf_only, k = 4)
    L = ocfg.code_len
    worst, flips, off = np.zeros(5), [], []
    for st in states:
        T_next = (oracle.exp_sim3(np.float32(ocfg.lr) * st["dx"][:7]) @ st["Toc"]).astype(np.float32)
        assert np.abs(T_next - st["Toc_next"]).max() < 2e-5 * max(1.0, np.abs(st["Toc_next"]).max()), (st["obj"], st["k"])
        np.testing.assert_array_equal((st["z"] + np.float32(ocfg.lr) * st["dx"][7:7 + L]).astype(np.float32), st["z_next"])
        it = oracle.gn_iteration(dw, ocfg, st["Toc"], st["z"], st["pts"], st.get("rays"), st.get("depth"), sdf_only=sdf_only)
        assert it["status"] == oracle.ST_OK
        eH, eb, edx = TS.system_errors(it["H"], it["b"], it["dx"], st, ocfg.k4)
        el_s = abs(float(it["sdf_loss"]) - st["sdf_loss"]) / st["sdf_loss"]
        el_r = abs(float(it["render_loss"]) - st["render_loss"]) / max(st["render_loss"], 1e-30)
        e = (eH, eb, edx, el_s, el_r)
        lim = (tol, tol, TS.dx_tol(ocfg.k4, st, 1e-4), 5e-5, 5e-5)
        if not sdf_only and (it["V"], it["m"]) != (st["V"], st["m"]):
            assert TS.flip_ok(it["V"] - st["V"], it["m"] - st["m"], st["V"], st["m"]), (st["obj"], st["k"], it["V"], it["m"])
            flips.append((st["obj"], st["k"], it["V"] - st["V"], it["m"] - st["m"]))
            if any(x >= 3 * y for x, y in zip(e, lim)):
                off.append((st["obj"], st["k"]) + tuple(round(x, 6) for x in e))
            continue
        worst = np.maximum(worst, e)
        assert all(x < y for x, y in zip(e, lim)), (st["obj"], st["k"], e)
    print(f"\n[teacher-forced oracle] {run}: {len(states)} states, max relH {worst[0]:.1e} relb {worst[1]:.1e} "
          f"|ddx| {worst[2]:.1e} sdf loss {worst[3]:.1e} render loss {worst[4]:.1e}; flips (obj, k, dV, dm) {flips}, "
          f"beyond 3x the tolerances {off}")
    assert len(off) <= 0.1 * len(states)


def test_teacher_forced_pose_only_cut_vs_reference(oracle, oracle_decoders):
    """pose_only_cut.npz: 8 iterations of estimate_pose_cam_obj on a car with 10 % gross outliers.  From the reference's
    state at every iteration, the oracle's 6x6 system and step equal the reference's; the stored inlier mask is |res| <= 0.05
    at state 4 (optimizer.py:76-78) and removes the outliers; state k+1 is exp_se3(dx_k) state k."""
    d = TS.load("pose_only_cut")
    dw = oracle_decoders["cars"]
    mask = d["inlier_mask"]
    assert mask.shape == (300,) and 0 < (~mask).sum() <= 30
    for st in TS.pose_states():
        T_next = (oracle.exp_se3(st["dx"]) @ st["Toc"]).astype(np.float32)
        assert np.abs(T_next - st["Toc_next"]).max() < 2e-5 * max(1.0, np.abs(st["Toc_next"]).max()), st["k"]
        it = TS.pose_iteration(oracle, dw, st["Toc"], st["z"], st["pts"])
        J, res, H, b, dx = it["J"], it["res"], it["H"], it["b"], it["dx"]
        n = np.float32(J.shape[0])
        _, loss, _ = oracle.robust_residual(res, 0.05)
        if st["k"] == TS.POSE_CUT_AT:
            np.testing.assert_array_equal(np.abs(res) <= np.float32(0.05), mask)
        assert rel(H, st["H"]) < (1e-3 if st["k"] > TS.POSE_CUT_AT else 5e-5), st["k"]     # 271 rows after the cut: 7e-4
        # b -> 0 as the pose converges: its rounding is relative to the summands, |J| |res| / n
        assert np.abs(b - st["b"]).max() < 1e-3 * float((np.abs(J) * np.abs(res)[:, None]).sum(0).max() / n), st["k"]
        assert np.abs(dx - st["dx"]).max() < 1e-5, st["k"]
        assert abs(float(loss) - st["sdf_loss"]) < 2e-5 * st["sdf_loss"], st["k"]
    T = oracle.inv4(d["Toc_iters"][-1]); T[:3, :3] /= np.float32(d["in_scale"])
    np.testing.assert_allclose(T, d["t_cam_obj"], rtol=0, atol=2e-6)


def test_every_hyper_parameter_is_read_like_the_reference(oracle, oracle_decoders, cfg_kitti, golden_dir):
    """`recon_hyper.npz`: a reference run with EVERY value of the `optimizer` block moved off the shipped configs (D = 24
    depth samples, band half-width 0.02, k1..k4, b1, b2, learning rate, scale damping, 6 iterations) and the initial pose
    tilted 3 degrees so that the rotation prior is active (optimizer.py:27-43,120-126,155-192; loss.py:84-141,155-178).
    The restatement must read each of them where the reference does: the render counters V and m of every iteration, the
    system of iteration 0 tightly (k4 |J_rot|^2 = 5.5 and s_damp = 2 against max |H| = 170: a wrong coefficient is a 1e-2
    effect), later systems and the end state to the noise floor (measured: H 3.5e-3 at iteration 5, |dT| 5e-4, |dcode| 2e-3).
    (This golden was added after the round's GPU budget was spent: it pins the oracle; the CUDA path has not been run on it.)"""
    import copy
    import json
    d = np.load(os.path.join(golden_dir, "recon_hyper.npz"))
    hyper = json.loads(bytes(d["hyper_json"]).decode())
    cfgd = copy.deepcopy(cfg_kitti)
    cfgd["optimizer"]["num_depth_samples"] = hyper["num_depth_samples"]
    cfgd["optimizer"]["cut_off_threshold"] = hyper["cut_off_threshold"]
    cfgd["optimizer"]["joint_optim"].update(hyper["joint_optim"])
    cfg = oracle.GNConfig.from_json_dict(cfgd)
    assert (cfg.num_depth_samples, cfg.num_iterations, cfg.cut_off, cfg.lr, cfg.s_damp, cfg.k4) == (24, 6, 0.02, 0.8, 2.0, 2000.0)
    trace = []
    out = oracle.reconstruct_object(oracle_decoders["cars"], cfg, d["in_t_cam_obj"], d["in_pts"], d["in_rays"], d["in_depth"],
                                    trace=trace)
    assert out["is_good"] and bool(d["is_good"]) and len(trace) == 6
    V, m = np.array([t["V"] for t in trace]), np.array([t["m"] for t in trace])
    assert V[0] == d["V_iters"][0] and m[0] == d["m_iters"][0]
    assert np.abs(V - d["V_iters"]).max() <= 2 and np.abs(m - d["m_iters"]).max() <= 4      # boundary flips only
    _, r_rot = oracle.rotation_prior(oracle.inv4(d["in_t_cam_obj"].astype(np.float32)))
    assert r_rot > 1e-3                                                                     # the prior is active
    assert rel(trace[0]["H"], d["H_iters"][0]) < 1e-4 and rel(trace[0]["b"], d["b_iters"][0]) < 1e-4
    assert np.abs(trace[0]["dx"] - d["dx_iters"][0]).max() < 2e-5
    for k in range(1, 6):
        assert rel(trace[k]["H"], d["H_iters"][k]) < 2e-2 and np.abs(trace[k]["dx"] - d["dx_iters"][k]).max() < 1e-2, k
    assert np.abs(out["t_cam_obj"] - d["t_cam_obj"]).max() < 5e-3
    assert np.abs(out["code"] - d["code"]).max() < 8e-3
    assert abs(float(out["loss"]) - float(d["loss"])) < 0.02 * abs(float(d["loss"]))
