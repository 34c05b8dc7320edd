"""The wide tensor-core engine (engine="tc_wide", DSPGN_ENGINE_TC_WIDE) on DeepSDF's own 8 x 512 decoder (built by
tests/wide_fixtures.py) against the reference's goldens, at the tolerances the 256-wide tensor-core engine meets on its
own: forward and input Jacobian (wide_stages.npz), one step from every state of the wide joint run (states_wide.npz),
the whole joint and pose-only runs (recon_wide.npz, pose_only_wide.npz); and the production paths on it: run-to-run
determinism, the gated, meshed keyframe call and its submitted form, a stopped object, meshes, a mixed-width solver, and
the refusal of a non-plain decoder.
"""
import copy
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import teacher_states as TS  # noqa: E402
import wide_fixtures as WF  # noqa: E402
from test_keyframe_batch import _bits, _cfg  # noqa: E402
from test_keyframe_mesh import _check_call, _stereo_keyframe  # noqa: E402
from test_teacher_forced import _check, _joint_obj, _one_iteration, _step_rows, _system_row  # noqa: E402

pytestmark = pytest.mark.gpu

WIDE_RUN = ("states_wide", "recon_wide", "wide", "kitti", 10, False, False)
STATUS_WORD, ITERS_WORD = 81, 84
ENGINE = "tc_wide"
TOL = "tc"          # tolerance keys of the teacher-forced helpers: the tensor-core engine's


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


_WIDE = {}


@pytest.fixture(scope="module", autouse=True)
def _wide_files(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("wide_decoders"))
    for n in WF.BUILDERS:
        _WIDE[n] = WF.write(n, d)


def _path(golden_dir, name):
    return _WIDE[name] if name in WF.BUILDERS else os.path.join(golden_dir, f"decoder_{name}.npz")


def _opt(golden_dir, cfg, name="wide", extra=("chairs",), engine=ENGINE, **kw):
    from dsp_slam_b200.optimizer import Optimizer
    return Optimizer(_path(golden_dir, name), cfg, extra_decoders=[_path(golden_dir, e) for e in extra], engine=engine, **kw)


@pytest.fixture(scope="module")
def wide_decoder(oracle, golden_dir, _wide_files):
    return oracle.DecoderWeights.from_npz(_path(golden_dir, "wide"))


def test_engine_choice_and_refusal(golden_dir, cfg_kitti):
    """tc_wide is taken when asked for, for a wide, a narrow and a mixed solver; AUTO and tc keep their choices; the
    LayerNorm + xyz_in_all variant is refused with a message that names the engine."""
    from dsp_slam_b200._lib import ENGINE_SIMT, ENGINE_TC_WIDE, DspgnError
    assert _opt(golden_dir, cfg_kitti, extra=()).solver.engine == ENGINE_TC_WIDE
    assert _opt(golden_dir, cfg_kitti, "cars", extra=()).solver.engine == ENGINE_TC_WIDE
    assert _opt(golden_dir, cfg_kitti, "cars", extra=("wide",)).solver.engine == ENGINE_TC_WIDE
    assert _opt(golden_dir, cfg_kitti, extra=(), engine=None).solver.engine == ENGINE_SIMT
    with pytest.raises(DspgnError, match="tensor-core engine unavailable for this decoder shape"):
        _opt(golden_dir, cfg_kitti, extra=(), engine="tc")
    with pytest.raises(DspgnError, match="DSPGN_ENGINE_TC_WIDE"):
        _opt(golden_dir, cfg_kitti, "wide_variant", extra=())


def test_forward_and_input_jacobian_vs_reference(golden_dir, cfg_kitti, oracle, wide_decoder):
    """decode_sdf and the SDF term's Jacobian rows and residuals against the reference's wide_stages.npz, at the levels
    of the 256-wide tensor-core engine (test_gpu_parity.py: forward 2e-5, rows 5e-4, residuals 2e-5)."""
    st = np.load(os.path.join(golden_dir, "wide_stages.npz"))
    opt = _opt(golden_dir, cfg_kitti, extra=())
    y = opt.solver.decode_sdf(st["dec_in"][0, :64], st["dec_in"][:, 64:67])
    print(f"\n[tc_wide] forward max |dy| {np.abs(y - st['dec_y']).max():.2e}")
    np.testing.assert_allclose(y, st["dec_y"], rtol=0, atol=2e-5)
    n_fg = st["rnd_rays"].shape[0] - 20
    opt.solver.upload([dict(t_cam_obj=TS.upload_pose(st["sdf_t_obj_cam"]), pts=st["sdf_pts"], code=st["sdf_z"],
                            rays=st["rnd_rays"], depth=st["rnd_depth_obs"][:n_fg])])
    g = opt.solver.debug_system(0, 0, want_rows=True, n_pts=st["sdf_pts"].shape[0])
    T = TS.library_state(st["sdf_t_obj_cam"])
    J, res = oracle.sdf_term(wide_decoder, st["sdf_pts"], T, st["sdf_z"])
    scale = np.abs(J).max()
    err = np.abs(g["J"] - J).max(axis=1) / scale
    err_ref = np.abs(g["J"] - st["sdf_J"]).max(axis=1) / scale
    kinks = _kink_units(oracle, wide_decoder, st["sdf_pts"], T, st["sdf_z"], 2e-6)
    off = [i for i in range(len(err)) if err[i] >= 5e-4]
    print(f"[tc_wide] relJ vs reference {err_ref.max():.2e}, vs oracle {err.max():.2e} (median row {np.median(err):.1e}), "
          f"rows beyond 5e-4 {off}, rows at a ReLU kink {kinks}, |dres| {np.abs(g['res'] - st['sdf_res']).max():.2e}")
    # A row beyond the tolerance must be one with a hidden unit whose pre-activation lies within the split-fp16 error of
    # the ReLU's kink (wide_stages row 181: layer 4 unit 177 at -3.7e-8): it matches the oracle with that unit's ReLU
    # mask taken the other way.  Every other row is within the tensor-core engine's tolerance.
    assert len(off) <= 0.01 * len(err), off
    for i in off:
        assert i in kinks and min(np.abs(g["J"][i] - _row_flipped(oracle, wide_decoder, st["sdf_pts"][i], T, st["sdf_z"], u)).max()
                                  for u in kinks[i]) / scale < 5e-4, i
    assert all(err_ref[i] < 5e-4 for i in range(len(err)) if i not in off)
    assert np.abs(g["res"] - st["sdf_res"]).max() < 2e-5 and np.abs(g["res"] - res).max() < 2e-5


def _pass(dw, inp, flip=None):
    """Pre-activations of every hidden layer and dy/d(input) of a plain decoder (one latent_in concat), with the ReLU
    mask of unit flip = (layer, unit) of every row taken the other way in the backward pass."""
    f32 = np.float32
    pre, masks, h = [], [], inp
    for k in range(dw.num_linear - 1):
        if k in dw.latent_in:
            h = np.concatenate([h, inp], 1)
        a = (h @ dw.W[k].T + dw.b[k]).astype(f32)
        m = a > 0
        if flip is not None and flip[0] == k:
            m[:, flip[1]] = ~m[:, flip[1]]
        pre.append(a); masks.append(m); h = np.maximum(a, f32(0))
    if dw.num_linear - 1 in dw.latent_in:
        h = np.concatenate([h, inp], 1)
    y = np.tanh((h @ dw.W[-1].T + dw.b[-1]).astype(f32)[:, 0]).astype(f32)
    g = ((f32(1) - y * y)[:, None] * dw.W[-1]).astype(f32)
    skip = np.zeros_like(inp)
    for k in range(dw.num_linear - 1, -1, -1):
        if k < dw.num_linear - 1:
            g = (g @ dw.W[k]).astype(f32)
        if k in dw.latent_in:
            skip += g[:, -inp.shape[1]:]
            g = g[:, :-inp.shape[1]]
        if k > 0:
            g = g * masks[k - 1]
    return pre, (g + skip).astype(f32)


def _inputs(oracle, pts, T, z):
    x = oracle.transform_points(T, pts).astype(np.float32)
    return x, np.concatenate([np.broadcast_to(z.astype(np.float32), (x.shape[0], z.shape[0])), x], 1)


def _kink_units(oracle, dw, pts, T, z, eps):
    """{row: [(layer, unit), ...]} of the hidden units whose pre-activation is within eps of 0."""
    pre, _ = _pass(dw, _inputs(oracle, pts, T, z)[1])
    out = {}
    for k, a in enumerate(pre):
        for i, j in zip(*np.nonzero(np.abs(a) < eps)):
            out.setdefault(int(i), []).append((k, int(j)))
    return out


def _row_flipped(oracle, dw, pt, T, z, unit):
    """The oracle's Jacobian row [pose | code] of one point with the ReLU mask of `unit` taken the other way."""
    x, inp = _inputs(oracle, pt[None, :], T, z)
    G = _pass(dw, inp, unit)[1]
    L = z.shape[0]
    return np.concatenate([oracle.pose_jacobian_rows(G[:, L:], x, 7), G[:, :L]], axis=1)[0]


def test_system_and_one_step_at_every_reference_state(golden_dir, cfg_kitti, cfg_redwood, oracle, wide_decoder):
    """Every state of the reference's wide joint run: the iteration-0 system (H, b, dx, V, m, losses) and the step a
    one-iteration reconstruct_batch applies, at the tensor-core single-step tolerances (H, b 3e-4; dx 2e-4)."""
    states, cfg = TS.joint_states(WIDE_RUN, cfg_kitti, cfg_redwood)
    opt = _opt(golden_dir, cfg, extra=())
    opt.solver.upload([_joint_obj(st) for st in states])
    rows = []
    for i, st in enumerate(states):
        it = oracle.gn_iteration(wide_decoder, oracle.GNConfig.from_json_dict(cfg), TS.library_state(st["Toc"]),
                                 st["z"], st["pts"], st["rays"], st["depth"])
        rows.append(_system_row(opt.solver.debug_system(i, 0), st, cfg, TOL, it))
    _check(rows, len(states), "wide tc_wide system (relH, relb, |ddx|, sdf loss, render loss)")
    j = cfg["optimizer"]["joint_optim"]
    for st in states:
        st.update(k1=j["k1"], k2=j["k2"], k4=j["k4"])
    cfg1 = _one_iteration(cfg)
    res = _opt(golden_dir, cfg1, extra=()).reconstruct_batch([_joint_obj(st) for st in states])
    _check(_step_rows(res, states, j["learning_rate"], TOL, oracle, {"wide": wide_decoder}, "wide", cfg1), len(states),
           "wide tc_wide one step (|dstep|, |dcode step|, loss)")


def test_whole_joint_and_pose_only_runs_vs_reference(golden_dir, cfg_kitti):
    """reconstruct_object and estimate_pose_cam_obj against the reference's whole runs, at the bounds of the fp32
    engine's test (test_wide_decoder_gpu.py); records are run-to-run bit-identical."""
    d = np.load(os.path.join(golden_dir, "recon_wide.npz"))
    opt = _opt(golden_dir, cfg_kitti, extra=())
    args = (np.asfortranarray(d["in_t_cam_obj"]), np.asfortranarray(d["in_pts"]), np.asfortranarray(d["in_rays"]), d["in_depth"])
    r = opt.reconstruct_object(*args)
    print(f"\n[tc_wide] whole run |dT| {np.abs(r.t_cam_obj - d['t_cam_obj']).max():.2e}, "
          f"|dz| {np.abs(r.code - d['code']).max():.2e}, loss {r.loss:.4e} vs {float(d['loss']):.4e}")
    assert r.is_good and bool(d["is_good"])
    assert np.abs(r.t_cam_obj - d["t_cam_obj"]).max() < 3e-2
    assert np.abs(r.code - d["code"]).max() < 1.5e-2
    assert abs(r.loss - float(d["loss"])) < 0.25 * abs(float(d["loss"])) + 1e-5
    r2 = opt.reconstruct_object(*args)
    assert np.array_equal(np.asarray(r2.t_cam_obj), np.asarray(r.t_cam_obj)) and np.array_equal(r2.code, r.code)
    p = np.load(os.path.join(golden_dir, "pose_only_wide.npz"))
    T = opt.estimate_pose_cam_obj(p["in_t_co_se3"].copy(), float(p["in_scale"]), p["in_pts"], p["in_code"])
    np.testing.assert_allclose(T, p["t_cam_obj"], rtol=0, atol=5e-4)


def test_gated_meshed_keyframe_submit_and_meshes(golden_dir, cfg_kitti):
    """The stereo keyframe of test_keyframe_mesh with the wide decoder as class 0 (chairs as class 1): records
    bit-identical run to run, the submitted call bit-identical to the blocking one, and each mesh bit-identical to
    mesh.marching_tetrahedra of the grid this engine decodes (MeshExtractor.sdf_grid, engine="tc_wide")."""
    from dsp_slam_b200.mesh import marching_tetrahedra
    from dsp_slam_b200.optimizer import MeshExtractor
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5))
    objs, modes, gates = _stereo_keyframe()
    n, dim = len(objs), 16
    got, meshes, words = _check_call(opt.solver, objs, modes, gates, dim)
    assert sum(m is not None for m in meshes) >= 2
    got2, _, _ = _check_call(opt.solver, objs, modes, gates, dim)
    assert np.array_equal(got, got2)
    opt.solver.keyframe_submit(objs, modes, gates, voxels_dim=dim)
    sub, sub_meshes = opt.solver.keyframe_wait()
    assert np.array_equal(_bits(sub, n), got)
    mx = {c: MeshExtractor(_path(golden_dir, nm), 64, dim, engine=ENGINE) for c, nm in ((0, "wide"), (1, "chairs"))}
    for i, (m, s) in enumerate(zip(meshes, sub_meshes)):
        assert (m is None) == (s is None), i
        if m is None:
            continue
        assert np.array_equal(m[0].view(np.uint32), s[0].view(np.uint32)) and np.array_equal(m[1], s[1]), i
        v, f = marching_tetrahedra(mx[objs[i]["class_id"]].sdf_grid(got[i, 16:80].view(np.float32)), 0.0,
                                   [2.0 / (dim - 1)] * 3)
        assert np.array_equal((v + np.array([-1.0, -1.0, -1.0])).astype(np.float32), m[0]), i
        assert np.array_equal(f.astype(np.int32), m[1]), i


def test_stop_of_a_wide_joint_object(golden_dir, cfg_kitti):
    """A stop raised by the device at iteration 3 of a wide joint object: it ends STOPPED with the record of the same
    call run for 4 iterations; every other record is bit-identical to the unstopped call."""
    from dsp_slam_b200 import _lib
    from test_keyframe_batch import _new, _tracked
    objs = [_new(961), _new(962), _tracked(963)]
    modes = [_lib.MODE_JOINT, _lib.MODE_JOINT, _lib.MODE_POSE]

    def call(iters, stop=None):
        cfg = copy.deepcopy(_cfg(cfg_kitti, 5))
        cfg["optimizer"]["joint_optim"]["num_iterations"] = iters
        opt = _opt(golden_dir, cfg)
        if stop is not None:
            opt.solver.debug_stop_at(*stop)
        out = _bits(opt.solver.keyframe(objs, modes), len(objs))
        opt.solver.close()
        return out

    base, got, short = call(10), call(10, (1, 3)), call(4)
    gi = got.view(np.int32)
    assert gi[1, STATUS_WORD] == _lib.ST_STOPPED and gi[1, ITERS_WORD] == 4
    want = short[1].copy(); have = got[1].copy()
    want[STATUS_WORD] = have[STATUS_WORD] = 0
    assert np.array_equal(have, want), np.flatnonzero(have != want)[:8]
    for i in (0, 2):
        if gi[i, STATUS_WORD] != _lib.ST_STOPPED:
            assert np.array_equal(got[i], base[i]), i


def test_mixed_width_solver(golden_dir, cfg_kitti):
    """A keyframe with a 256-wide class (cars) and the 512-wide class on the one engine: the objects succeed, and each
    record is bit-identical to the same object run alone (tiles never mix objects)."""
    from dsp_slam_b200 import _lib
    from test_keyframe_batch import _new, _tracked
    cfg = _cfg(cfg_kitti, 5)
    objs = [_new(971), dict(_new(972), class_id=1), _tracked(973), dict(_tracked(974), class_id=1), dict(_new(975), class_id=1)]
    modes = [_lib.MODE_JOINT, _lib.MODE_JOINT, _lib.MODE_POSE, _lib.MODE_POSE, _lib.MODE_JOINT]
    mixed = _opt(golden_dir, cfg, "cars", extra=("wide",))
    got = _bits(mixed.solver.keyframe(objs, modes), len(objs))
    assert (got.view(np.int32)[:, STATUS_WORD] == 0).sum() >= 4
    for i, (o, m) in enumerate(zip(objs, modes)):
        alone = _bits(mixed.solver.keyframe([o], [m]), 1)[0]
        assert np.array_equal(got[i], alone), (i, np.flatnonzero(got[i] != alone)[:8])
