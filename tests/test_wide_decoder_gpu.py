"""Decoders with layers wider than 256 on the GPU: DeepSDF's own 8 x 512 network and a 512-wide LayerNorm + xyz_in_all
variant (both built by tests/wide_fixtures.py) run on the fp32 SIMT engine's 512 instantiation.

The engine choice; forward and input Jacobian against the reference's stages (wide_stages.npz, wide_variant.npz); one
step from every state of the reference's joint run (states_wide.npz) at the fp32 engine's single-step tolerances; the
whole joint and pose-only runs at the whole-run levels of DESIGN.md section 2; the gated, meshed keyframe call, its
submitted form and its stop; and a mixed batch of a 256-wide and a 512-wide class.
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


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


_WIDE = {}     # the 512-wide decoders (tests/wide_fixtures.py), written once per module


@pytest.fixture(scope="module", autouse=True)
def _wide_files(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("wide_decoders"))
    for n in WF.BUILDERS:
        _WIDE[n] = WF.write(n, d)


def _path(golden_dir, name):
    return _WIDE[name] if name in WF.BUILDERS else os.path.join(golden_dir, f"decoder_{name}.npz")


def _opt(golden_dir, cfg, name="wide", extra=("chairs",), **kw):
    from dsp_slam_b200.optimizer import Optimizer
    return Optimizer(_path(golden_dir, name), cfg, extra_decoders=[_path(golden_dir, e) for e in extra], **kw)


@pytest.fixture(scope="module")
def wide_decoders(oracle, golden_dir, _wide_files):
    return {n: oracle.DecoderWeights.from_npz(_path(golden_dir, n)) for n in ("wide", "wide_variant")}


def test_engine_choice(golden_dir, cfg_kitti):
    from dsp_slam_b200._lib import ENGINE_SIMT, DspgnError
    assert _opt(golden_dir, cfg_kitti, extra=()).solver.engine == ENGINE_SIMT
    assert _opt(golden_dir, cfg_kitti, extra=("cars",)).solver.engine == ENGINE_SIMT
    assert _opt(golden_dir, cfg_kitti, "cars", extra=("wide",)).solver.engine == ENGINE_SIMT
    with pytest.raises(DspgnError, match="tensor-core engine unavailable for this decoder shape"):
        _opt(golden_dir, cfg_kitti, extra=(), engine="tc")


@pytest.mark.parametrize("name,golden", [("wide", "wide_stages"), ("wide_variant", "wide_variant")])
def test_forward_and_input_jacobian_vs_reference(name, golden, golden_dir, cfg_kitti, oracle, wide_decoders):
    """decode_sdf against the reference's forward; the SDF term's Jacobian rows (d sdf / d input through the pose and
    code columns) and residuals against the reference's compute_sdf_loss, and against the oracle at the state the
    library holds after the upload."""
    st = np.load(os.path.join(golden_dir, golden + ".npz"))
    opt = _opt(golden_dir, cfg_kitti, name, extra=(), engine="simt")
    y = opt.solver.decode_sdf(st["dec_in"][0, :64], st["dec_in"][:, 64:67])
    np.testing.assert_allclose(y, st["dec_y"], rtol=0, atol=2e-6)
    n_fg = st["rnd_rays"].shape[0] - 20
    opt.solver.upload([dict(t_cam_obj=TS.upload_pose(st["sdf_t_obj_cam"]), pts=st["sdf_pts"], code=st["sdf_z"],
                            rays=st["rnd_rays"], depth=st["rnd_depth_obs"][:n_fg])])
    g = opt.solver.debug_system(0, 0, want_rows=True, n_pts=st["sdf_pts"].shape[0])
    J, res = oracle.sdf_term(wide_decoders[name], st["sdf_pts"], TS.library_state(st["sdf_t_obj_cam"]), st["sdf_z"])
    print(f"\n[{name}] relJ vs reference {rel(g['J'], st['sdf_J']):.2e}, vs oracle {rel(g['J'], J):.2e}")
    assert rel(g["J"], st["sdf_J"]) < 5e-5
    assert np.abs(g["res"] - st["sdf_res"]).max() < 2e-6
    assert rel(g["J"], J) < 2e-5 and np.abs(g["res"] - res).max() < 2e-6


@pytest.mark.parametrize("name", ["variant", "wide_variant"])
def test_layernorm_rows_with_the_render_term(name, golden_dir, cfg_kitti, oracle):
    """A LayerNorm decoder's SDF rows while the ray-sample pass runs beside them (it has its own LayerNorm scratch), at
    both SIMT instantiations, against the oracle at the state the library holds."""
    from dsp_slam_b200 import synth
    dw = oracle.DecoderWeights.from_npz(_path(golden_dir, name))
    o = synth.make_object(31, 400, 300, 60)
    z = (0.3 * np.random.default_rng(31).standard_normal(64)).astype(np.float32)
    opt = _opt(golden_dir, cfg_kitti, name, extra=(), engine="simt")
    opt.solver.upload([dict(t_cam_obj=o["t_cam_obj_init"], pts=o["pts"], rays=o["rays"], depth=o["depth"], code=z)])
    g = opt.solver.debug_system(0, 0, want_rows=True, n_pts=400)
    J, res = oracle.sdf_term(dw, np.asarray(o["pts"]), oracle.inv4(np.asarray(o["t_cam_obj_init"], np.float32)), z)
    assert g["V"] > 0 and rel(g["J"], J) < 5e-5 and np.abs(g["res"] - res).max() < 2e-6


def test_system_at_every_reference_state(golden_dir, cfg_kitti, cfg_redwood, oracle, wide_decoders):
    """Every state of the reference's wide joint run uploaded as one batch: each object's iteration-0 system against the
    reference's iteration k (H, b, dx, V, m, both losses) at the fp32 engine's tolerances."""
    states, cfg = TS.joint_states(WIDE_RUN, cfg_kitti, cfg_redwood)
    opt = _opt(golden_dir, cfg, extra=(), engine="simt")
    opt.solver.upload([_joint_obj(st) for st in states])
    rows = []
    for i, st in enumerate(states):
        it = oracle.gn_iteration(wide_decoders["wide"], oracle.GNConfig.from_json_dict(cfg), TS.library_state(st["Toc"]),
                                 st["z"], st["pts"], st["rays"], st["depth"])
        rows.append(_system_row(opt.solver.debug_system(i, 0), st, cfg, "simt", it))
    _check(rows, len(states), "wide simt system (relH, relb, |ddx|, sdf loss, render loss)")


def test_one_step_through_the_production_path(golden_dir, cfg_kitti, cfg_redwood, oracle, wide_decoders):
    """reconstruct_batch with one iteration from every state of the wide run: the applied steps, n_valid / n_band and the
    loss against the reference's iteration k."""
    states, cfg = TS.joint_states(WIDE_RUN, cfg_kitti, cfg_redwood)
    j = cfg["optimizer"]["joint_optim"]
    for st in states:
        st.update(k1=j["k1"], k2=j["k2"], k4=j["k4"])
    cfg = _one_iteration(cfg)
    res = _opt(golden_dir, cfg, extra=(), engine="simt").reconstruct_batch([_joint_obj(st) for st in states])
    _check(_step_rows(res, states, j["learning_rate"], "simt", oracle, wide_decoders, "wide", cfg), len(states),
           "wide simt one step (|dstep|, |dcode step|, loss)")


def test_whole_joint_and_pose_only_runs_vs_reference(golden_dir, cfg_kitti):
    """reconstruct_object and estimate_pose_cam_obj against the reference's whole runs, at the levels of
    recon_kitti250 / pose_only in test_gpu_parity.py."""
    d = np.load(os.path.join(golden_dir, "recon_wide.npz"))
    opt = _opt(golden_dir, cfg_kitti, extra=())
    r = opt.reconstruct_object(np.asfortranarray(d["in_t_cam_obj"]), np.asfortranarray(d["in_pts"]),
                               np.asfortranarray(d["in_rays"]), d["in_depth"])
    assert r.is_good and bool(d["is_good"])
    assert np.abs(r.t_cam_obj - d["t_cam_obj"]).max() < 3e-2
    assert np.abs(r.code - d["code"]).max() < 1.5e-2
    assert abs(r.loss - float(d["loss"])) < 0.25 * abs(float(d["loss"])) + 1e-5
    p = np.load(os.path.join(golden_dir, "pose_only_wide.npz"))
    T = opt.estimate_pose_cam_obj(p["in_t_co_se3"].copy(), float(p["in_scale"]), p["in_pts"], p["in_code"])
    np.testing.assert_allclose(T, p["t_cam_obj"], rtol=0, atol=5e-4)


def test_gated_meshed_keyframe_and_submit(golden_dir, cfg_kitti):
    """The stereo keyframe of test_keyframe_mesh with the wide decoder as class 0 (chairs as class 1): the meshed call
    against the unmeshed call and dspgn_mesh_batch, its submitted form bit-identical to the blocking call, and each mesh
    bit-identical to mesh.marching_tetrahedra of MeshExtractor.sdf_grid on the fp32 engine (a grid row's forward pass is
    the same FMA chain in both SIMT instantiations)."""
    from dsp_slam_b200.mesh import marching_tetrahedra
    from dsp_slam_b200.optimizer import MeshExtractor
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5))
    objs, modes, gates = _stereo_keyframe()
    n, dim = len(objs), 16
    got, meshes, words = _check_call(opt.solver, objs, modes, gates, dim)
    assert sum(m is not None for m in meshes) >= 2
    opt.solver.keyframe_submit(objs, modes, gates, voxels_dim=dim)
    sub, sub_meshes = opt.solver.keyframe_wait()
    assert np.array_equal(_bits(sub, n), got)
    opt.solver.keyframe_submit(objs, modes, gates)
    assert np.array_equal(_bits(opt.solver.keyframe_wait(), n), _bits(opt.solver.keyframe(objs, modes, gates), n))
    mx = {c: MeshExtractor(_path(golden_dir, nm), 64, dim, engine="simt") for c, nm in ((0, "wide"), (1, "chairs"))}
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
    """dspgn_keyframe_stop raised by the device at iteration 3 of a wide joint object: it ends STOPPED with the record of
    the same call run for 4 iterations; every other record is bit-identical to the unstopped call."""
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


def test_mixed_width_batch_matches_single_class_runs(golden_dir, cfg_kitti):
    """A keyframe with a 256-wide class (cars) and the 512-wide class: every class runs through the 512 instantiation
    (32-row tiles), so each object's record is bit-identical to the same object run alone in a solver that holds the
    same two classes, and the wide objects also to a solver of the wide class only.  The cars objects are not compared
    with the 256 instantiation: its 64-row tiles sum the normal equations in another order."""
    from dsp_slam_b200 import _lib
    from test_keyframe_batch import _new, _tracked
    cfg = _cfg(cfg_kitti, 5)
    objs = [_new(971), dict(_new(972), class_id=1), _tracked(973), dict(_tracked(974), class_id=1), dict(_new(975), class_id=1)]
    modes = [_lib.MODE_JOINT, _lib.MODE_JOINT, _lib.MODE_POSE, _lib.MODE_POSE, _lib.MODE_JOINT]
    mixed = _opt(golden_dir, cfg, "cars", extra=("wide",), engine="simt")
    got = _bits(mixed.solver.keyframe(objs, modes), len(objs))
    assert (got.view(np.int32)[:, STATUS_WORD] == 0).sum() >= 4
    wide_only = _opt(golden_dir, cfg, "wide", extra=(), engine="simt")
    for i, (o, m) in enumerate(zip(objs, modes)):
        alone = _bits(mixed.solver.keyframe([o], [m]), 1)[0]
        assert np.array_equal(got[i], alone), (i, np.flatnonzero(got[i] != alone)[:8])
        if o["class_id"] == 1:
            single = _bits(wide_only.solver.keyframe([dict(o, class_id=0)], [m]), 1)[0]
            assert np.array_equal(got[i], single), (i, np.flatnonzero(got[i] != single)[:8])
