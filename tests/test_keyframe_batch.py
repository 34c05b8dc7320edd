"""Per-object run modes: a keyframe's tracked objects (estimate_pose_cam_obj) and new objects (reconstruct_object) in
one batched call (dspgn_keyframe_batch / dspgn_run_batch_modes, Optimizer.keyframe_batch).

GPU: every object of a mixed batch is bit-identical to the same object run alone through dspgn_reconstruct_batch or
dspgn_estimate_pose_batch (per-object partial sums are reduced in a fixed tile order that does not depend on the batch),
on both engines and both schedules.  CPU: the new entry points reject misuse before touching CUDA.
"""
import copy
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
NATIVE = os.path.join(ROOT, "tests", "native")

ENGINES = [("simt", "launches"), ("tc", "launches"), ("tc", "persistent")]


def _new(seed, n_pts=200, n_fg=120, n_bg=40, cls="cars"):
    from dsp_slam_b200 import synth
    o = synth.make_object(seed, n_pts, n_fg, n_bg, cls=cls)
    return dict(t_cam_obj=o["t_cam_obj_init"], pts=o["pts"], rays=o["rays"], depth=o["depth"],
                class_id=0 if cls == "cars" else 1)


def _tracked(seed, n_pts=200, cls="cars", outliers=20):
    """A detection associated with an existing map object: SE(3) pose, scale and shape code
    (src/LocalMapping_util.cc:105-109).  It carries rays too: a pose-only object must ignore them."""
    from dsp_slam_b200 import synth
    o = synth.make_object(seed, n_pts, 60, 20, cls=cls)
    pts = np.array(o["pts"])
    rng = np.random.default_rng(seed)
    bad = rng.choice(n_pts, outliers, replace=False)
    pts[bad] += rng.normal(0, 0.6, size=(outliers, 3)).astype(np.float32)
    T = np.array(o["t_cam_obj_init"], dtype=np.float32)
    s = float(np.cbrt(np.linalg.det(T[:3, :3].astype(np.float64))))
    se3 = T.copy()
    se3[:3, :3] /= np.float32(s)
    return dict(t_cam_obj=se3, pts=np.asfortranarray(pts), rays=o["rays"], depth=o["depth"],
                code=(0.8 * o["code_gt"]).astype(np.float32), scale=s, class_id=0 if cls == "cars" else 1)


def _cfg(cfg_kitti, pose_iters):
    cfg = copy.deepcopy(cfg_kitti)
    cfg["optimizer"]["pose_only_optim"]["num_iterations"] = pose_iters
    # pose_only_iterations 7 > num_iterations 6: the pose-only objects keep running after the joint ones finished
    cfg["optimizer"]["joint_optim"]["num_iterations"] = 10 if pose_iters <= 5 else 6
    return cfg


def _opt(golden_dir, cfg, engine, schedule, sdf_only=False):
    from dsp_slam_b200.optimizer import Optimizer
    from dsp_slam_b200._lib import DspgnError
    try:
        return Optimizer(os.path.join(golden_dir, "decoder_cars.npz"), cfg, engine=engine, schedule=schedule,
                         sdf_only=sdf_only, extra_decoders=[os.path.join(golden_dir, "decoder_chairs.npz")])
    except DspgnError as e:
        if engine == "tc" and "unavailable" in str(e):
            pytest.skip("tensor-core engine not available in this build")
        raise


def _bits(out, n):
    from dsp_slam_b200 import _lib
    return np.frombuffer(out, dtype=np.uint32, count=n * _lib.RESULT_FLOATS).reshape(n, _lib.RESULT_FLOATS).copy()


def _alone(solver, objs, modes):
    """Each object run by itself through the single-mode entry point of its mode."""
    rows = []
    for o, m in zip(objs, modes):
        out = solver.estimate_pose([o]) if m else solver.reconstruct([o])
        rows.append(_bits(out, 1)[0])
    return np.stack(rows)


def _assert_same(got, want, what=""):
    for i in range(want.shape[0]):
        assert np.array_equal(got[i], want[i]), (what, i, np.flatnonzero(got[i] != want[i])[:8])


def _mixed_batch():
    objs = [_tracked(301), _new(302), _tracked(303, 150, "chairs"), _new(304, 180, 90, 30, "chairs"),
            _new(305, 250, 250, 200), _tracked(306, 250), _tracked(307, 64, "chairs", 6), _new(308, 65, 64, 10)]
    modes = [1, 0, 1, 0, 0, 1, 1, 0]
    return objs, modes


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
@pytest.mark.parametrize("sdf_only", [False, True])
@pytest.mark.parametrize("pose_iters", [5, 7])
def test_mixed_batch_is_bit_identical_to_objects_run_alone(golden_dir, cfg_kitti, engine, schedule, sdf_only, pose_iters):
    opt = _opt(golden_dir, _cfg(cfg_kitti, pose_iters), engine, schedule, sdf_only)
    objs, modes = _mixed_batch()
    got = _bits(opt.solver.keyframe(objs, modes), len(objs))
    want = _alone(opt.solver, objs, modes)
    _assert_same(got, want, (engine, schedule, sdf_only, pose_iters))
    st = got.view(np.int32)[:, 81]
    assert (st == 0).sum() >= 6, st
    iters = got.view(np.int32)[:, 84]
    for i, m in enumerate(modes):
        if st[i] == 0:
            assert iters[i] == (opt.num_iterations_pose_only if m else opt.num_iterations_joint_optim)
    # the resident-batch form of the same call
    opt.solver.upload(objs)
    opt.solver.run_modes(modes)
    _assert_same(_bits(opt.solver.results_raw(), len(objs)), want, "run_modes")


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_uniform_mode_arrays_equal_run_batch(golden_dir, cfg_kitti, engine, schedule):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 7), engine, schedule)
    objs = [_tracked(311), _tracked(312, 150, "chairs"), _tracked(313, 300)]
    s = opt.solver
    s.upload(objs)
    for m in (0, 1):
        s.run(m)
        ref = _bits(s.results_raw(), len(objs))
        s.run_modes([m] * len(objs))
        _assert_same(_bits(s.results_raw(), len(objs)), ref, m)


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_soft_failures_stay_per_object(golden_dir, cfg_kitti, engine, schedule):
    from dsp_slam_b200 import _lib
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    few = _new(321)
    few["rays"] = np.asfortranarray(np.tile(np.array([[3.0, 3.0, 1.0]], np.float32), (40, 1)))   # rays that miss the object:
    few["depth"] = np.zeros(0, np.float32)                                                       # < 10 samples in the unit sphere
    empty = _new(322)
    empty["pts"] = np.zeros((0, 3), np.float32)                                            # unusable detection
    bad_pose = _tracked(324)
    bad_pose["pts"] = np.zeros((0, 3), np.float32)
    objs = [_tracked(325), few, _tracked(326), empty, _new(327), bad_pose, _tracked(328)]
    modes = [1, 0, 1, 0, 0, 1, 1]
    got = _bits(opt.solver.keyframe(objs, modes), len(objs))
    _assert_same(got, _alone(opt.solver, objs, modes))
    st = got.view(np.int32)[:, 81]
    assert st[1] == _lib.ST_RENDER_FEW and st[3] == _lib.ST_BAD_INPUT and st[5] == _lib.ST_BAD_INPUT, st
    assert all(st[i] == _lib.ST_OK for i in (0, 2, 4, 6)), st


@pytest.mark.gpu
def test_more_than_one_resident_batch_with_alternating_modes(golden_dir, cfg_kitti):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), None, None)
    n = 1030
    objs = [(_tracked(1000 + i, 64, outliers=4) if i % 2 else _new(1000 + i, 64, 24, 8)) for i in range(n)]
    modes = [i % 2 for i in range(n)]
    got = _bits(opt.solver.keyframe(objs, modes), n)
    joint = [o for o, m in zip(objs, modes) if m == 0]
    pose = [o for o, m in zip(objs, modes) if m == 1]
    want_j = _bits(opt.solver.reconstruct(joint), len(joint))
    want_p = _bits(opt.solver.estimate_pose(pose), len(pose))
    _assert_same(got[0::2], want_j, "joint")
    _assert_same(got[1::2], want_p, "pose")
    # the objects on both sides of the resident-batch boundary (1024) each against a run alone
    idx = [1022, 1023, 1024, 1025]
    _assert_same(got[idx], _alone(opt.solver, [objs[i] for i in idx], [modes[i] for i in idx]), "boundary")


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_counters_sum_per_mode(golden_dir, cfg_kitti, engine, schedule):
    cfg = _cfg(cfg_kitti, 7)
    opt = _opt(golden_dir, cfg, engine, schedule, sdf_only=True)
    objs, modes = _mixed_batch()
    it_j, it_p = opt.num_iterations_joint_optim, opt.num_iterations_pose_only
    s = opt.solver
    s.keyframe(objs, modes)
    c = s.counters()
    want = sum(o["pts"].shape[0] * (it_p if m else it_j) for o, m in zip(objs, modes))
    assert c["rows_fwd_bwd"] == want, (c, want)
    if schedule == "persistent":
        s.reconstruct([o for o, m in zip(objs, modes) if m == 0])
        assert c["kernel_launches"] == s.counters()["kernel_launches"]
    # with the render term too: the SDF rows still sum per mode (band rows come on top)
    opt2 = _opt(golden_dir, cfg, engine, schedule)
    opt2.solver.keyframe(objs, modes)
    c2 = opt2.solver.counters()
    assert c2["rows_fwd_bwd"] >= want
    if schedule == "persistent":
        opt2.solver.reconstruct([o for o, m in zip(objs, modes) if m == 0])
        assert c2["kernel_launches"] == opt2.solver.counters()["kernel_launches"]
    else:
        smp = sum(o["rays"].shape[0] * opt2.num_depth_samples * it_j for o, m in zip(objs, modes) if m == 0)
        assert c2["rows_fwd_bwd"] == want and c2["rows_fwd_only"] == smp


@pytest.mark.gpu
def test_misuse_returns_e_arg(golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), None, None)
    objs, modes = _mixed_batch()
    for bad_modes in ([2] + modes[1:], modes[:-1] + [-1]):
        with pytest.raises(_lib.DspgnError) as e:
            opt.solver.keyframe(objs, bad_modes)
        assert e.value.code == _lib.E_ARG
    no_code = [dict(o, code=None) if m else o for o, m in zip(objs, modes)]
    with pytest.raises(_lib.DspgnError) as e:
        opt.solver.keyframe(no_code, modes)
    assert e.value.code == _lib.E_ARG
    no_scale = [dict(o, scale=0.0) if m else o for o, m in zip(objs, modes)]
    with pytest.raises(_lib.DspgnError) as e:
        opt.solver.keyframe(no_scale, modes)
    assert e.value.code == _lib.E_ARG
    opt.solver.upload(no_code)
    with pytest.raises(_lib.DspgnError) as e:
        opt.solver.run_modes(modes)
    assert e.value.code == _lib.E_ARG
    with pytest.raises(_lib.DspgnError) as e:
        opt.solver.run_modes([2] * len(objs))
    assert e.value.code == _lib.E_ARG
    # the solver stays usable
    got = _bits(opt.solver.keyframe(objs, modes), len(objs))
    _assert_same(got, _alone(opt.solver, objs, modes))


@pytest.mark.gpu
def test_optimizer_keyframe_batch_equals_the_two_calls(golden_dir, cfg_kitti):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), None, None)
    new = [_new(331), _new(332, 180, 90, 30, "chairs"), _new(333)]
    new[2]["pts"] = np.zeros((0, 3), np.float32)                       # a failed reconstruction
    tracked = [_tracked(334), _tracked(335, 150, "chairs"), _tracked(336)]
    tracked[2]["pts"] = np.zeros((0, 3), np.float32)                   # a failed pose: the input pose comes back
    res, Ts, st = opt.keyframe_batch(new, tracked, return_status=True)
    ref_res = opt.reconstruct_batch(new)
    ref_Ts, ref_st = opt.estimate_pose_batch(tracked, return_status=True)
    assert st == ref_st and st[2] != 0
    for a, b in zip(Ts, ref_Ts):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(Ts[2], tracked[2]["t_cam_obj"])
    assert len(res) == len(ref_res)
    for a, b in zip(res, ref_res):
        assert a.is_good == b.is_good and np.float32(a.loss) == np.float32(b.loss)
        if a.is_good:
            np.testing.assert_array_equal(a.t_cam_obj, b.t_cam_obj)
            np.testing.assert_array_equal(a.code, b.code)
    assert not res[2].is_good
    r2, T2 = opt.keyframe_batch([], tracked)
    assert r2 == [] and all(np.array_equal(a, b) for a, b in zip(T2, Ts))
    r3, T3 = opt.keyframe_batch(new, [])
    assert T3 == [] and all(a.is_good == b.is_good for a, b in zip(r3, res))


def _build_caller(tmp):
    exe = os.path.join(tmp, "keyframe_caller")
    libd = os.path.join(ROOT, "dsp_slam_b200")
    subprocess.check_call(["gcc", "-O1", "-std=c11", f"-I{os.path.join(ROOT, 'include')}",
                           os.path.join(NATIVE, "keyframe_caller.c"), "-o", exe, f"-L{libd}", "-ldspgn",
                           f"-Wl,-rpath,{libd}"])
    return exe


def test_keyframe_caller_compiles_and_links(tmp_path):
    exe = _build_caller(str(tmp_path))
    assert subprocess.run([exe]).returncode == 2


@pytest.mark.gpu
def test_plain_c_keyframe_caller_matches_python(tmp_path, golden_dir, cfg_kitti):
    from dsp_slam_b200.decoder import DecoderWeights
    from dsp_slam_b200.optimizer import Optimizer
    exe = _build_caller(str(tmp_path))
    d = np.load(os.path.join(golden_dir, "recon_kitti250.npz"))
    dec = os.path.join(golden_dir, "decoder_cars.npz")
    w = DecoderWeights.from_npz(dec)
    wp, inp, outp = str(tmp_path / "w.bin"), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(wp, "wb") as f:
        f.write(struct.pack("<3i", len(w.W), w.latent_size, w.latent_in_layer))
        for W, b in zip(w.W, w.b):
            f.write(struct.pack("<2i", *W.shape)); f.write(W.tobytes()); f.write(b.tobytes())
    T = np.array(d["in_t_cam_obj"], dtype=np.float32)
    scale = np.float32(np.cbrt(np.linalg.det(T[:3, :3].astype(np.float64))))
    code = (0.5 * d["gt_code"]).astype(np.float32)
    P = np.asfortranarray(d["in_pts"], dtype=np.float32)
    R = np.asfortranarray(d["in_rays"], dtype=np.float32)
    dep = np.ascontiguousarray(d["in_depth"], dtype=np.float32)
    with open(inp, "wb") as f:
        f.write(struct.pack("<3i", P.shape[0], R.shape[0], dep.shape[0]))
        for a in (np.asfortranarray(T), P, R):
            f.write(a.tobytes(order="F"))
        f.write(dep.tobytes()); f.write(struct.pack("<f", scale)); f.write(code.tobytes())
    r = subprocess.run([exe, wp, inp, outp], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "kernel launches" in r.stdout
    from dsp_slam_b200 import _lib
    got = np.frombuffer(open(outp, "rb").read(), np.uint32).reshape(3, _lib.RESULT_FLOATS)
    opt = Optimizer(dec, cfg_kitti)
    se3 = T.copy(); se3[:3, :3] /= scale
    Tf = se3.copy(); Tf[:, 0] *= -1; Tf[:, 2] *= -1
    objs = [dict(t_cam_obj=se3, pts=P, code=code, scale=float(scale)),
            dict(t_cam_obj=T, pts=P, rays=R, depth=dep),
            dict(t_cam_obj=Tf, pts=P, code=code, scale=float(scale))]
    want = _bits(opt.solver.keyframe(objs, [1, 0, 1]), 3)
    _assert_same(got, want, "c caller")
    assert got.view(np.int32)[1, 81] == 0 and got.view(np.int32)[0, 81] == 0


def test_c_abi_rejects_per_object_mode_misuse_before_touching_cuda():
    """dspgn_run_batch_modes / dspgn_keyframe_batch return DSPGN_E_ARG (-1) for misuse without needing a GPU."""
    from dsp_slam_b200 import _lib
    lib = _lib.load()
    T = np.eye(4, dtype=np.float32)
    P = np.zeros((8, 3), np.float32)
    FP = C.POINTER(C.c_float)
    ins = (_lib.ObjectIn * 2)()
    for o in ins:
        o.t_cam_obj = T.ctypes.data_as(FP); o.t_rs = 4; o.t_cs = 1
        o.pts = P.ctypes.data_as(FP); o.n_pts = 8; o.pts_rs = 3; o.pts_cs = 1
        o.scale = 1.0
    outs = (_lib.ObjectOut * 2)()
    modes = (C.c_int32 * 2)(0, 1)
    # a handle that must never be dereferenced: every call below fails on its arguments first
    fake = C.create_string_buffer(64)
    h = C.cast(fake, C.c_void_p)
    assert lib.dspgn_run_batch_modes(None, modes) == -1
    assert lib.dspgn_run_batch_modes(h, None) == -1
    assert lib.dspgn_keyframe_batch(None, 2, ins, modes, outs) == -1
    assert lib.dspgn_keyframe_batch(h, 0, ins, modes, outs) == -1
    assert lib.dspgn_keyframe_batch(h, -3, ins, modes, outs) == -1
    assert lib.dspgn_keyframe_batch(h, 2, ins, None, outs) == -1
    assert lib.dspgn_keyframe_batch(h, 2, ins, (C.c_int32 * 2)(0, 2), outs) == -1
    assert b"mode" in lib.dspgn_last_error()
    assert lib.dspgn_keyframe_batch(h, 2, ins, modes, outs) == -1              # pose-only object 1 has no code
    assert b"code" in lib.dspgn_last_error()
    code = np.zeros(64, np.float32)
    ins[1].code = code.ctypes.data_as(FP); ins[1].scale = 0.0
    assert lib.dspgn_keyframe_batch(h, 2, ins, modes, outs) == -1              # ... and now scale <= 0
    assert b"scale" in lib.dspgn_last_error()


def test_ctypes_argtypes_of_the_per_object_entry_points_match_the_header():
    import re
    from dsp_slam_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "dspgn.h")).read()
    sym = {n: (r, a) for n, r, a in _lib.SYMBOLS}
    want = {"dspgn_run_batch_modes": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
            "dspgn_keyframe_batch": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(_lib.ObjectIn), C.POINTER(C.c_int32),
                                               C.POINTER(_lib.ObjectOut)])}
    for name, (res, args) in want.items():
        assert sym[name] == (res, args), name
        decl = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", hdr).group(1)
        ctypes_of = {"DspgnSolver*": C.c_void_p, "int": C.c_int, "const DspgnObjectIn*": C.POINTER(_lib.ObjectIn),
                     "const int32_t*": C.POINTER(C.c_int32), "DspgnObjectOut*": C.POINTER(_lib.ObjectOut)}
        params = [" ".join(p.split()[:-1]) for p in decl.split(",")]
        assert [ctypes_of[p] for p in params] == args, (name, params)
    assert (_lib.MODE_JOINT, _lib.MODE_POSE) == (0, 1)
    assert re.search(r"#define DSPGN_MODE_JOINT 0\b", hdr) and re.search(r"#define DSPGN_MODE_POSE\s+1\b", hdr)
