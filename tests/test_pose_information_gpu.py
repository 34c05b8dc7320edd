"""dspgn_pose_information on the GPU (BatchSolver / Optimizer.pose_information).

  teacher-forced   the library started at the reference's state before its last iteration, one iteration run, and its
                   Lambda compared with the fp64 restatement (tests/pose_info_model.py) of the reference's last H, on the
                   fp32, tensor-core and wide tensor-core engines and both schedules.  The bound is the single-step H
                   tolerance of tests/test_teacher_forced.py carried through the Schur complement to first order, plus
                   the difference of the two records' scales; it is printed with the eliminated block's condition number.
  bit identity     between the two schedules of an engine, and between two runs.
  production       every call that returns records gives each record the Lambda of the call that makes that record alone
                   (the records are bit-identical by the calls' contracts, so the systems are too): mixed, gated, meshed,
                   submitted, stopped, mono pair, more than 1024 objects, rejected at upload.
  arguments        DSPGN_E_ARG / DSPGN_E_BUSY.
"""
import copy
import ctypes as C
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import pose_info_model as PI  # noqa: E402
import teacher_states as TS  # noqa: E402
import wide_fixtures as WF  # noqa: E402
from test_keyframe_batch import NATIVE, ROOT, _cfg, _new, _opt, _tracked  # noqa: E402
from test_keyframe_gate import _gate_in, _gated, _joint_of  # noqa: E402

pytestmark = pytest.mark.gpu

TOL_H = {"simt": 1e-4, "tc": 3e-4, "tc_wide": 3e-4}     # single-step |dH| / max|H| of test_teacher_forced.py
SCHEDULES = ("persistent", "launches")
_WIDE = {}


@pytest.fixture(scope="module", autouse=True)
def _wide_files(tmp_path_factory):
    _WIDE["wide"] = WF.write("wide", str(tmp_path_factory.mktemp("wide_decoders")))


def _optimizer(golden_dir, dec, cfg, engine, schedule):
    from dsp_slam_b200.optimizer import Optimizer
    path = _WIDE["wide"] if dec == "wide" else os.path.join(golden_dir, f"decoder_{dec}.npz")
    return Optimizer(path, cfg, engine=engine, schedule=schedule)


def _info(solver):
    info, st = solver.pose_information()
    return np.array(info), np.array(st)


# ---- teacher-forced at the last state --------------------------------------------------------------------------------
RUNS = {  # states run spec (teacher_states.STATE_RUNS layout), engines
    "cfg1": (("states_cfg1", "recon_cfg1", "cars", "kitti", 5, False, False), ("simt", "tc")),
    "kitti250": (("states_kitti250", "recon_kitti250", "cars", "kitti", 10, False, False), ("simt", "tc")),
    "cfg3_b8": (("states_cfg3_b8", "recon_cfg3_b8", "chairs", "redwood", 10, True, False), ("simt", "tc")),
    "hyper": (("states_hyper", "recon_hyper", "cars", "hyper", 6, False, False), ("simt", "tc")),
    "wide": (("states_wide", "recon_wide", "wide", "kitti", 10, False, False), ("tc_wide",)),
}
CASES = [(r, e, s) for r, (_, engs) in RUNS.items() for e in engs for s in SCHEDULES]


def _bound(Hu, st, tol, k4, s_ref, s_lib, L_ref):
    """Elementwise bound on |Lambda_lib - Lambda_ref|: |dH| <= tol max|H| (+ the rotation prior's rounding allowance on
    its rows, TS.rot_allowance) through the Schur complement to first order, dS_ij <= eps_i eps_j-weighted
    (1 + |X_:i|_1)(1 + |X_:j|_1) with X = C^-1 B^T, mapped by |f_a f_b|; plus |Lambda_ab| times the relative scale
    difference of the two records for each 1/s factor.  Returns (bound, condition number of C)."""
    eps = tol * np.abs(Hu).max()
    rot = TS.rot_allowance(k4, st["Toc"])
    B, Cm = Hu[:6, 6:], Hu[6:, 6:]
    X = np.linalg.solve(Cm, B.T) if Cm.shape[0] else np.zeros((0, 6))
    a = 1.0 + np.abs(X).sum(axis=0)
    dS = eps * np.outer(a, a)
    dS[3:6, :] += rot
    dS[:, 3:6] += rot
    perm = [3, 4, 5, 0, 1, 2]
    f = np.array([1, 1, 1, 1 / s_ref, 1 / s_ref, 1 / s_ref])
    nf = np.array([0, 0, 0, 1, 1, 1])
    bound = np.outer(f, f) * dS[np.ix_(perm, perm)] + np.abs(L_ref) * np.add.outer(nf, nf) * abs(s_lib / s_ref - 1.0) * 1.01
    return bound, (np.linalg.cond(Cm) if Cm.shape[0] else 1.0)


@pytest.mark.parametrize("run,engine,schedule", CASES)
def test_teacher_forced_at_the_last_state(run, engine, schedule, golden_dir, cfg_kitti, cfg_redwood):
    spec, _ = RUNS[run]
    states, cfg = TS.joint_states(spec, cfg_kitti, cfg_redwood)
    last = [st for st in states if st["k"] == spec[4] - 1]
    cfg = copy.deepcopy(cfg)
    cfg["optimizer"]["joint_optim"]["num_iterations"] = 1
    j = cfg["optimizer"]["joint_optim"]
    opt = _optimizer(golden_dir, spec[2], cfg, engine, schedule)
    objs = [dict(t_cam_obj=TS.upload_pose(st["Toc"]), pts=st["pts"], code=st["z"], rays=st["rays"], depth=st["depth"])
            for st in last]
    res = opt.reconstruct_batch(objs)
    info, status = opt.pose_information()
    assert info.shape == (len(last), 6, 6) and info.dtype == np.float64
    for i, (st, r) in enumerate(zip(last, res)):
        assert r.is_good and status[i] == 0, (run, i)
        np.testing.assert_array_equal(info[i], info[i].T)
        Hu = PI.undamped(st["H"], j["scale_damping"])
        s_ref = PI.record_scale(np.linalg.inv(np.asarray(st["Toc_next"], np.float64)))
        s_lib = PI.record_scale(r.t_cam_obj)
        L_ref = PI.information(Hu, s_ref)
        bound, cond = _bound(Hu, st, TOL_H[engine], j["k4"], s_ref, s_lib, L_ref)
        flipped = (r.n_valid, r.n_band) != (st["V"], st["m"])
        if flipped:                                   # a boundary flip of the render rows: test_teacher_forced's 3x
            assert TS.flip_ok(r.n_valid - st["V"], r.n_band - st["m"], st["V"], st["m"]), (run, i)
            bound = 3 * bound
        ratio = float((np.abs(info[i] - L_ref) / bound).max())
        print(f"\n[pose information] {run}[{i}] {engine} {schedule}: cond(C) {cond:.1e}, max |dLambda| / bound {ratio:.1e}"
              f"{' (flipped)' if flipped else ''}")
        assert ratio < 1.0, (run, i, ratio)
        assert np.all(np.linalg.eigvalsh(info[i]) > 0)


@pytest.mark.parametrize("engine", ["simt", "tc"])
@pytest.mark.parametrize("schedule", SCHEDULES)
@pytest.mark.parametrize("call", ["estimate_pose", "keyframe"])
def test_pose_only_teacher_forced_at_the_last_state(engine, schedule, call, golden_dir, cfg_kitti, oracle, oracle_decoders):
    """pose_only_cut.npz at k = 7 (after the inlier cut): one pose-only iteration from the reference's state, through
    estimate_pose_batch and as the tracked object of a keyframe call, against the restatement of the reference's 6x6 H
    with its 1e-2 I removed, at the call's scale argument.  The H tolerance is test_teacher_forced's pose-only one: the
    single-step tolerance, or twice the distance of the oracle evaluated at the state the library holds."""
    from dsp_slam_b200 import _lib
    st = [x for x in TS.pose_states() if x["k"] == TS.POSE_CUT_ITERS - 1][0]
    cfg = copy.deepcopy(cfg_kitti)
    cfg["optimizer"]["pose_only_optim"] = dict(cfg["optimizer"].get("pose_only_optim", {}), num_iterations=1)
    opt = _optimizer(golden_dir, "cars", cfg, engine, schedule)
    obj = dict(t_cam_obj=TS.upload_pose(st["Toc"], st["scale"]), pts=np.asfortranarray(st["pts"]), code=st["z"],
               scale=st["scale"])
    if call == "estimate_pose":
        _, status = opt.estimate_pose_batch([obj], return_status=True)
    else:
        _, _, status = opt.keyframe_batch([], [obj], return_status=True)
    assert status == [0]
    info, ist = opt.pose_information()
    assert ist.tolist() == [_lib.INFO_OK]
    np.testing.assert_array_equal(info[0], info[0].T)
    it = TS.pose_iteration(oracle, oracle_decoders["cars"], TS.library_state(st["Toc"], st["scale"]), st["z"], st["pts"])
    od = float(np.abs(it["H"] - st["H"]).max() / np.abs(st["H"]).max())
    tol = max(TOL_H[engine], 2 * od)
    Hu = PI.undamped(st["H"])
    L_ref = PI.information(Hu, st["scale"])
    bound, _ = _bound(Hu, st, tol, 0.0, st["scale"], st["scale"], L_ref)
    ratio = float((np.abs(info[0] - L_ref) / bound).max())
    print(f"\n[pose information] pose_only_cut k=7 {engine} {schedule} {call}: s {st['scale']:.4f}, H tolerance {tol:.1e}, "
          f"max |dLambda| / bound {ratio:.1e}")
    assert ratio < 1.0, ratio
    # the scale enters as 1/s and 1/s^2: a map at any other s would be far outside the bound
    assert float((np.abs(info[0] - PI.information(Hu, 1.0)) / bound).max()) > 10.0


# ---- bit identity ------------------------------------------------------------------------------------------------------
def _keyframe_objs():
    objs = [_new(3101), _tracked(3102), _gated(3103, dict()), _gated(3104, dict(dx=2.0)), _new(3105, 150, 80, 30)]
    return objs, [0, 1, 1, 1, 0]


@pytest.mark.parametrize("engine", ["simt", "tc", "tc_wide"])
def test_schedules_and_repeats_are_bit_identical(engine, golden_dir, cfg_kitti):
    objs, modes = _keyframe_objs()
    if engine == "tc_wide":
        objs = [dict(o, class_id=0) for o in objs]
    gates = [_gate_in(o) if m else None for o, m in zip(objs, modes)]
    got = {}
    for sch in SCHEDULES:
        opt = _optimizer(golden_dir, "wide" if engine == "tc_wide" else "cars", _cfg(cfg_kitti, 5), engine, sch)
        runs = []
        for _ in range(2):
            out = opt.solver.keyframe(objs, modes, gates)
            runs.append(_info(opt.solver))
        # a linearisation exactly where the record's final update came from a completed solve
        want = [0 if out[i].status in (0, 6) and out[i].iters_done > 0 else 1 for i in range(len(objs))]
        assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])
        got[sch] = runs[0]
        opt.solver.close()
    assert np.array_equal(got["persistent"][0], got["launches"][0])
    assert np.array_equal(got["persistent"][1], got["launches"][1])
    assert got["persistent"][1].tolist() == want and 0 in want


# ---- production paths -----------------------------------------------------------------------------------------------
def _alone(solver, call):
    call(solver)
    return _info(solver)


def _eq(a, b, what):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), what


@pytest.mark.parametrize("schedule", SCHEDULES)
def test_keyframe_calls(schedule, golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), "tc", schedule)
    S = opt.solver
    objs, modes = _keyframe_objs()
    gates = [_gate_in(o) if m else None for o, m in zip(objs, modes)]
    # mixed stereo keyframe: each object's Lambda is its single-mode call's
    S.keyframe(objs, modes)
    mixed = _info(S)
    new = [i for i, m in enumerate(modes) if m == 0]
    trk = [i for i, m in enumerate(modes) if m == 1]
    rn = _alone(S, lambda s: s.reconstruct([objs[i] for i in new]))
    rp = _alone(S, lambda s: s.estimate_pose([objs[i] for i in trk]))
    _eq((mixed[0][new], mixed[1][new]), rn, "mixed: new objects")
    _eq((mixed[0][trk], mixed[1][trk]), rp, "mixed: tracked objects")
    # gated: a kept detection has its pose-only Lambda, a rejected one its joint run's
    out = S.keyframe(objs, modes, gates)
    gated = _info(S)
    gw = [out[i].gate for i in range(len(objs))]
    assert gw[2] == _lib.GATE_KEPT and gw[3] == _lib.GATE_REJECTED, gw
    _eq((gated[0][[0, 1, 2, 4]], gated[1][[0, 1, 2, 4]]),
        (mixed[0][[0, 1, 2, 4]], mixed[1][[0, 1, 2, 4]]), "gated: kept and ungated objects")
    rj = _alone(S, lambda s: s.reconstruct([_joint_of(objs[3])]))
    _eq((gated[0][[3]], gated[1][[3]]), rj, "gated: the rejected detection")
    assert not np.array_equal(gated[0][3], mixed[0][3])
    # meshed: the gated call's
    S.keyframe(objs, modes, gates, voxels_dim=16)
    _eq(_info(S), gated, "meshed")
    # submitted: the blocking call's; BUSY while in flight
    S.keyframe_submit(objs, modes, gates, voxels_dim=16)
    with pytest.raises(_lib.DspgnError) as e:
        S.pose_information()
    assert e.value.code == _lib.E_BUSY
    S.keyframe_wait()
    _eq(_info(S), gated, "submit / wait")
    # mono pair: each hypothesis has its own record's Lambda
    a = _new(3201)
    b = dict(a, t_cam_obj=np.array(a["t_cam_obj"]) @ np.diag([-1, 1, -1, 1]).astype(np.float32))
    S.keyframe([a, b], [0, 0], voxels_dim=16, pairs=[1, 0])
    pair = _info(S)
    _eq(pair, _alone(S, lambda s: s.reconstruct([a, b])), "mono pair")
    assert not np.array_equal(pair[0][0], pair[0][1])


def test_stopped_objects(golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib
    cfg = _cfg(cfg_kitti, 5)
    opt = _opt(golden_dir, cfg, "tc", "persistent")
    S = opt.solver
    objs = [_new(3301), _new(3302)]
    S.debug_stop_at(1, 2)
    out = S.reconstruct(objs)
    assert out[1].status == _lib.ST_STOPPED and out[1].iters_done == 3
    got = _info(S)
    c3 = copy.deepcopy(cfg)
    c3["optimizer"]["joint_optim"]["num_iterations"] = 3
    want = _alone(_opt(golden_dir, c3, "tc", "persistent").solver, lambda s: s.reconstruct([objs[1]]))
    _eq((got[0][[1]], got[1][[1]]), want, "stopped after iteration 3: the 3-iteration call's Lambda")
    assert got[1][0] == _lib.INFO_OK
    # a rejected detection whose joint run the stop keeps from starting: no linearisation
    g = [_gated(3303, dict(dx=2.0))]
    S.debug_stop_at(0, 4)
    out = S.keyframe(g, [1], [_gate_in(g[0])])
    assert out[0].gate == _lib.GATE_REJECTED and out[0].status == _lib.ST_STOPPED and out[0].iters_done == 0
    info, st = _info(S)
    assert st[0] == _lib.INFO_NONE and not info[0].any()


def test_more_than_one_resident_batch_and_bad_input(golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib
    S = _opt(golden_dir, _cfg(cfg_kitti, 5), "tc", "persistent").solver
    n = 1030
    objs = [_tracked(4000 + i, 48, outliers=2) for i in range(n)]
    objs[7] = dict(objs[7], pts=np.zeros((0, 3), np.float32))        # rejected at upload
    S.estimate_pose(objs)
    info, st = _info(S)
    assert info.shape == (n, 6, 6) and st[7] == _lib.INFO_NONE and not info[7].any()
    assert (np.delete(st, 7) == _lib.INFO_OK).all()
    for idx in ([1020, 1025, 1029], [3, 8]):
        _eq((info[idx], st[idx]), _alone(S, lambda s: s.estimate_pose([objs[i] for i in idx])), f"objects {idx}")
    # the keyframe walk across chunks, gated objects (two slots each) included
    k = [_gated(5000 + i, dict(dx=2.0) if i % 2 else dict(), n_pts=48) if i % 3 == 0 else _tracked(5000 + i, 48, outliers=2)
         for i in range(900)]
    m = [1] * len(k)
    gates = [_gate_in(o) for o in k]
    S.keyframe(k, m, gates)
    kinfo = _info(S)
    tail = list(range(890, 900))
    S.keyframe([k[i] for i in tail], [1] * len(tail), [gates[i] for i in tail])
    _eq((kinfo[0][tail], kinfo[1][tail]), _info(S), "the last chunk of a gated keyframe call")


def test_argument_errors(golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), "tc", "persistent")
    S = opt.solver
    lib = _lib.load()
    buf = np.zeros((4, 36)); st = np.zeros(4, np.int32)
    dp, ip = buf.ctypes.data_as(C.POINTER(C.c_double)), st.ctypes.data_as(C.POINTER(C.c_int32))
    assert lib.dspgn_pose_information(S.handle, 1, dp, ip) == _lib.E_ARG                 # no call yet
    S.reconstruct([_new(3401), _new(3402)])
    assert lib.dspgn_pose_information(S.handle, 1, dp, ip) == _lib.E_ARG                 # n != the call's count
    assert lib.dspgn_pose_information(S.handle, 2, None, ip) == _lib.E_ARG
    assert lib.dspgn_pose_information(S.handle, 2, dp, ip) == 0
    before = S.counters()
    assert lib.dspgn_pose_information(S.handle, 2, dp, ip) == 0
    assert S.counters() == before                                                          # not a run
    S.mesh(np.zeros((1, 64), np.float32), 8)
    assert lib.dspgn_pose_information(S.handle, 2, dp, ip) == _lib.E_ARG                 # a call without records
    S.reconstruct([_new(3401), _new(3402)])
    S.decode_sdf(np.zeros(64, np.float32), np.zeros((4, 3), np.float32))
    assert lib.dspgn_pose_information(S.handle, 2, dp, ip) == _lib.E_ARG
    S.upload([_new(3401)]); S.run(0); S.results_raw()
    assert lib.dspgn_pose_information(S.handle, 1, dp, ip) == _lib.E_ARG                 # the split-phase run


def test_plain_c_caller_matches_python(tmp_path, golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib
    from dsp_slam_b200.decoder import DecoderWeights
    exe = str(tmp_path / "pose_info_caller")
    libd = os.path.join(ROOT, "dsp_slam_b200")
    subprocess.check_call(["gcc", "-O1", "-std=c11", f"-I{os.path.join(ROOT, 'include')}",
                           os.path.join(NATIVE, "pose_info_caller.c"), "-o", exe, f"-L{libd}", "-ldspgn",
                           f"-Wl,-rpath,{libd}", "-lm"])
    w = DecoderWeights.from_npz(os.path.join(golden_dir, "decoder_cars.npz"))
    wp, inp, outp = str(tmp_path / "w.bin"), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(wp, "wb") as f:
        f.write(struct.pack("<3i", len(w.W), w.latent_size, w.latent_in_layer))
        for W, b in zip(w.W, w.b):
            f.write(struct.pack("<2i", *W.shape)); f.write(W.tobytes()); f.write(b.tobytes())
    dets = [_gated(3501, dict()), _gated(3502, dict(dx=2.0)), _gated(3503, dict(angle=2.0))]
    with open(inp, "wb") as f:
        f.write(struct.pack("<i", len(dets)))
        for d in dets:
            P, R, dep = np.asfortranarray(d["pts"]), np.asfortranarray(d["rays"]), np.ascontiguousarray(d["depth"])
            f.write(struct.pack("<3i", P.shape[0], R.shape[0], dep.shape[0]))
            for a in (d["t_cam_obj"], d["t_cam_obj_map"], d["t_cam_obj_sim3"], P, R):
                f.write(np.asfortranarray(a, dtype=np.float32).tobytes(order="F"))
            f.write(dep.tobytes()); f.write(struct.pack("<f", d["scale"])); f.write(np.ascontiguousarray(d["code"]).tobytes())
    r = subprocess.run([exe, wp, inp, outp], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    raw = open(outp, "rb").read()
    n, RB = len(dets), 4 * _lib.RESULT_FLOATS
    info_c = np.frombuffer(raw[n * RB:n * RB + 288 * n], np.float64).reshape(n, 6, 6)
    st_c = np.frombuffer(raw[n * RB + 288 * n:], np.int32)
    cfg = copy.deepcopy(cfg_kitti)
    cfg["optimizer"]["pose_only_optim"]["num_iterations"] = 5
    cfg["optimizer"]["joint_optim"]["num_iterations"] = 10
    opt = _opt(golden_dir, cfg, None, None)
    opt.solver.keyframe(dets, [1] * n, [_gate_in(d) for d in dets])
    info_p, st_p = opt.pose_information()
    assert np.array_equal(info_c, info_p) and np.array_equal(st_c, st_p)
    assert (st_p == _lib.INFO_OK).any()
