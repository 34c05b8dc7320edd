"""Teacher-forced parity with the reference: the CUDA path started from the reference's OWN state at every iteration k
(tests/golden/states_*.npz, pose_only_cut.npz) and compared with the reference's iteration k at the single-step
tolerances (tests/test_gpu_parity.py), on both engines.  Whole trajectories separate exponentially between two correct fp32
implementations; one step from a shared state does not, so these tests pin every iteration, including the non-default
hyper-parameters of recon_hyper (D = 24, band half-width 0.02, lr = 0.8, ...) and the pose-only inlier cut.

The numpy oracle, an independent fp32 implementation, is evaluated at the state the library holds after the upload; its
distance from the reference is the reference's own fp32 noise there.  A state whose render row sets (V, m) differ from the
reference's by boundary flips is a slightly different system; _limits gives the bound for each case.
"""
import copy
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import teacher_states as TS  # noqa: E402

pytestmark = pytest.mark.gpu

ENGINES = ["simt", "tc"]
TOL_HB = {"simt": 1e-4, "tc": 3e-4}
TOL_LOSS = {"simt": 1e-4, "tc": 5e-4}


def _opt(engine, dec, cfg, **kw):
    from dsp_slam_b200.optimizer import Optimizer
    from dsp_slam_b200._lib import DspgnError
    try:
        return Optimizer(os.path.join(TS.GOLDEN, f"decoder_{dec}.npz"), cfg, engine=engine, **kw)
    except DspgnError as e:
        if engine == "tc" and "unavailable" in str(e):
            pytest.skip("tensor-core engine not available in this build")
        raise


def _joint_obj(st):
    o = dict(t_cam_obj=TS.upload_pose(st["Toc"]), pts=st["pts"], code=st["z"])
    if "rays" in st:
        o.update(rays=st["rays"], depth=st["depth"])
    return o


def _pose_obj(st):
    return dict(t_cam_obj=TS.upload_pose(st["Toc"], st["scale"]), pts=np.asfortranarray(st["pts"]), code=st["z"],
                scale=st["scale"])


_ORACLE = {}


def _oracle_at(oracle, oracle_decoders, dec, cfg, st, sdf_only=False, pose=False):
    """The oracle's iteration at the state the library holds after the upload (TS.library_state): the reference's own fp32
    noise at that state, one-ulp perturbation included.  Cached per state."""
    key = (st["run"], st["obj"], st["k"], pose)
    if key not in _ORACLE:
        Tl = TS.library_state(st["Toc"], st["scale"] if pose else None)
        if pose:
            _ORACLE[key] = TS.pose_iteration(oracle, oracle_decoders[dec], Tl, st["z"], st["pts"])
        else:
            ocfg = oracle.GNConfig.from_json_dict(cfg)
            _ORACLE[key] = oracle.gn_iteration(oracle_decoders[dec], ocfg, Tl, st["z"], st["pts"], st.get("rays"),
                                               st.get("depth"), sdf_only=sdf_only)
    return _ORACLE[key]


def _limits(base, od, vm_gpu, vm_ref, vm_or):
    """Per-state limits from the engine tolerances `base` and the oracle's own distances `od` from the reference at the same
    state.  vm_* = the render row counts (V, m) of the engine, the reference and the oracle (None without a render term).
    - engine and reference agree on the row sets: the tolerance, or twice the oracle's distance where the oracle agrees too
      and is further away (the reference's fp32 noise at that state);
    - engine and oracle made the same boundary flip: 3x the tolerance or twice the oracle's distance, whichever is larger
      (one band row of ~100 moves H by 5e-2: cfg3_b8 object 1, state 6);
    - any other flip: 3x the first case's limit."""
    same = [max(b, 2 * o) for b, o in zip(base, od)] if vm_or == vm_ref else list(base)
    if vm_gpu == vm_ref:
        return tuple(same)
    if vm_gpu == vm_or:
        return tuple(max(3 * b, 2 * o) for b, o in zip(base, od))
    return tuple(3 * x for x in same)


def _check(rows, n_states, label, known=()):
    """rows: (id, k, flipped, errors, limits, base).  Every state must be within its limits; at most 10 % of a run's states
    may be flipped states beyond the unflipped tolerance `base`.  `known`: (id, k) of states checked by
    test_tensor_core_near_band_edge_states instead."""
    worst = np.max([r[3] for r in rows], axis=0)
    flips = [(r[0], r[1]) for r in rows if r[2]]
    costly = [(r[0], r[1]) for r in rows if r[2] and any(e >= b for e, b in zip(r[3], r[5]))]
    print(f"\n[teacher-forced] {label}: {n_states} states, max errors {np.array2string(np.asarray(worst), precision=2)}, "
          f"flipped states {len(flips)} {flips}, of them beyond the unflipped tolerance {costly}")
    for i, k, fl, e, t, _ in rows:
        if (i, k) not in known:
            assert all(x < y for x, y in zip(e, t)), (label, i, k, e, t)
    assert len(costly) <= 0.1 * n_states, (label, costly)


# Tensor-core states whose reference band holds a sample with sdf within 1e-5 of -th (cfg3_b8 object 1 state 8: 1.2e-5,
# object 5 state 7: 6.8e-6).  There 1 - o = (sdf + th) / 2th is ~5e-4, and de_do = sum T / (1 - o) (loss.py:118-122) turns the
# split-fp16 engine's SDF error (<= 2e-5, test_single_step_system_vs_oracle_and_reference) into a different Jacobian row.
# Perturbing the oracle's SDF values by +-1e-5 at object 5 state 7 moves its H by 8.9e-3: the tensor-core engine is at
# 8.7e-3; the fp32 engine (SDF error 2e-6) stays within 6e-5.  Scaling the split operands is the remedy (out of scope here).
TC_NEAR_BAND_EDGE = {
    ("system", "states_cfg3_b8", 1, 8): "relH 4.1e-4 against 3e-4",
    ("system", "states_cfg3_b8", 5, 7): "relH 8.7e-3, relb 2.8e-3, |ddx| 3.2e-4 against 3e-4, 3e-4, 2e-4",
    ("step", "states_cfg3_b8", 5, 7): "step 3.2e-4 against 2e-4",
}


def _known(kind, engine):
    return {(f"{r}[{o}]", k) for (kd, r, o, k) in TC_NEAR_BAND_EDGE if kd == kind} if engine == "tc" else set()


def _system_row(g, st, cfg, engine, it):
    """One row of (a): the engine's iteration-0 system at state st against the reference's iteration k."""
    k4 = cfg["optimizer"]["joint_optim"]["k4"]
    vm_ref = (st["V"], st["m"]) if "V" in st else None
    vm_gpu = (g["V"], g["m"]) if vm_ref else None
    vm_or = (it["V"], it["m"]) if vm_ref else None
    if vm_gpu != vm_ref:
        assert TS.flip_ok(g["V"] - st["V"], g["m"] - st["m"], st["V"], st["m"]), (st["obj"], st["k"], vm_gpu, vm_ref)
    e = TS.system_errors(g["H"], g["b"], g["dx"], st, k4) + (
        abs(float(g["sdf_loss"]) - st["sdf_loss"]) / st["sdf_loss"],
        abs(float(g["render_loss"]) - st["render_loss"]) / max(st["render_loss"], 1e-30))
    od = TS.system_errors(it["H"], it["b"], it["dx"], st, k4) + (
        abs(float(it["sdf_loss"]) - st["sdf_loss"]) / st["sdf_loss"],
        abs(float(it["render_loss"]) - st["render_loss"]) / max(st["render_loss"], 1e-30))
    base = (TOL_HB[engine], TOL_HB[engine], TS.dx_tol(k4, st, 2e-4), TOL_LOSS[engine], TOL_LOSS[engine])
    return (f"{st['run']}[{st['obj']}]", st["k"], vm_gpu != vm_ref, e, _limits(base, od, vm_gpu, vm_ref, vm_or), base)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("run", [r[0] for r in TS.STATE_RUNS])
def test_system_at_every_reference_state(engine, run, cfg_kitti, cfg_redwood, oracle, oracle_decoders):
    """(a) Every state of a run uploaded as one batch; object i's iteration-0 system (per-iteration schedule) against the
    reference's iteration i: H, b, dx, V, m and the two losses."""
    spec = next(r for r in TS.STATE_RUNS if r[0] == run)
    states, cfg = TS.joint_states(spec, cfg_kitti, cfg_redwood)
    opt = _opt(engine, spec[2], cfg, sdf_only=spec[6])
    opt.solver.upload([_joint_obj(st) for st in states])
    rows = [_system_row(opt.solver.debug_system(i, 0), st, cfg, engine,
                        _oracle_at(oracle, oracle_decoders, spec[2], cfg, st, sdf_only=spec[6]))
            for i, st in enumerate(states)]
    _check(rows, len(states), f"{run} {engine} system (relH, relb, |ddx|, sdf loss, render loss)", _known("system", engine))


@pytest.mark.parametrize("engine", ENGINES)
def test_pose_only_system_at_every_reference_state(engine, cfg_kitti, oracle, oracle_decoders):
    """(a) pose_only_cut.npz: the 6x6 pose-only system at all 8 states (after the cut: the reference's inlier points)
    against the reference, to the single-step tolerance or twice the distance of the oracle evaluated at the state the
    library holds (the SE(3) pose times the scale, re-inverted in fp32), whichever is larger.  That re-inversion moves
    H by 1.5e-4 at state 4 (10 % gross outliers; the oracle at the exact state: 3e-7)."""
    states = TS.pose_states()
    opt = _opt(engine, "cars", cfg_kitti)
    opt.solver.upload([_pose_obj(st) for st in states])
    rows = []
    for i, st in enumerate(states):
        g = opt.solver.debug_system(i, 1)
        it = _oracle_at(oracle, oracle_decoders, "cars", cfg_kitti, st, pose=True)
        relH = lambda H, ref: float(np.abs(H - ref).max() / np.abs(ref).max())  # noqa: E731
        e = (relH(g["H"], st["H"]), float(np.abs(g["dx"] - st["dx"]).max()))
        od = (relH(it["H"], st["H"]), float(np.abs(it["dx"] - st["dx"]).max()))
        base = (TOL_HB[engine], 2e-4)
        rows.append(("pose_only_cut[0]", st["k"], False, e, tuple(max(b, 2 * o) for b, o in zip(base, od)), base))
    _check(rows, len(states), f"pose_only_cut {engine} system (relH, |ddx|)")


def _step_rows(res, states, lr, engine, oracle, oracle_decoders, dec, cfg, pose=False):
    """(b) The step a one-iteration call applied, against the reference's step from the same state; the oracle's own step
    from the library's state gives the reference's fp32 noise there (see _limits)."""
    from oracle import dsp_oracle as O

    def step_err(T, st):
        if pose:
            T = np.asarray(T, np.float64).copy(); T[:3, :3] *= st["scale"]
            ref = O.exp_se3(st["dx"]).astype(np.float64)
        else:
            ref = O.exp_sim3(np.float32(lr) * st["dx"][:7]).astype(np.float64)
        step = np.linalg.inv(np.asarray(T, np.float64)) @ np.linalg.inv(np.asarray(st["Toc"], np.float64))
        return float(np.abs(step - ref).max()) / max(1.0, lr * float(np.abs(st["dx"]).max()))

    rows = []
    for r, st in zip(res, states):
        it = _oracle_at(oracle, oracle_decoders, dec, cfg, st, sdf_only="V" not in st and not pose, pose=pose)
        if pose:
            T_or = np.linalg.inv(O.exp_se3(it["dx"]).astype(np.float64) @ st["Toc"].astype(np.float64))
            T_or[:3, :3] /= st["scale"]
            e, od = [step_err(r, st)], [step_err(T_or, st)]
            base, vm = [2e-4], (None, None, None)
        else:
            assert r.is_good, (st["run"], st["obj"], st["k"])
            T_or = np.linalg.inv(O.exp_sim3(np.float32(lr) * it["dx"][:7]).astype(np.float64) @ st["Toc"].astype(np.float64))
            loss_ref = st["k1"] * st["render_loss"] + st["k2"] * st["sdf_loss"]
            e = [step_err(r.t_cam_obj, st), float(np.abs((np.asarray(r.code) - st["z"]) - np.float32(lr) * st["dx"][7:]).max()),
                 abs(r.loss - loss_ref) / loss_ref]
            od = [step_err(T_or, st), lr * float(np.abs(it["dx"][7:] - st["dx"][7:]).max()),
                  abs(float(st["k1"] * it["render_loss"] + st["k2"] * it["sdf_loss"]) - loss_ref) / loss_ref]
            base = [lr * TS.dx_tol(st["k4"], st, 2e-4), lr * 2e-4, TOL_LOSS[engine]]
            vm = ((r.n_valid, r.n_band), (st["V"], st["m"]), (it["V"], it["m"])) if "V" in st else (None, None, None)
            if vm[0] != vm[1]:
                assert TS.flip_ok(r.n_valid - st["V"], r.n_band - st["m"], st["V"], st["m"]), (st["run"], st["obj"], st["k"])
        rows.append((f"{st['run']}[{st['obj']}]", st["k"], vm[0] != vm[1], tuple(e), _limits(base, od, *vm), tuple(base)))
    return rows


def _one_iteration(cfg):
    cfg = copy.deepcopy(cfg)
    cfg["optimizer"]["joint_optim"]["num_iterations"] = 1
    cfg["optimizer"]["pose_only_optim"] = dict(cfg["optimizer"].get("pose_only_optim", {}), num_iterations=1)
    return cfg


GROUPS = {  # one production call per group: states of these runs, decoder
    "kitti_cars": (["states_cfg1", "states_kitti250", "states_cfg2full"], "cars"),
    "redwood_chairs": (["states_cfg3", "states_cfg3_b8"], "chairs"),
    "hyper": (["states_hyper"], "cars"),
    "sdf_only": (["states_sdf_only"], "cars"),
}


def _group_states(group, cfg_kitti, cfg_redwood):
    names, dec = GROUPS[group]
    states, cfg = [], None
    for run in TS.STATE_RUNS:
        if run[0] in names:
            s, cfg = TS.joint_states(run, cfg_kitti, cfg_redwood)
            j = cfg["optimizer"]["joint_optim"]
            for st in s:
                st.update(k1=j["k1"], k2=j["k2"], k4=j["k4"])
            states += s
    return states, cfg, dec


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("group", list(GROUPS))
def test_one_step_through_the_production_path(engine, group, cfg_kitti, cfg_redwood, oracle, oracle_decoders):
    """(b) reconstruct_batch with one iteration from every state of a group (kitti cars 25 objects, redwood chairs 90, hyper 6,
    sdf_only 10): the applied Sim(3) and code steps, n_valid / n_band and the loss against the reference's iteration k,
    through the persistent kernel and the per-iteration schedule, which must agree bit for bit."""
    states, cfg, dec = _group_states(group, cfg_kitti, cfg_redwood)
    cfg = _one_iteration(cfg)
    lr = cfg["optimizer"]["joint_optim"]["learning_rate"]
    sdf_only = group == "sdf_only"
    objs = [_joint_obj(st) for st in states]
    res = {}
    for sched in ("persistent", "launches"):
        res[sched] = _opt(engine, dec, cfg, sdf_only=sdf_only, schedule=sched).reconstruct_batch(objs)
    for a, b in zip(res["persistent"], res["launches"]):
        assert a.is_good == b.is_good and a.loss == b.loss
        np.testing.assert_array_equal(a.t_cam_obj, b.t_cam_obj)
        np.testing.assert_array_equal(a.code, b.code)
        if not sdf_only:
            assert (a.n_valid, a.n_band) == (b.n_valid, b.n_band)
    _check(_step_rows(res["persistent"], states, lr, engine, oracle, oracle_decoders, dec, cfg), len(states),
           f"{group} {engine} one step (|dstep|, |dcode step|, loss)", _known("step", engine))


@pytest.mark.parametrize("engine", ENGINES)
def test_one_pose_only_step_through_the_production_path(engine, cfg_kitti, oracle, oracle_decoders):
    """(b) estimate_pose_batch with pose_only_optim.num_iterations = 1 from each of the 8 pose_only_cut states: the applied
    SE(3) step against exp_se3(dx_k); both schedules bit-identical."""
    states = TS.pose_states()
    cfg = _one_iteration(cfg_kitti)
    objs = [_pose_obj(st) for st in states]
    Ts = {s: _opt(engine, "cars", cfg, schedule=s).estimate_pose_batch(objs, return_status=True) for s in ("persistent", "launches")}
    assert Ts["persistent"][1] == [0] * 8
    for a, b in zip(Ts["persistent"][0], Ts["launches"][0]):
        np.testing.assert_array_equal(a, b)
    _check(_step_rows(Ts["persistent"][0], states, 1.0, engine, oracle, oracle_decoders, "cars", cfg, pose=True), 8,
           f"pose_only_cut {engine} one step (|dstep|)")


@pytest.mark.parametrize("engine", ENGINES)
def test_mixed_keyframe_one_step_vs_reference(engine, cfg_kitti, cfg_redwood, oracle, oracle_decoders):
    """(c) One Optimizer.keyframe_batch call: the kitti joint states as new objects and the pose_only_cut states k < 5 as
    tracked objects, one iteration each; every object meets the one-step criteria above."""
    states, cfg, _ = _group_states("kitti_cars", cfg_kitti, cfg_redwood)
    pstates = [st for st in TS.pose_states() if st["k"] <= TS.POSE_CUT_AT]
    cfg = _one_iteration(cfg)
    opt = _opt(engine, "cars", cfg)
    res, Ts, status = opt.keyframe_batch([_joint_obj(st) for st in states], [_pose_obj(st) for st in pstates], return_status=True)
    assert status == [0] * len(pstates)
    _check(_step_rows(res, states, 1.0, engine, oracle, oracle_decoders, "cars", cfg), len(states),
           f"keyframe {engine} one step, new objects")
    _check(_step_rows(Ts, pstates, 1.0, engine, oracle, oracle_decoders, "cars", cfg, pose=True), len(pstates),
           f"keyframe {engine} one step, tracked objects")


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("D,n_rays", [(2, 300), (3, 300), (64, 300), (64, 8192)])
def test_depth_sample_count_edges(engine, D, n_rays, cfg_kitti, oracle, oracle_decoders, monkeypatch):
    """(e) num_depth_samples at both ends of the accepted range [2, 64], and D = 64 at the ray limit (8192 rays, the largest
    n_rays x D the kernels accept): the iteration-0 system against the oracle, and a 2-iteration call whose persistent
    schedule is bit-identical to the per-iteration schedule and to the full ray enumeration (DSPGN_COMPACT_RAYS=0).
    D = 2 covers only the failure path: both samples lie on the object's bounding sphere (depth t_z -/+ scale), none is
    inside it, and the oracle and both schedules report the too-few-samples soft failure (status 2).  D = 3 is the
    smallest D with a system to compare."""
    from dsp_slam_b200 import synth
    cfg = copy.deepcopy(cfg_kitti)
    cfg["optimizer"]["num_depth_samples"] = D
    cfg["optimizer"]["joint_optim"]["num_iterations"] = 2
    o = synth.make_object(300 + D, 400, n_rays - n_rays // 5, n_rays // 5)
    obj = dict(t_cam_obj=o["t_cam_obj_init"], pts=o["pts"], rays=o["rays"], depth=o["depth"])
    assert np.asarray(obj["rays"]).shape[0] == n_rays
    opt = _opt(engine, "cars", cfg, schedule="launches")
    it = oracle.gn_iteration(oracle_decoders["cars"], oracle.GNConfig.from_json_dict(cfg), oracle.inv4(o["t_cam_obj_init"]),
                             np.zeros(64, np.float32), np.asarray(o["pts"]), np.asarray(o["rays"]), np.asarray(o["depth"]))
    if D == 2:
        assert it["status"] == oracle.ST_RENDER_FEW
        rs = [_opt(engine, "cars", cfg, schedule=sc).reconstruct_batch([obj])[0] for sc in ("launches", "persistent")]
        assert [(r.is_good, r.status) for r in rs] == [(False, 2)] * 2
        return
    opt.solver.upload([obj])
    g = opt.solver.debug_system(0, 0)
    assert it["status"] == oracle.ST_OK and g["V"] == it["V"] and abs(g["m"] - it["m"]) <= (0 if engine == "simt" else 2)
    eH = float(np.abs(g["H"] - it["H"]).max() / np.abs(it["H"]).max())
    eb = float(np.abs(g["b"] - it["b"]).max() / np.abs(it["b"]).max())
    edx = float(np.abs(g["dx"] - it["dx"]).max())
    print(f"\n[depth-samples] D={D} rays={n_rays} {engine}: V={g['V']} m={g['m']} relH {eH:.1e} relb {eb:.1e} |ddx| {edx:.1e}")
    if g["m"] == it["m"]:
        assert eH < TOL_HB[engine] and eb < TOL_HB[engine] and edx < 2e-4
    runs = [opt.reconstruct_batch([obj])[0], _opt(engine, "cars", cfg, schedule="persistent").reconstruct_batch([obj])[0]]
    monkeypatch.setenv("DSPGN_COMPACT_RAYS", "0")
    runs.append(_opt(engine, "cars", cfg, schedule="persistent").reconstruct_batch([obj])[0])
    assert runs[0].is_good
    for r in runs[1:]:
        assert r.is_good and r.loss == runs[0].loss and (r.n_valid, r.n_band) == (runs[0].n_valid, runs[0].n_band)
        np.testing.assert_array_equal(r.t_cam_obj, runs[0].t_cam_obj)
        np.testing.assert_array_equal(r.code, runs[0].code)


@pytest.mark.parametrize("kind,run,obj,k", [pytest.param(*key, marks=pytest.mark.xfail(strict=True, reason=why))
                                           for key, why in TC_NEAR_BAND_EDGE.items()])
def test_tensor_core_near_band_edge_states(kind, run, obj, k, cfg_kitti, cfg_redwood, oracle, oracle_decoders):
    """The tensor-core states of TC_NEAR_BAND_EDGE, each alone, at the limits every other state meets.  They fail today
    (strict: a pass means the engine's SDF precision improved and the entry must go)."""
    spec = next(r for r in TS.STATE_RUNS if r[0] == run)
    states, cfg = TS.joint_states(spec, cfg_kitti, cfg_redwood)
    st = next(s for s in states if (s["obj"], s["k"]) == (obj, k))
    it = _oracle_at(oracle, oracle_decoders, spec[2], cfg, st)
    if kind == "system":
        opt = _opt("tc", spec[2], cfg)
        opt.solver.upload([_joint_obj(st)])
        row = _system_row(opt.solver.debug_system(0, 0), st, cfg, "tc", it)
    else:
        cfg = _one_iteration(cfg)
        j = cfg["optimizer"]["joint_optim"]
        st.update(k1=j["k1"], k2=j["k2"], k4=j["k4"])
        r = _opt("tc", spec[2], cfg).reconstruct_batch([_joint_obj(st)])
        row = _step_rows(r, [st], j["learning_rate"], "tc", oracle, oracle_decoders, spec[2], cfg)[0]
    print(f"\n[teacher-forced] tc near band edge {kind} {run}[{obj}] k={k}: errors {row[3]} limits {row[4]}")
    assert all(x < y for x, y in zip(row[3], row[4]))
