"""Gated keyframe calls (dspgn_keyframe_batch_gated, BatchSolver.keyframe(..., gates), Optimizer.keyframe_batch with
t_cam_obj_map / t_cam_obj_sim3): GetNewObservations' map-consistency check on the device and the joint run of every
rejected detection in the same call.

GPU, both engines and both schedules: every gate word equals the numpy check (oracle/gate_check.py) applied to the
library's own pose-only record; a rejected record is bit-identical to dspgn_reconstruct_batch of the detection alone; a
kept or ungated record, and every new object, is bit-identical to the same call without gates; the schedules agree bit
for bit.  CPU: misuse returns DSPGN_E_ARG without a GPU, and the result record keeps its size and offsets.
"""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle import gate_check as G
from test_keyframe_batch import ENGINES, NATIVE, ROOT, _bits, _cfg, _new, _opt, _tracked

GATE_WORD = 85


def _sim3(seed, cls="cars"):
    from dsp_slam_b200 import synth
    return np.array(synth.make_object(seed + 7, 64, 8, 2, cls=cls)["t_cam_obj_init"], dtype=np.float32)


def _moved(T, dx=0.0, dz=0.0, angle=0.0):
    """T moved by (dx, 0, dz) in the camera frame and rotated by `angle` about the object's own y axis."""
    M = np.array(T, dtype=np.float32)
    if angle:
        M[:3, :3] = (M[:3, :3].astype(np.float64) @ Rotation.from_rotvec([0.0, angle, 0.0]).as_matrix()).astype(np.float32)
    M[0, 3] += np.float32(dx)
    M[2, 3] += np.float32(dz)
    return M


def _gated(seed, move, n_pts=200, cls="cars"):
    d = _tracked(seed, n_pts, cls)
    d["t_cam_obj_map"] = _moved(d["t_cam_obj"], **move)
    d["t_cam_obj_sim3"] = _sim3(seed, cls)
    return d


# the moves of the synthesised tracked detections: inside both thresholds, beyond 1 m in x/z, beyond 1.5 in |e| only
MOVES = [dict(), dict(dx=0.1, dz=-0.2), dict(dx=1.5), dict(dz=-2.0), dict(angle=2.0), dict(angle=-2.5)]


def _gate_in(d):
    return dict(t_cam_obj_map=d["t_cam_obj_map"], t_cam_obj_sim3=d["t_cam_obj_sim3"]) if "t_cam_obj_sim3" in d else None


def _joint_of(d):
    return dict(t_cam_obj=d["t_cam_obj_sim3"], pts=d["pts"], rays=d["rays"], depth=d["depth"], class_id=d["class_id"])


def _run_and_check(solver, objs, modes):
    """One gated call, checked object by object.  Returns (records, verdicts, near-threshold cases)."""
    gates = [_gate_in(o) if m else None for o, m in zip(objs, modes)]
    n = len(objs)
    got = _bits(solver.keyframe(objs, modes, gates), n)
    plain = _bits(solver.keyframe(objs, modes), n)            # the same call without gates
    gw = got.view(np.int32)[:, GATE_WORD]
    verdicts, near = [], 0
    rejected = [i for i in range(n) if gw[i] == G.REJECTED]
    want_j = _bits(solver.reconstruct([_joint_of(objs[i]) for i in rejected]), len(rejected)) if rejected else None
    for i in range(n):
        if gates[i] is None:
            assert gw[i] == 0, i
            assert np.array_equal(got[i], plain[i]), (i, np.flatnonzero(got[i] != plain[i])[:8])
            continue
        rec = plain[i].view(np.float32)
        Z = rec[:16].reshape(4, 4) if plain[i].view(np.int32)[81] == 0 else np.asarray(objs[i]["t_cam_obj"], np.float32)
        dist2d, e = G.gate_values(Z, gates[i]["t_cam_obj_map"])
        if abs(float(dist2d) - 1.0) < 1e-6 or abs(e - 1.5) < 1e-6:
            near += 1
        else:
            assert gw[i] == G.gate(Z, gates[i]["t_cam_obj_map"]), (i, dist2d, e, gw[i])
        verdicts.append(int(gw[i]))
        if gw[i] == G.KEPT:
            w = plain[i].copy()
            w.view(np.int32)[GATE_WORD] = G.KEPT
            assert np.array_equal(got[i], w), (i, np.flatnonzero(got[i] != w)[:8])
        else:
            assert gw[i] == G.REJECTED, (i, gw[i])
            w = want_j[rejected.index(i)].copy()
            w.view(np.int32)[GATE_WORD] = G.REJECTED
            assert np.array_equal(got[i], w), (i, np.flatnonzero(got[i] != w)[:8])
    return got, verdicts, near


def _keyframe(seed0=500):
    new = [_new(seed0 + 1), _new(seed0 + 2, 180, 90, 30, "chairs")]
    tracked = [_gated(seed0 + 10 + k, mv, cls="chairs" if k % 3 == 2 else "cars") for k, mv in enumerate(MOVES)]
    plain = _tracked(seed0 + 30)                                # gate = 0 with a large move: stays pose-only
    plain["t_cam_obj_map"] = _moved(plain["t_cam_obj"], dx=5.0)
    objs = [tracked[0], new[0]] + tracked[1:4] + [plain, new[1]] + tracked[4:]
    modes = [1, 0, 1, 1, 1, 1, 0, 1, 1]
    return objs, modes


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["simt", "tc"])
@pytest.mark.parametrize("pose_iters", [5, 7])
def test_gates_match_the_oracle_and_records_match_the_separate_calls(golden_dir, cfg_kitti, engine, pose_iters):
    objs, modes = _keyframe()
    recs = {}
    for schedule in (["launches", "persistent"] if engine == "tc" else ["launches"]):
        opt = _opt(golden_dir, _cfg(cfg_kitti, pose_iters), engine, schedule)
        got, verdicts, near = _run_and_check(opt.solver, objs, modes)
        assert near <= 1, near
        assert verdicts.count(G.KEPT) >= 1 and verdicts.count(G.REJECTED) >= 3, verdicts
        recs[schedule] = got
        if schedule == "persistent":
            opt.solver.keyframe(objs, modes, [_gate_in(o) if m else None for o, m in zip(objs, modes)])
            assert opt.solver.counters()["kernel_launches"] == 2
    if len(recs) == 2:
        assert np.array_equal(recs["launches"], recs["persistent"])


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_every_gated_object_rejected_at_once(golden_dir, cfg_kitti, engine, schedule):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    objs = [_gated(600 + k, dict(dx=3.0 + k), n_pts=150, cls="cars" if k % 2 else "chairs") for k in range(6)] + [_new(620)]
    modes = [1] * 6 + [0]
    _, verdicts, _ = _run_and_check(opt.solver, objs, modes)
    assert verdicts == [G.REJECTED] * 6


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_zero_rays_soft_failure_and_rejected_at_upload(golden_dir, cfg_kitti, engine, schedule):
    from dsp_slam_b200 import _lib
    opt = _opt(golden_dir, _cfg(cfg_kitti, 7), engine, schedule)
    no_rays = _gated(701, dict(dx=2.0))
    no_rays["rays"] = np.zeros((0, 3), np.float32); no_rays["depth"] = np.zeros(0, np.float32)
    nan_kept = _gated(702, dict())                                  # pose-only soft failure: checked with the input pose
    nan_kept["pts"] = np.array(nan_kept["pts"]); nan_kept["pts"][3] = np.nan
    nan_rej = _gated(703, dict(dz=2.0))
    nan_rej["pts"] = np.array(nan_rej["pts"]); nan_rej["pts"][5] = np.nan
    empty_kept = _gated(704, dict())                                # rejected at upload: the input pose too
    empty_kept["pts"] = np.zeros((0, 3), np.float32)
    empty_rej = _gated(705, dict(angle=2.2))
    empty_rej["pts"] = np.zeros((0, 3), np.float32)
    objs = [no_rays, _new(706), nan_kept, nan_rej, empty_kept, empty_rej, _gated(707, dict())]
    modes = [1, 0, 1, 1, 1, 1, 1]
    got, verdicts, _ = _run_and_check(opt.solver, objs, modes)
    assert verdicts == [G.REJECTED, G.KEPT, G.REJECTED, G.KEPT, G.REJECTED, G.KEPT], verdicts
    st = got.view(np.int32)[:, 81]
    assert st[0] == _lib.ST_RENDER_FEW and st[2] != 0 and st[3] != 0 and st[4] == _lib.ST_BAD_INPUT and st[5] == _lib.ST_BAD_INPUT, st


@pytest.mark.gpu
def test_more_than_one_resident_batch_with_gates_across_the_edges(golden_dir, cfg_kitti):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), "tc", "persistent")
    n = 1040
    objs, modes = [], []
    for i in range(n):
        if i % 4 == 0:
            objs.append(_new(2000 + i, 64, 24, 8)); modes.append(0)
        elif i % 4 == 2 or (1000 <= i <= 1030):
            objs.append(_gated(2000 + i, dict(dx=2.0) if i % 3 else dict(), n_pts=64)); modes.append(1)
        else:
            objs.append(_tracked(2000 + i, 64, outliers=4)); modes.append(1)
    _, verdicts, _ = _run_and_check(opt.solver, objs, modes)
    assert G.KEPT in verdicts and G.REJECTED in verdicts


@pytest.mark.gpu
def test_optimizer_keyframe_batch_with_gated_tracked_objects(golden_dir, cfg_kitti):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), None, None)
    new = [_new(801)]
    tracked = [_gated(802, dict()), _gated(803, dict(dx=2.0)), _tracked(804)]
    res, Ts, st, rejected = opt.keyframe_batch(new, tracked, return_status=True)
    res0, Ts0, st0 = opt.keyframe_batch(new, [dict(t) for t in tracked[2:]], return_status=True)
    assert rejected[0] is None and rejected[2] is None and rejected[1] is not None
    assert Ts[1] is None and st[1] is None
    np.testing.assert_array_equal(Ts[2], Ts0[0])
    ref = opt.reconstruct_batch([_joint_of(tracked[1])])[0]
    assert rejected[1].is_good == ref.is_good and np.float32(rejected[1].loss) == np.float32(ref.loss)
    if ref.is_good:
        np.testing.assert_array_equal(rejected[1].t_cam_obj, ref.t_cam_obj)
        np.testing.assert_array_equal(rejected[1].code, ref.code)
    np.testing.assert_array_equal(res[0].t_cam_obj, res0[0].t_cam_obj)
    # without the gate keys: today's two-element return
    assert len(opt.keyframe_batch(new, [_tracked(805)])) == 2


def _build_caller(tmp):
    exe = os.path.join(tmp, "keyframe_gate_caller")
    libd = os.path.join(ROOT, "dsp_slam_b200")
    subprocess.check_call(["gcc", "-O1", "-std=c11", f"-I{os.path.join(ROOT, 'include')}",
                           os.path.join(NATIVE, "keyframe_gate_caller.c"), "-o", exe, f"-L{libd}", "-ldspgn",
                           f"-Wl,-rpath,{libd}", "-lm"])
    return exe


def test_gate_caller_compiles_and_links(tmp_path):
    exe = _build_caller(str(tmp_path))
    assert subprocess.run([exe]).returncode == 2


@pytest.mark.gpu
def test_plain_c_gate_caller_matches_python(tmp_path, golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib
    from dsp_slam_b200.decoder import DecoderWeights
    from dsp_slam_b200.optimizer import Optimizer
    exe = _build_caller(str(tmp_path))
    dec = os.path.join(golden_dir, "decoder_cars.npz")
    w = DecoderWeights.from_npz(dec)
    wp, inp, outp = str(tmp_path / "w.bin"), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(wp, "wb") as f:
        f.write(struct.pack("<3i", len(w.W), w.latent_size, w.latent_in_layer))
        for W, b in zip(w.W, w.b):
            f.write(struct.pack("<2i", *W.shape)); f.write(W.tobytes()); f.write(b.tobytes())
    dets = [_gated(901, dict()), _gated(902, dict(dx=2.0)), _gated(903, dict(angle=2.0))]
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
    got = np.frombuffer(open(outp, "rb").read(), np.uint32).reshape(len(dets), _lib.RESULT_FLOATS)
    opt = Optimizer(dec, cfg_kitti)
    objs = [dict(d, class_id=0) for d in dets]
    want = _bits(opt.solver.keyframe(objs, [1] * len(dets), [_gate_in(d) for d in dets]), len(dets))
    assert np.array_equal(got, want)
    assert list(got.view(np.int32)[:, GATE_WORD]) == [G.KEPT, G.REJECTED, G.REJECTED]


def test_result_record_layout_is_unchanged():
    from dsp_slam_b200 import _lib
    assert C.sizeof(_lib.ObjectOut) == 352
    offs = {n: getattr(_lib.ObjectOut, n).offset for n, _ in _lib.ObjectOut._fields_}
    assert offs == {"t_cam_obj": 0, "code": 64, "loss": 320, "status": 324, "n_valid": 328, "n_band": 332,
                    "iters_done": 336, "gate": 340, "pad_": 344}
    hdr = open(os.path.join(ROOT, "include", "dspgn.h")).read()
    assert "int32_t gate;" in hdr and "int32_t pad_[2];" in hdr
    assert (_lib.GATE_OFF, _lib.GATE_KEPT, _lib.GATE_REJECTED) == (0, 1, 2) == (0, G.KEPT, G.REJECTED)


def test_gated_misuse_returns_e_arg_before_touching_cuda():
    from dsp_slam_b200 import _lib
    lib = _lib.load()
    FP = C.POINTER(C.c_float)
    T = np.eye(4, dtype=np.float32)
    P = np.zeros((8, 3), np.float32)
    code = np.zeros(64, np.float32)
    Tcw = np.eye(4, dtype=np.float32)
    ins = (_lib.ObjectIn * 2)()
    for o in ins:
        o.t_cam_obj = T.ctypes.data_as(FP); o.t_rs = 4; o.t_cs = 1
        o.pts = P.ctypes.data_as(FP); o.n_pts = 8; o.pts_rs = 3; o.pts_cs = 1
        o.code = code.ctypes.data_as(FP); o.scale = 1.0
    outs = (_lib.ObjectOut * 2)()
    modes = (C.c_int32 * 2)(0, 1)
    fake = C.create_string_buffer(64)
    h = C.cast(fake, C.c_void_p)

    def gates():
        g = (_lib.GateIn * 2)()
        g[1].t_cam_obj_map = T.ctypes.data_as(FP); g[1].map_rs = 4; g[1].map_cs = 1
        g[1].t_cam_obj_sim3 = T.ctypes.data_as(FP); g[1].sim3_rs = 4; g[1].sim3_cs = 1
        g[1].gate = 1
        return g

    assert lib.dspgn_keyframe_batch_gated(None, 2, ins, modes, gates(), outs) == -1
    assert lib.dspgn_keyframe_batch_gated(h, 0, ins, modes, gates(), outs) == -1
    assert lib.dspgn_keyframe_batch_gated(h, 2, ins, None, gates(), outs) == -1
    g = gates(); g[0].t_cam_obj_map = T.ctypes.data_as(FP); g[0].t_cam_obj_sim3 = T.ctypes.data_as(FP); g[0].gate = 1
    assert lib.dspgn_keyframe_batch_gated(h, 2, ins, modes, g, outs) == -1          # gate on a joint object
    assert b"pose-only" in lib.dspgn_last_error()
    g = gates(); g[1].t_cam_obj_map = None
    assert lib.dspgn_keyframe_batch_gated(h, 2, ins, modes, g, outs) == -1          # no map pose
    assert b"t_cam_obj_map" in lib.dspgn_last_error()
    g = gates(); g[1].t_cam_obj_sim3 = None
    assert lib.dspgn_keyframe_batch_gated(h, 2, ins, modes, g, outs) == -1          # no Sim(3) pose
    g = gates(); g[1].gate = 3
    assert lib.dspgn_keyframe_batch_gated(h, 2, ins, modes, g, outs) == -1
    assert b"gate must be" in lib.dspgn_last_error()
    ins[1].t_cam_world = Tcw.ctypes.data_as(FP)
    assert lib.dspgn_keyframe_batch_gated(h, 2, ins, modes, gates(), outs) == -1    # world-frame inputs
    assert b"t_cam_world" in lib.dspgn_last_error()
    ins[1].t_cam_world = None
    ins[1].code = None
    assert lib.dspgn_keyframe_batch_gated(h, 2, ins, modes, gates(), outs) == -1    # the keyframe checks still apply
    assert b"code" in lib.dspgn_last_error()
