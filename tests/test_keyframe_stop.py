"""Cooperative stop of a running keyframe call (dspgn_keyframe_stop, dspgn_solver_set_stop_flag, dspgn_debug_stop_at;
BatchSolver.request_stop / set_stop_flag, KeyframeFuture.stop): LocalMapping's mbAbortBA exits of CreateNewMapObjects.

What holds at any timing of the stop, and is checked on every stopped call: an object that ends DSPGN_ST_STOPPED is a
stoppable one (a joint object outside a mono pair, or the joint slot of a rejected gated object), its record is -- status
and mesh word aside -- bit-identical to the record of the same call run with num_iterations = iters_done, its mesh word
is DSPGN_MESH_FAILED and its grid NaN; every other record, gate word and mesh is bit-identical to the unstopped call.
GPU: both engines, both schedules, the device-side trigger, a second thread, a registered flag.  CPU: the argument checks
and the ctypes mirror of the new entry points.
"""
import copy
import ctypes as C
import os
import re
import struct
import subprocess
import threading
import time

import numpy as np
import pytest

from test_keyframe_batch import ENGINES, NATIVE, ROOT, _bits, _cfg, _new, _opt
from test_keyframe_mesh import _stereo_keyframe

GATE_WORD, MESH_WORD, STATUS_WORD, ITERS_WORD = 85, 86, 81, 84
DIM = 8
ITERS = 10            # _cfg(cfg, 5): 10 joint iterations, 5 pose-only ones
NEW = 1               # the first new object of _stereo_keyframe


def _call(solver, objs, modes, gates, pairs=None):
    """One meshed keyframe call: (records as uint32 bits, meshes, grids)."""
    out, meshes, sdf = solver.keyframe(objs, modes, gates, voxels_dim=DIM, pairs=pairs, want_sdf=True)
    return _bits(out, len(objs)), meshes, np.asarray(sdf).reshape(len(objs), -1)


def _same_mesh(a, b):
    if a is None or b is None:
        return a is None and b is None
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


class _Reference:
    """The unstopped call, and the same call at fewer joint iterations (one solver per iteration count)."""

    def __init__(self, golden_dir, cfg_kitti, engine, schedule, objs, modes, gates, pairs=None):
        self.args = (golden_dir, cfg_kitti, engine, schedule)
        self.call = (objs, modes, gates, pairs)
        self.cache = {}
        self.base = self.at(ITERS)

    def at(self, iters):
        if iters not in self.cache:
            golden_dir, cfg_kitti, engine, schedule = self.args
            cfg = copy.deepcopy(_cfg(cfg_kitti, 5))
            cfg["optimizer"]["joint_optim"]["num_iterations"] = iters
            opt = _opt(golden_dir, cfg, engine, schedule)
            self.cache[iters] = _call(opt.solver, *self.call)
            opt.solver.close()
        return self.cache[iters]


def _check_stopped(ref, got, meshes, grids):
    """The properties of a stopped call that hold whenever the stop came.  Returns the indices that ended STOPPED."""
    from dsp_slam_b200 import _lib
    objs, modes, gates, pairs = ref.call
    base, base_meshes, base_grids = ref.base
    bi, gi = base.view(np.int32), got.view(np.int32)
    stopped = []
    for i in range(len(objs)):
        if gi[i, STATUS_WORD] != _lib.ST_STOPPED:
            assert np.array_equal(got[i], base[i]), (i, np.flatnonzero(got[i] != base[i])[:8])
            assert _same_mesh(meshes[i], base_meshes[i]), i
            assert np.array_equal(grids[i], base_grids[i], equal_nan=True), i
            continue
        paired = pairs is not None and pairs[i] >= 0
        assert not paired and (modes[i] == _lib.MODE_JOINT or bi[i, GATE_WORD] == _lib.GATE_REJECTED), i
        assert gi[i, GATE_WORD] == bi[i, GATE_WORD], i
        assert gi[i, MESH_WORD] == _lib.MESH_FAILED and meshes[i] is None, i
        assert np.isnan(grids[i]).all(), i
        k = int(gi[i, ITERS_WORD])
        assert 0 <= k < ITERS, (i, k)
        if k == 0:                          # the joint slot of a rejected gated object that never woke
            assert gates[i] is not None, i
            T = np.asarray(gates[i]["t_cam_obj_sim3"], dtype=np.float32).reshape(16)
            assert np.array_equal(got[i, :16], T.view(np.uint32)), i
            assert not got[i, 16:81].any() and not got[i, 82:85].any(), i
        else:
            want = ref.at(k)[0][i].copy()
            have = got[i].copy()
            have[[STATUS_WORD, MESH_WORD]] = 0
            want[[STATUS_WORD, MESH_WORD]] = 0
            assert np.array_equal(have, want), (i, k, np.flatnonzero(have != want)[:8])
        stopped.append(i)
    return stopped


@pytest.fixture(scope="module")
def stereo():
    objs, modes, gates = _stereo_keyframe()
    return objs, modes, gates


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_device_trigger_stops_at_the_iteration_with_the_prefix_records(golden_dir, cfg_kitti, engine, schedule, stereo):
    from dsp_slam_b200 import _lib
    objs, modes, gates = stereo
    ref = _Reference(golden_dir, cfg_kitti, engine, schedule, objs, modes, gates)
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    for k in (0, ITERS // 2, ITERS - 1):
        opt.solver.debug_stop_at(NEW, k)
        got, meshes, grids = _call(opt.solver, objs, modes, gates)
        stopped = _check_stopped(ref, got, meshes, grids)
        if k == ITERS - 1:                  # a last solve reads nothing and raises nothing
            assert stopped == []
        else:
            gi = got.view(np.int32)
            assert NEW in stopped and gi[NEW, ITERS_WORD] == k + 1
            assert gi[NEW, STATUS_WORD] == _lib.ST_STOPPED
        c = opt.solver.counters()
        assert c["rows_fwd_bwd"] > 0
    # the hook was one call's: the next call runs to the end
    got, meshes, grids = _call(opt.solver, objs, modes, gates)
    assert np.array_equal(got, ref.base[0])


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_stop_before_a_rejected_slot_wakes_leaves_it_unrun(golden_dir, cfg_kitti, engine, schedule, stereo):
    from dsp_slam_b200 import _lib
    objs, modes, gates = stereo
    ref = _Reference(golden_dir, cfg_kitti, engine, schedule, objs, modes, gates)
    bi = ref.base[0].view(np.int32)
    rejected = [i for i in range(len(objs)) if bi[i, GATE_WORD] == _lib.GATE_REJECTED]
    assert rejected
    g = rejected[0]
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    opt.solver.debug_stop_at(g, 4)          # its last pose-only iteration: the stop comes before its verdict wakes the slot
    got, meshes, grids = _call(opt.solver, objs, modes, gates)
    stopped = _check_stopped(ref, got, meshes, grids)
    gi = got.view(np.int32)
    assert g in stopped
    assert gi[g, ITERS_WORD] == 0 and gi[g, GATE_WORD] == _lib.GATE_REJECTED and gi[g, MESH_WORD] == _lib.MESH_FAILED


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_mono_pairs_and_reconstruct_batch(golden_dir, cfg_kitti, engine, schedule):
    """Both hypotheses of a pair run to the end; dspgn_reconstruct_batch stops like the keyframe calls."""
    from dsp_slam_b200 import _lib
    d = _new(760)
    Tf = np.array(d["t_cam_obj"], np.float32)
    Tf[:, 0] *= -1; Tf[:, 2] *= -1
    objs = [d, dict(d, t_cam_obj=Tf), _new(761, cls="chairs"), _new(762)]
    pairs, modes, gates = [1, 0, -1, -1], [0, 0, 0, 0], [None] * 4
    ref = _Reference(golden_dir, cfg_kitti, engine, schedule, objs, modes, gates, pairs)
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    opt.solver.debug_stop_at(0, 2)          # raised by no one: the paired object's solves never read the word
    got, meshes, grids = _call(opt.solver, objs, modes, gates, pairs)
    assert _check_stopped(ref, got, meshes, grids) == []
    opt.solver.debug_stop_at(2, 2)
    got, meshes, grids = _call(opt.solver, objs, modes, gates, pairs)
    stopped = _check_stopped(ref, got, meshes, grids)
    assert 2 in stopped and got.view(np.int32)[2, ITERS_WORD] == 3 and 0 not in stopped and 1 not in stopped
    # dspgn_reconstruct_batch: the same prefix records
    plain = [objs[2], objs[3]]
    opt.solver.debug_stop_at(0, 3)
    rec = _bits(opt.solver.reconstruct(plain), 2)
    assert rec.view(np.int32)[0, STATUS_WORD] == _lib.ST_STOPPED and rec.view(np.int32)[0, ITERS_WORD] == 4
    cfg = copy.deepcopy(_cfg(cfg_kitti, 5))
    for i in range(2):
        k = int(rec.view(np.int32)[i, ITERS_WORD])
        cfg["optimizer"]["joint_optim"]["num_iterations"] = k
        want = _bits(_opt(golden_dir, cfg, engine, schedule).solver.reconstruct(plain), 2)[i]
        have = rec[i].copy()
        have[STATUS_WORD] = want[STATUS_WORD]
        assert np.array_equal(have, want), i
    res = opt.reconstruct_batch(plain)
    assert all(r.is_good for r in res)      # no stop without a request
    opt.solver.debug_stop_at(1, 0)
    res = opt.reconstruct_batch(plain)
    assert not res[1].is_good and res[1].status == _lib.ST_STOPPED
    # object 0 stopped too when its solve of the same iteration read the word after the trigger (same launch)
    assert res[0].is_good or res[0].status == _lib.ST_STOPPED


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_submitted_call_stopped_from_another_thread(golden_dir, cfg_kitti, engine, schedule, stereo):
    objs, modes, gates = stereo
    ref = _Reference(golden_dir, cfg_kitti, engine, schedule, objs, modes, gates)
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    s = opt.solver
    s.request_stop()                        # idle solver: no effect, neither on a blocking call nor on a submit
    s.request_stop()
    got, meshes, grids = _call(s, objs, modes, gates)
    assert np.array_equal(got, ref.base[0])
    s.request_stop()
    s.keyframe_submit(objs, modes, gates, voxels_dim=DIM)
    out, meshes, sdf = s.keyframe_wait(want_sdf=True)
    assert np.array_equal(_bits(out, len(objs)), ref.base[0])
    assert all(_same_mesh(a, b) for a, b in zip(meshes, ref.base[1]))
    for delay in (0.0, 0.001, 0.003, 0.010):
        s.keyframe_submit(objs, modes, gates, voxels_dim=DIM)
        t = threading.Thread(target=lambda: (time.sleep(delay), s.request_stop()))
        t.start()
        out, meshes, sdf = s.keyframe_wait(want_sdf=True)
        t.join()
        _check_stopped(ref, _bits(out, len(objs)), meshes, np.asarray(sdf).reshape(len(objs), -1))
    s.request_stop()                        # after the wait: never reaches the next call
    got, meshes, grids = _call(s, objs, modes, gates)
    assert np.array_equal(got, ref.base[0])
    assert all(_same_mesh(a, b) for a, b in zip(meshes, ref.base[1]))
    # the Optimizer surface: KeyframeFuture.stop.  A result that did not stop is the unstopped call's; a stopped one is
    # is_good=False with status STOPPED and the loss of the same call at fewer iterations
    from dsp_slam_b200 import _lib
    new = [objs[i] for i in range(len(objs)) if modes[i] == 0]
    ref_new = _Reference(golden_dir, cfg_kitti, engine, schedule, new, [0] * len(new), [None] * len(new))
    base_res = opt.reconstruct_mono_batch([dict(o) for o in new])
    fut = opt.reconstruct_mono_batch_async([dict(o) for o in new])
    fut.stop()
    res = fut.result()
    assert len(res) == len(new)
    for i, (r, b) in enumerate(zip(res, base_res)):
        if r.status != _lib.ST_STOPPED:
            assert r.status == b.status and np.float32(r.loss) == np.float32(b.loss), i
            if b.is_good:
                assert np.array_equal(r.code, b.code) and np.array_equal(r.t_cam_obj, b.t_cam_obj), i
            continue
        assert not r.is_good and r.t_cam_obj is None and r.code is None, i
        losses = [ref_new.at(k)[0][i].view(np.float32)[80] for k in range(1, ITERS)]
        assert any(np.float32(r.loss).view(np.uint32) == l.view(np.uint32) for l in losses), i
    fut.stop()                              # settled: no effect


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_registered_flag(golden_dir, cfg_kitti, engine, schedule, stereo):
    objs, modes, gates = stereo
    ref = _Reference(golden_dir, cfg_kitti, engine, schedule, objs, modes, gates)
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    s = opt.solver
    flag = C.c_uint8(0)
    s.set_stop_flag(C.addressof(flag))
    h0 = s.host_syncs()
    got, meshes, grids = _call(s, objs, modes, gates)
    assert np.array_equal(got, ref.base[0]) and all(_same_mesh(a, b) for a, b in zip(meshes, ref.base[1]))
    assert s.host_syncs() > h0
    for delay in (0.0005, 0.002):
        flag.value = 0
        t = threading.Thread(target=lambda: (time.sleep(delay), setattr(flag, "value", 1)))
        t.start()
        got, meshes, grids = _call(s, objs, modes, gates)
        t.join()
        _check_stopped(ref, got, meshes, grids)
    flag.value = 1                          # set before the call: the first wait stops it
    got, meshes, grids = _call(s, objs, modes, gates)
    _check_stopped(ref, got, meshes, grids)
    s.set_stop_flag(None)                   # unregistered: the flag is not read any more
    got, meshes, grids = _call(s, objs, modes, gates)
    assert np.array_equal(got, ref.base[0])


@pytest.mark.gpu
def test_stop_at_ranges(golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), None, None)
    lib, h = _lib.load(), opt.solver.handle
    for obj, it in [(-1, 0), (0, -1), (-2, -2), (0, ITERS), (0, 1 << 30)]:
        assert lib.dspgn_debug_stop_at(h, obj, it) == _lib.E_ARG, (obj, it)
    assert lib.dspgn_debug_stop_at(h, 0, ITERS - 1) == 0
    assert lib.dspgn_debug_stop_at(h, -1, -1) == 0
    assert lib.dspgn_keyframe_stop(h) == 0


# ---- plain-C caller: CreateNewMapObjects with mbAbortBA raised by a second pthread ----------------------------------
def _build_stop_caller(tmp):
    exe = os.path.join(tmp, "keyframe_stop_caller")
    libd = os.path.join(ROOT, "dsp_slam_b200")
    subprocess.check_call(["gcc", "-O1", "-std=c11", "-Wall", "-Werror", f"-I{os.path.join(ROOT, 'include')}",
                           os.path.join(NATIVE, "keyframe_stop_caller.c"), "-o", exe, f"-L{libd}", "-ldspgn",
                           f"-Wl,-rpath,{libd}", "-lpthread", "-lm"])
    return exe


def test_keyframe_stop_caller_compiles_and_links(tmp_path):
    exe = _build_stop_caller(str(tmp_path))
    assert subprocess.run([exe]).returncode == 2


@pytest.mark.gpu
def test_plain_c_stop_caller_matches_python(tmp_path, golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib
    from dsp_slam_b200.decoder import DecoderWeights
    from dsp_slam_b200.optimizer import Optimizer
    from test_keyframe_gate import _gate_in, _gated
    from test_keyframe_mesh import _read_call
    exe = _build_stop_caller(str(tmp_path))
    dec = os.path.join(golden_dir, "decoder_cars.npz")
    w = DecoderWeights.from_npz(dec)
    wp, inp, outp = str(tmp_path / "w.bin"), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(wp, "wb") as f:
        f.write(struct.pack("<3i", len(w.W), w.latent_size, w.latent_in_layer))
        for W, b in zip(w.W, w.b):
            f.write(struct.pack("<2i", *W.shape)); f.write(W.tobytes()); f.write(b.tobytes())
    dets = [_gated(960, dict()), _gated(961, dict(dx=2.0)), _gated(962, dict(angle=2.5))]
    new = _new(963)
    with open(inp, "wb") as f:
        f.write(struct.pack("<i", len(dets)))
        for d in dets:
            f.write(struct.pack("<3i", d["pts"].shape[0], d["rays"].shape[0], d["depth"].shape[0]))
            for a in (d["t_cam_obj"], d["t_cam_obj_map"], d["t_cam_obj_sim3"], d["pts"], d["rays"]):
                f.write(np.asarray(a, np.float32).tobytes(order="F"))
            f.write(np.asarray(d["depth"], np.float32).tobytes())
            f.write(struct.pack("<f", float(d["scale"])))
            f.write(np.asarray(d["code"], np.float32).reshape(-1)[:64].tobytes())
        f.write(struct.pack("<3i", new["pts"].shape[0], new["rays"].shape[0], new["depth"].shape[0]))
        for a in (new["t_cam_obj"], new["pts"], new["rays"]):
            f.write(np.asarray(a, np.float32).tobytes(order="F"))
        f.write(np.asarray(new["depth"], np.float32).tobytes())
    r = subprocess.run([exe, wp, inp, outp, "200"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    raw = open(outp, "rb").read()
    n = len(dets) + 1
    calls, off = [], 0
    for _ in range(3):
        rec, m, off = _read_call(raw, off, n)
        calls.append((rec, m))
    assert off == len(raw)
    objs = [dict(d, class_id=0) for d in dets] + [new]
    modes, gates = [1] * len(dets) + [0], [_gate_in(d) for d in dets] + [None]

    def python_call(iters):
        cfg = copy.deepcopy(cfg_kitti)
        cfg["optimizer"]["joint_optim"]["num_iterations"] = iters
        opt = Optimizer(dec, cfg)
        out, meshes = opt.solver.keyframe(objs, modes, gates, voxels_dim=16)
        return _bits(out, n), meshes

    iters = int(cfg_kitti["optimizer"]["joint_optim"]["num_iterations"])
    want, want_m = python_call(iters)
    for c in (0, 2):                        # the flag never raised, and the call after the stopped one
        rec, m = calls[c]
        assert np.array_equal(rec, want), c
        for g_, w_ in zip(m, want_m):
            assert (w_ is None and g_[0].shape[0] == 0) or (np.array_equal(g_[0], w_[0]) and np.array_equal(g_[1], w_[1]))
    rec, m = calls[1]
    ri = rec.view(np.int32)
    stopped = [i for i in range(n) if ri[i, STATUS_WORD] == _lib.ST_STOPPED]
    assert stopped, "the flag raised 200 us after the submit stopped nothing"
    nums = [int(x) for x in re.findall(r"-?\d+", r.stdout.split(":", 1)[1])]
    done = int((want.view(np.int32)[:, MESH_WORD] == _lib.MESH_DONE).sum())
    assert nums == [done, 0, done, 0, len(stopped), 0], r.stdout     # a stopped call creates no object
    for i in range(n):
        if i not in stopped:
            assert np.array_equal(rec[i], want[i]), i
            continue
        assert modes[i] == 0 or want.view(np.int32)[i, GATE_WORD] == _lib.GATE_REJECTED, i
        assert ri[i, MESH_WORD] == _lib.MESH_FAILED and m[i][0].shape[0] == 0, i
        k = int(ri[i, ITERS_WORD])
        if k == 0:
            T = np.asarray(dets[i]["t_cam_obj_sim3"], np.float32).reshape(16)
            assert np.array_equal(rec[i, :16], T.view(np.uint32)) and not rec[i, 16:81].any(), i
        else:
            ref = python_call(k)[0][i].copy()
            have = rec[i].copy()
            have[[STATUS_WORD, MESH_WORD]] = 0
            ref[[STATUS_WORD, MESH_WORD]] = 0
            assert np.array_equal(have, ref), (i, k)


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_null_solver_is_e_arg_without_a_gpu():
    from dsp_slam_b200 import _lib
    lib = _lib.load()
    flag = C.c_uint8(0)
    assert lib.dspgn_keyframe_stop(None) == _lib.E_ARG
    assert lib.dspgn_solver_set_stop_flag(None, C.addressof(flag)) == _lib.E_ARG
    assert lib.dspgn_solver_set_stop_flag(None, None) == _lib.E_ARG
    assert lib.dspgn_debug_stop_at(None, 0, 0) == _lib.E_ARG
    assert lib.dspgn_debug_stop_at(None, -1, -1) == _lib.E_ARG


def test_ctypes_mirror_of_the_stop_entry_points():
    from dsp_slam_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "dspgn.h")).read()
    assert re.search(r"#define DSPGN_ST_STOPPED 6\b", hdr) and _lib.ST_STOPPED == 6
    assert (_lib.ST_OK, _lib.ST_BAD_INPUT) == (0, 5)
    sym = {n: (r, a) for n, r, a in _lib.SYMBOLS}
    ctypes_of = {"DspgnSolver*": C.c_void_p, "int": C.c_int, "const volatile uint8_t*": C.c_void_p}
    for name in ("dspgn_keyframe_stop", "dspgn_solver_set_stop_flag", "dspgn_debug_stop_at"):
        decl = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", hdr).group(1)
        params = [" ".join(p.split()[:-1]) for p in decl.split(",")]
        assert sym[name] == (C.c_int, [ctypes_of[p] for p in params]), (name, params)
    # the in-flight exception list names the stop
    assert "dspgn_keyframe_stop, dspgn_solver_sync" in hdr


def test_future_stop_of_a_settled_future_calls_nothing():
    from dsp_slam_b200.optimizer import KeyframeFuture
    f = KeyframeFuture.resolved([1])
    f.stop()
    assert f.result() == [1]
