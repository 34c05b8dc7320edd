"""Non-blocking keyframe calls (dspgn_keyframe_submit / _query / _wait, BatchSolver.keyframe_submit / keyframe_wait,
Optimizer.keyframe_batch_async / reconstruct_mono_batch_async and their KeyframeFuture).

GPU, both engines and both schedules: submit + wait returns records, mesh counts, vertices and faces bit-identical to
the blocking call; a warm solver's submit never blocks on the device; the inputs are not read after the submit; a mesh
arena that is far too small changes nothing; every other entry point is busy while a call is in flight; two solvers
can have calls in flight at once; the plain-C caller gets the blocking call's results.  CPU: the futures and the busy
rule of the Python layer with the library stubbed, and the C ABI's argument checks.
"""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

from test_keyframe_batch import ENGINES, NATIVE, ROOT, _bits, _cfg, _new, _opt, _tracked
from test_keyframe_gate import _gate_in, _gated, _moved

GATE_WORD = 85


# ---- fixtures --------------------------------------------------------------------------------------------------------
def _stereo():
    """A stereo keyframe: three new objects (cars and a chair), six gated tracked objects of which the map check rejects
    two (moved 1.5 m, turned by 2 rad), and one ungated tracked object."""
    from dsp_slam_b200 import _lib
    new = [_new(900), _new(901, cls="chairs"), _new(902)]
    moves = [dict(), dict(dx=0.1, dz=-0.2), dict(dx=1.5), dict(dz=0.2), dict(angle=2.0), dict(dx=-0.2)]
    tracked = [_gated(910 + k, mv, cls="chairs" if k == 3 else "cars") for k, mv in enumerate(moves)]
    tracked.append(_tracked(920))
    objs = new + tracked
    modes = [_lib.MODE_JOINT] * len(new) + [_lib.MODE_POSE] * len(tracked)
    gates = [None] * len(new) + [_gate_in(o) for o in tracked]
    return objs, modes, gates


def _mono():
    """Three mono detections as pairs (map pose, flipped about y), one of them a duplicated hypothesis, and one unpaired."""
    objs, pairs = [], []
    for k, cls in enumerate(["cars", "chairs", "cars"]):
        d = _new(930 + k, cls=cls)
        Tf = np.array(d["t_cam_obj"], np.float32)
        Tf[:, 0] *= -1; Tf[:, 2] *= -1
        i = len(objs)
        objs += [d, dict(d, t_cam_obj=Tf) if k < 2 else dict(d)]
        pairs += [i + 1, i]
    objs.append(_new(935)); pairs.append(-1)
    return objs, [0] * len(objs), pairs


def _no_candidates():
    """A keyframe with tracked objects only, none gated: nothing to wake and nothing to mesh."""
    objs = [_tracked(940 + k) for k in range(3)]
    return objs, [1] * 3, None


def _async(solver, objs, modes, gates, dim, pairs=None):
    solver.keyframe_submit(objs, modes, gates, voxels_dim=dim, pairs=pairs)
    return solver.keyframe_wait()


def _same(got, want, n, dim):
    """(records[, meshes]) of two calls are bit-identical."""
    if dim is None:
        assert np.array_equal(_bits(got, n), _bits(want, n))
        return
    assert np.array_equal(_bits(got[0], n), _bits(want[0], n))
    for i, (a, b) in enumerate(zip(got[1], want[1])):
        assert (a is None) == (b is None), i
        if a is not None:
            assert a[0].dtype == b[0].dtype and a[1].dtype == b[1].dtype
            assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1]), i


def _fresh(objs):
    """Deep copies of every array of the objects (the originals stay untouched)."""
    return [{k: (np.array(v, copy=True, order="K") if isinstance(v, np.ndarray) else v) for k, v in o.items()} for o in objs]


# ---- GPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dim", [32, 64, None])
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_stereo_keyframe_submit_wait_equals_blocking(golden_dir, cfg_kitti, engine, schedule, dim):
    from dsp_slam_b200 import _lib
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    objs, modes, gates = _stereo()
    n = len(objs)
    want = opt.solver.keyframe(objs, modes, gates, voxels_dim=dim)
    got = _async(opt.solver, objs, modes, gates, dim)
    _same(got, want, n, dim)
    rec = _bits(got if dim is None else got[0], n).view(np.int32)
    assert [int(g) for g in rec[3:9, GATE_WORD]].count(_lib.GATE_REJECTED) == 2
    if dim is not None:                                          # the rejected detections are mesh candidates
        rejected = [i for i in range(3, 9) if rec[i, GATE_WORD] == _lib.GATE_REJECTED]
        assert all(rec[i, 86] in (_lib.MESH_DONE, _lib.MESH_FAILED) for i in rejected)
        assert any(m is not None for m in got[1][:3])
    again = _async(opt.solver, objs, modes, gates, dim)          # a second submit on the same solver
    _same(again, want, n, dim)


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_mono_pairs_and_a_keyframe_without_candidates(golden_dir, cfg_kitti, engine, schedule):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    objs, modes, pairs = _mono()
    want = opt.solver.keyframe(objs, modes, voxels_dim=64, pairs=pairs)
    _same(_async(opt.solver, objs, modes, None, 64, pairs), want, len(objs), 64)
    objs, modes, gates = _no_candidates()
    for dim in (32, None):
        want = opt.solver.keyframe(objs, modes, gates, voxels_dim=dim)
        got = _async(opt.solver, objs, modes, gates, dim)
        _same(got, want, len(objs), dim)
        if dim is not None:
            assert all(m is None for m in got[1])


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_submit_never_blocks_and_reads_no_input_afterwards(golden_dir, cfg_kitti, engine, schedule):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    objs, modes, gates = _stereo()
    n = len(objs)
    want = opt.solver.keyframe(objs, modes, gates, voxels_dim=32)
    _async(opt.solver, objs, modes, gates, 32)                   # warm: the solver's buffers fit this keyframe
    mine = _fresh(objs)
    my_gates = [None if g is None else dict(t_cam_obj_map=np.array(g["t_cam_obj_map"], np.float32),
                                            t_cam_obj_sim3=np.array(g["t_cam_obj_sim3"], np.float32)) for g in gates]
    before = opt.solver.host_syncs()
    opt.solver.keyframe_submit(mine, modes, my_gates, voxels_dim=32)
    assert opt.solver.host_syncs() == before                     # submit added no host synchronisation
    for o in mine:                                               # every input array overwritten right after the submit
        for v in o.values():
            if isinstance(v, np.ndarray) and v.dtype.kind == "f":
                v[...] = np.nan
    for g in my_gates:
        if g is not None:
            g["t_cam_obj_map"][...] = np.nan
            g["t_cam_obj_sim3"][...] = np.nan
    _same(opt.solver.keyframe_wait(), want, n, 32)


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_an_arena_of_a_few_vertices_gives_the_same_meshes(golden_dir, cfg_kitti, engine, schedule):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    objs, modes, gates = _stereo()
    want = opt.solver.keyframe(objs, modes, gates, voxels_dim=64)
    assert sum(m[0].shape[0] for m in want[1] if m is not None) > 8
    opt.solver.set_mesh_arena(4, 4)
    _same(_async(opt.solver, objs, modes, gates, 64), want, len(objs), 64)
    opt.solver.set_mesh_arena(0, 0)
    _same(_async(opt.solver, objs, modes, gates, 64), want, len(objs), 64)


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_every_other_entry_point_is_busy_in_flight(golden_dir, cfg_kitti, engine, schedule):
    from dsp_slam_b200 import _lib
    lib = _lib.load()
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    s = opt.solver
    objs, modes, gates = _stereo()
    n = len(objs)
    want = s.keyframe(objs, modes, gates, voxels_dim=32)
    arr, m, g, spec, keep = s._keyframe_args(objs, modes, gates, 32, None)
    h = s.handle
    out = (_lib.ObjectOut * n)()
    nv, nf = (C.c_int32 * n)(), (C.c_int32 * n)()
    FP = C.POINTER(C.c_float)
    buf = np.zeros(1 << 16, np.float32)
    p = buf.ctypes.data_as(FP)
    ip = C.cast(p, C.POINTER(C.c_int32))
    code = np.zeros(64, np.float32).ctypes.data_as(FP)
    _lib.check(lib.dspgn_keyframe_submit(h, n, arr, m, g, C.byref(spec)))
    B = _lib.E_BUSY
    busy = {
        "keyframe_submit": lib.dspgn_keyframe_submit(h, n, arr, m, g, C.byref(spec)),
        "keyframe_batch": lib.dspgn_keyframe_batch(h, n, arr, m, out),
        "keyframe_batch_gated": lib.dspgn_keyframe_batch_gated(h, n, arr, m, g, out),
        "keyframe_batch_meshed": lib.dspgn_keyframe_batch_meshed(h, n, arr, m, g, C.byref(spec), out, nv, nf),
        "reconstruct_batch": lib.dspgn_reconstruct_batch(h, 1, arr, out),
        "estimate_pose_batch": lib.dspgn_estimate_pose_batch(h, 1, arr, out),
        "upload_batch": lib.dspgn_upload_batch(h, 1, arr),
        "run_batch": lib.dspgn_run_batch(h, 0),
        "run_batch_modes": lib.dspgn_run_batch_modes(h, m),
        "results": lib.dspgn_results(h, out),
        "decode_sdf": lib.dspgn_decode_sdf(h, 0, code, p, 4, 3, 1, p),
        "mesh_batch": lib.dspgn_mesh_batch(h, 1, code, 64, None, 8, nv, nf),
        "mesh_results": lib.dspgn_mesh_results(h, p, ip, None),
        "debug_mesh_grid": lib.dspgn_debug_mesh_grid(h, 1, 8, p, nv, nf),
        "counters": lib.dspgn_counters(h, C.byref(_lib.Counters())),
        "enable_timing": lib.dspgn_enable_timing(h, 0),
        "set_stream": lib.dspgn_solver_set_stream(h, None),
        "debug_system": lib.dspgn_debug_system(h, 0, 0, p, p, p, None, None, None),
        "debug_system_iter": lib.dspgn_debug_system_iter(h, 0, 0, 1, p, p, p, None, None, None),
        "debug_inputs": lib.dspgn_debug_inputs(h, 0, p, None, None),
        "debug_events": lib.dspgn_debug_events(h, C.cast(p, C.POINTER(C.c_longlong)), 4),
        "debug_mesh_arena": lib.dspgn_debug_mesh_arena(h, 4, 4),
        "gather_create": lib.dspgn_gather_create(h, 4, 1, C.byref(_lib.IpcHandle())),
        "gather_bind": lib.dspgn_gather_bind(h, None, 0),
        "run_batch_gather": lib.dspgn_run_batch_gather(h, 0, 1),
        "gather_results": lib.dspgn_gather_results(h, 1, 1, out),
    }
    assert {k: v for k, v in busy.items() if v != B} == {}
    assert lib.dspgn_results_device(h) is None
    assert lib.dspgn_keyframe_query(h) in (0, 1)
    assert lib.dspgn_solver_engine(h) in (_lib.ENGINE_SIMT, _lib.ENGINE_TC)
    _lib.check(lib.dspgn_solver_sync(h))
    assert lib.dspgn_keyframe_query(h) == 1
    assert lib.dspgn_keyframe_wait(h, out, None, None) == _lib.E_ARG   # the counts are required: the call stays in flight
    _lib.check(lib.dspgn_keyframe_wait(h, out, nv, nf))
    s._flight = None
    assert np.array_equal(_bits(out, n), _bits(want[0], n))
    assert list(nv) == [0 if w is None else w[0].shape[0] for w in want[1]]
    assert lib.dspgn_keyframe_wait(h, out, nv, nf) == _lib.E_ARG       # nothing in flight any more
    assert lib.dspgn_keyframe_query(h) == _lib.E_ARG
    _same(s._meshed(out, n, 32, nv, nf, False), want, n, 32)


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_two_solvers_in_flight_at_once(golden_dir, cfg_kitti, engine, schedule):
    a = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    b = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    objs, modes, gates = _stereo()
    mono, mmodes, pairs = _mono()
    want_a = a.solver.keyframe(objs, modes, gates, voxels_dim=32)
    want_b = b.solver.keyframe(mono, mmodes, voxels_dim=64, pairs=pairs)
    a.solver.keyframe_submit(objs, modes, gates, voxels_dim=32)
    b.solver.keyframe_submit(mono, mmodes, voxels_dim=64, pairs=pairs)
    _same(b.solver.keyframe_wait(), want_b, len(mono), 64)
    _same(a.solver.keyframe_wait(), want_a, len(objs), 32)


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_optimizer_futures_equal_the_blocking_methods(golden_dir, cfg_kitti, engine, schedule):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    objs, modes, gates = _stereo()
    new, tracked = objs[:3], objs[3:]

    def same_results(x, y):
        assert len(x) == len(y)
        for r, w in zip(x, y):
            if r is None or w is None:
                assert r is None and w is None
                continue
            assert set(r) == set(w)
            for k in r:
                assert np.array_equal(np.asarray(r[k]), np.asarray(w[k]), equal_nan=True) if r[k] is not None else w[k] is None, k

    want = opt.keyframe_batch(new, tracked, return_status=True, voxels_dim=32)
    fut = opt.keyframe_batch_async(new, tracked, voxels_dim=32, return_status=True)
    got = fut.result()
    assert fut.done() and len(got) == len(want) == 4
    same_results(got[0], want[0])
    for T, W in zip(got[1], want[1]):
        assert (T is None and W is None) or np.array_equal(T, W)
    assert got[2] == want[2]
    same_results(got[3], want[3])
    mono = [dict(objs[0], t_cam_obj_flipped=_moved(objs[0]["t_cam_obj"], angle=np.pi)), objs[1]]
    want_m = opt.reconstruct_mono_batch(mono, voxels_dim=32)
    fut = opt.reconstruct_mono_batch_async(mono, voxels_dim=32)
    # another method called while the future is outstanding collects it first
    poses = opt.estimate_pose_batch(tracked[-1:])
    assert fut.done()
    same_results(fut.result(), want_m)
    assert np.array_equal(poses[0], want[1][-1])


# ---- plain-C caller --------------------------------------------------------------------------------------------------
def _build_caller(tmp):
    exe = os.path.join(tmp, "keyframe_async_caller")
    libd = os.path.join(ROOT, "dsp_slam_b200")
    subprocess.check_call(["gcc", "-O1", "-std=c11", "-Wall", "-Werror", f"-I{os.path.join(ROOT, 'include')}",
                           os.path.join(NATIVE, "keyframe_async_caller.c"), "-o", exe, f"-L{libd}", "-ldspgn",
                           f"-Wl,-rpath,{libd}", "-lm"])
    return exe


def test_keyframe_async_caller_compiles_and_links(tmp_path):
    exe = _build_caller(str(tmp_path))
    assert subprocess.run([exe]).returncode == 2


@pytest.mark.gpu
def test_plain_c_async_caller_matches_the_blocking_call(tmp_path, golden_dir, cfg_kitti):
    from dsp_slam_b200.decoder import DecoderWeights
    from dsp_slam_b200.optimizer import Optimizer
    from test_keyframe_mesh import _read_call
    exe = _build_caller(str(tmp_path))
    dec = os.path.join(golden_dir, "decoder_cars.npz")
    w = DecoderWeights.from_npz(dec)
    wp, inp, outp = str(tmp_path / "w.bin"), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(wp, "wb") as f:
        f.write(struct.pack("<3i", len(w.W), w.latent_size, w.latent_in_layer))
        for W, b in zip(w.W, w.b):
            f.write(struct.pack("<2i", *W.shape)); f.write(W.tobytes()); f.write(b.tobytes())
    dets = [_gated(950, dict()), _gated(951, dict(dx=2.0)), _gated(952, dict(angle=2.5))]
    new = _new(953)
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
    r = subprocess.run([exe, wp, inp, outp], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    raw = open(outp, "rb").read()
    n = len(dets) + 1
    rec1, m1, off = _read_call(raw, 0, n)
    rec2, m2, off = _read_call(raw, off, 2)
    assert off == len(raw)
    opt = Optimizer(dec, cfg_kitti)
    objs = [dict(d, class_id=0) for d in dets] + [new]
    out, want1 = opt.solver.keyframe(objs, [1] * len(dets) + [0], [_gate_in(d) for d in dets] + [None], voxels_dim=16)
    assert np.array_equal(rec1, _bits(out, n))
    Tf = np.array(new["t_cam_obj"], np.float32)
    Tf[:, 0] *= -1; Tf[:, 2] *= -1
    out, want2 = opt.solver.keyframe([new, dict(new, t_cam_obj=Tf)], [0, 0], voxels_dim=16, pairs=[1, 0])
    assert np.array_equal(rec2, _bits(out, 2))
    for got, want in ((m1, want1), (m2, want2)):
        for g_, w_ in zip(got, want):
            if w_ is None:
                assert g_[0].shape[0] == 0 and g_[1].shape[0] == 0
            else:
                assert np.array_equal(g_[0], w_[0]) and np.array_equal(g_[1], w_[1])
    assert any(w_ is not None for w_ in want1)
    assert "meshes" in r.stdout


# ---- no GPU ----------------------------------------------------------------------------------------------------------
def test_c_abi_of_the_async_calls_checks_arguments_before_touching_cuda():
    import re
    from dsp_slam_b200 import _lib
    lib = _lib.load()
    for name in ("dspgn_keyframe_submit", "dspgn_keyframe_query", "dspgn_keyframe_wait", "dspgn_debug_host_syncs",
                 "dspgn_debug_mesh_arena"):
        assert hasattr(lib, name)
    hdr = open(os.path.join(ROOT, "include", "dspgn.h")).read()
    assert re.search(r"#define DSPGN_E_BUSY \(-6\)", hdr) and _lib.E_BUSY == -6
    sym = {n: a for n, _, a in _lib.SYMBOLS}
    assert len(sym["dspgn_keyframe_submit"]) == 6 and len(sym["dspgn_keyframe_wait"]) == 4
    FP = C.POINTER(C.c_float)
    T = np.eye(4, dtype=np.float32)
    P = np.zeros((8, 3), np.float32)
    ins = (_lib.ObjectIn * 2)()
    for o in ins:
        o.t_cam_obj = T.ctypes.data_as(FP); o.t_rs = 4; o.t_cs = 1
        o.pts = P.ctypes.data_as(FP); o.n_pts = 8; o.pts_rs = 3; o.pts_cs = 1
    h = C.cast(C.create_string_buffer(64), C.c_void_p)      # never dereferenced: the arguments fail first
    spec = _lib.MeshSpec()
    spec.voxels_dim = 1
    assert lib.dspgn_keyframe_submit(None, 2, ins, None, None, None) == _lib.E_ARG
    assert lib.dspgn_keyframe_submit(h, 0, ins, None, None, None) == _lib.E_ARG
    assert lib.dspgn_keyframe_submit(h, 2, None, None, None, None) == _lib.E_ARG
    assert lib.dspgn_keyframe_submit(h, 2, ins, (C.c_int32 * 2)(0, 3), None, None) == _lib.E_ARG
    assert lib.dspgn_keyframe_submit(h, 2, ins, None, None, C.byref(spec)) == _lib.E_ARG
    assert b"voxels_dim" in lib.dspgn_last_error()
    assert lib.dspgn_keyframe_query(None) == _lib.E_ARG
    assert lib.dspgn_keyframe_wait(None, (_lib.ObjectOut * 2)(), None, None) == _lib.E_ARG
    assert lib.dspgn_debug_host_syncs(None, C.byref(C.c_int64())) == _lib.E_ARG
    assert lib.dspgn_debug_mesh_arena(None, 0, 0) == _lib.E_ARG
    assert lib.dspgn_debug_mesh_arena(h, 4, 0) == _lib.E_ARG


class _FakeLib:
    """The library calls the Python layer makes, on the host: one call in flight, DSPGN_E_BUSY otherwise."""

    def __init__(self, wait_rc=0, finish_after=1):
        self.log, self.inflight, self.wait_rc, self.polls, self.finish_after = [], None, wait_rc, 0, finish_after

    def dspgn_last_error(self):
        return b"stub"

    def dspgn_keyframe_submit(self, h, n, arr, m, g, spec):
        if self.inflight is not None:
            return -6
        self.log.append("submit")
        self.inflight = (n, [arr[i].n_pts for i in range(n)], [m[i] for i in range(n)])
        return 0

    def dspgn_keyframe_query(self, h):
        self.polls += 1
        return 1 if self.polls > self.finish_after else 0

    def dspgn_keyframe_wait(self, h, out, nv, nf):
        self.log.append("wait")
        n, npts, modes = self.inflight
        self.inflight = None
        if self.wait_rc:
            return self.wait_rc
        for i in range(n):
            out[i].status = 0
            out[i].loss = float(npts[i])
            for r in range(4):
                out[i].t_cam_obj[5 * r] = 2.0
            out[i].code[0] = float(i)
        return 0

    def dspgn_estimate_pose_batch(self, h, n, arr, out):
        if self.inflight is not None:
            return -6
        self.log.append("estimate_pose")
        for i in range(n):
            out[i].status = 4                      # soft failure: the input pose comes back
        return 0


def _stub_optimizer(monkeypatch, fake):
    from dsp_slam_b200 import _lib
    from dsp_slam_b200.optimizer import BatchSolver, Optimizer
    monkeypatch.setattr(_lib, "load", lambda: fake)
    s = BatchSolver.__new__(BatchSolver)
    s.handle, s.cfg, s.n_obj, s._keep = None, _lib.Config(), 0, None      # close() has nothing to destroy
    s.cfg.code_len = 8
    opt = Optimizer.__new__(Optimizer)
    opt.solver, opt.code_len, opt._pending = s, 8, None
    return opt


def _objs():
    new = [dict(t_cam_obj=np.eye(4, dtype=np.float32), pts=np.zeros((5 + k, 3), np.float32)) for k in range(2)]
    tracked = [dict(t_cam_obj=np.eye(4, dtype=np.float32) * 3, pts=np.zeros((9, 3), np.float32),
                    code=np.zeros(8, np.float32), scale=1.0)]
    return new, tracked


def test_future_done_never_blocks_and_result_is_the_blocking_value(monkeypatch):
    fake = _FakeLib(finish_after=2)
    opt = _stub_optimizer(monkeypatch, fake)
    new, tracked = _objs()
    fut = opt.keyframe_batch_async(new, tracked, return_status=True)
    assert fake.log == ["submit"] and fake.inflight[2] == [0, 0, 1]
    assert not fut.done() and not fut.done() and fut.done()      # query only, no wait
    assert fake.log == ["submit"]
    results, poses, status = fut.result()
    assert fake.log == ["submit", "wait"]
    assert [r.loss for r in results] == [5.0, 6.0] and all(r.is_good for r in results)
    assert status == [0] and np.array_equal(poses[0], np.diag([2.0, 2.0, 2.0, 2.0]).astype(np.float32))
    assert fut.result() is fut.result() and fake.log == ["submit", "wait"]   # collected once


def test_another_method_collects_the_outstanding_future_first(monkeypatch):
    fake = _FakeLib()
    opt = _stub_optimizer(monkeypatch, fake)
    new, tracked = _objs()
    fut = opt.keyframe_batch_async(new, tracked)
    T = opt.estimate_pose_batch(tracked)                         # would be E_BUSY without the collection
    assert fake.log == ["submit", "wait", "estimate_pose"]
    assert np.array_equal(T[0], tracked[0]["t_cam_obj"])
    assert fut.done() and len(fut.result()[0]) == 2
    f2 = opt.reconstruct_mono_batch_async([dict(new[0], t_cam_obj_flipped=np.eye(4, dtype=np.float32))])
    f3 = opt.keyframe_batch_async(new, [])                       # a second submit collects the first
    assert fake.log[-3:] == ["submit", "wait", "submit"]
    kept = f2.result()
    assert len(kept) == 1 and kept[0].flipped is False           # equal losses keep the map pose
    assert [r.loss for r in f3.result()[0]] == [5.0, 6.0]


def test_a_failed_call_is_a_soft_failure_of_every_object(monkeypatch):
    fake = _FakeLib(wait_rc=-2)
    opt = _stub_optimizer(monkeypatch, fake)
    new, tracked = _objs()
    tracked[0]["t_cam_obj_map"] = np.eye(4, dtype=np.float32)
    tracked[0]["t_cam_obj_sim3"] = np.eye(4, dtype=np.float32)
    tracked[0]["rays"] = np.zeros((4, 3), np.float32)
    tracked[0]["depth"] = np.zeros(2, np.float32)
    fut = opt.keyframe_batch_async(new, tracked, return_status=True)
    tracked[0]["t_cam_obj"][...] = 7.0                           # the fallback pose is the one given at submit
    results, poses, status, rejected = fut.result()               # never raises
    assert [r.is_good for r in results] == [False, False] and status == [-1] and rejected == [None]
    assert np.array_equal(poses[0], np.eye(4, dtype=np.float32) * 3)
    fake.wait_rc = 0
    fake.inflight = ("busy",)                                     # the library refuses the submit
    fut = opt.reconstruct_mono_batch_async([new[0]])
    assert fut.done() and [r.is_good for r in fut.result()] == [False]
    assert opt.keyframe_batch_async([], []).result() == ([], [])
