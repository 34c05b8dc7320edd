"""Meshed keyframe calls (dspgn_keyframe_batch_meshed, BatchSolver.keyframe(..., voxels_dim, pairs),
Optimizer.reconstruct_batch / keyframe_batch / reconstruct_mono_batch with voxels_dim): poses, codes and meshes of a
keyframe's new objects from one call.

Every call is checked against the calls it replaces: its records are bit-identical to the same call without meshes
(dspgn_keyframe_batch_gated) but for the mesh word; the mesh word follows CreateNewMapObjects / ProcessDetectedObjects
applied to those records; every DSPGN_MESH_DONE mesh is bit-identical to dspgn_mesh_batch of the record's code and class.
GPU: both engines, both schedules, dims 8 to 128, pairs, chunks.  CPU: misuse returns DSPGN_E_ARG without a GPU, the
Python wrappers check their arguments, and the plain-C caller compiles and links.
"""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

from test_keyframe_batch import ENGINES, NATIVE, ROOT, _bits, _cfg, _new, _opt, _tracked
from test_keyframe_gate import _gate_in, _gated, _keyframe, _moved

MESH_WORD = 86
GATE_WORD = 85


def _expected_words(plain, modes, gates, pairs):
    """The mesh word of every object from the unmeshed call's records: LocalMapping's rules restated."""
    from dsp_slam_b200 import _lib
    ints, flts = plain.view(np.int32), plain.view(np.float32)
    n = len(modes)
    want = []
    for i in range(n):
        cand = modes[i] == 0 or (gates[i] is not None and ints[i, GATE_WORD] == _lib.GATE_REJECTED)
        if not cand:
            want.append(_lib.MESH_OFF)
            continue
        j = pairs[i] if pairs is not None else -1
        if j >= 0:
            lo, hi = min(i, j), max(i, j)
            winner = hi if flts[lo, 80] > flts[hi, 80] else lo
            if winner != i:
                want.append(_lib.MESH_LOST)
                continue
        want.append(_lib.MESH_DONE if ints[i, 81] == _lib.ST_OK else _lib.MESH_FAILED)
    return want


def _check_call(solver, objs, modes, gates, dim, pairs=None, want_sdf=False):
    """One meshed call against the unmeshed call and dspgn_mesh_batch.  Returns (records, meshes, words[, sdf])."""
    from dsp_slam_b200 import _lib
    n = len(objs)
    ret = solver.keyframe(objs, modes, gates, voxels_dim=dim, pairs=pairs, want_sdf=want_sdf)
    got, meshes = _bits(ret[0], n), ret[1]
    words = got.view(np.int32)[:, MESH_WORD].tolist()
    plain = _bits(solver.keyframe(objs, modes, gates if gates is not None else None), n)
    gl = gates if gates is not None else [None] * n
    assert words == _expected_words(plain, modes, gl, pairs), words
    stripped = got.copy()
    stripped.view(np.int32)[:, MESH_WORD] = 0
    for i in range(n):
        assert np.array_equal(stripped[i], plain[i]), (i, np.flatnonzero(stripped[i] != plain[i])[:8])
    done = [i for i in range(n) if words[i] == _lib.MESH_DONE]
    assert [i for i in range(n) if meshes[i] is not None] == done
    if done:
        codes = got.view(np.float32)[done, 16:16 + solver.cfg.code_len]
        want = solver.mesh(codes, dim, [int(objs[i].get("class_id", 0)) for i in done])
        for k, i in enumerate(done):
            assert np.array_equal(meshes[i][0], want[k][0]) and np.array_equal(meshes[i][1], want[k][1]), i
    return (got, meshes, words, ret[2]) if want_sdf else (got, meshes, words)


def _stereo_keyframe():
    """_keyframe (new cars and chairs, kept / rejected gated objects, a plain pose-only one) plus a new object whose rays
    miss it (render soft failure) and an unusable detection."""
    from dsp_slam_b200 import _lib
    objs, modes = _keyframe(700)
    few = _new(731)
    few["rays"] = np.asfortranarray(np.tile(np.array([[3.0, 3.0, 1.0]], np.float32), (40, 1)))
    few["depth"] = np.zeros(0, np.float32)
    empty = _new(732, cls="chairs")
    empty["pts"] = np.zeros((0, 3), np.float32)
    objs = objs + [few, empty]
    modes = modes + [_lib.MODE_JOINT, _lib.MODE_JOINT]
    gates = [_gate_in(o) if m else None for o, m in zip(objs, modes)]
    return objs, modes, gates


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [8, 32, 64])
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_stereo_keyframe_records_words_and_meshes(golden_dir, cfg_kitti, engine, schedule, dim):
    from dsp_slam_b200 import _lib
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    objs, modes, gates = _stereo_keyframe()
    got, meshes, words = _check_call(opt.solver, objs, modes, gates, dim)
    gw, st = got.view(np.int32)[:, GATE_WORD], got.view(np.int32)[:, 81]
    assert words[-1] == _lib.MESH_FAILED and st[-1] == _lib.ST_BAD_INPUT               # unusable detection
    assert words[-2] == _lib.MESH_FAILED and st[-2] == _lib.ST_RENDER_FEW              # render soft failure
    assert all(w == _lib.MESH_OFF for w, g in zip(words, gw) if g == _lib.GATE_KEPT)
    rejected = [i for i in range(len(objs)) if gw[i] == _lib.GATE_REJECTED]
    assert rejected and any(words[i] == _lib.MESH_DONE for i in rejected)
    assert words[modes.index(_lib.MODE_POSE, 5)] == _lib.MESH_OFF                      # the ungated pose-only object
    assert {objs[i]["class_id"] for i in range(len(objs)) if words[i] == _lib.MESH_DONE} == {0, 1}
    assert all(meshes[i][1].shape[0] > 0 for i in range(len(objs)) if words[i] == _lib.MESH_DONE)
    c = opt.solver.counters()
    assert c["rows_fwd_only"] >= words.count(_lib.MESH_DONE) * dim ** 3


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", ENGINES)
def test_mono_pairs_follow_the_loss_rule(golden_dir, cfg_kitti, engine, schedule):
    from dsp_slam_b200 import _lib
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    objs, pairs = [], []

    def add_pair(a, b):
        i = len(objs)
        objs.extend([a, b])
        pairs.extend([i + 1, i])

    for k, cls in enumerate(["cars", "chairs", "cars"]):
        d = _new(740 + k, cls=cls)
        Tf = np.array(d["t_cam_obj"], np.float32)
        Tf[:, 0] *= -1; Tf[:, 2] *= -1                               # LocalMapping_util.cc:394-401: flipped about y
        add_pair(d, dict(d, t_cam_obj=Tf))
    dup = _new(750)
    add_pair(dup, dict(dup))                                         # duplicated detection: a tie keeps i
    bad = _new(751)
    add_pair(dict(bad, pts=np.zeros((0, 3), np.float32)), bad)       # the better-loss member failed
    objs.insert(2, _new(752)); pairs.insert(2, -1)                   # an unpaired object between pairs
    pairs = [p + (1 if p >= 2 else 0) if p >= 0 else -1 for p in pairs]
    modes = [0] * len(objs)
    got, meshes, words = _check_call(opt.solver, objs, modes, None, 16, pairs)
    i_dup = next(k for k, o in enumerate(objs) if o is dup)
    assert (words[i_dup], words[i_dup + 1]) == (_lib.MESH_DONE, _lib.MESH_LOST)
    assert (words[-2], words[-1]) == (_lib.MESH_FAILED, _lib.MESH_LOST) and meshes[-2] is None
    # the Optimizer surface keeps the winner and says which hypothesis it was
    mono = [dict(objs[0], t_cam_obj_flipped=objs[1]["t_cam_obj"]), objs[2], dict(dup, t_cam_obj_flipped=dup["t_cam_obj"])]
    res = opt.reconstruct_mono_batch(mono, voxels_dim=16)
    for r, (i, j) in zip(res, [(0, 1), (2, -1), (i_dup, i_dup + 1)]):
        w = j if j >= 0 and words[i] == _lib.MESH_LOST else i
        assert r.flipped == (w != i)
        rec = got[w].view(np.float32)
        assert r.loss == rec[80]
        if words[w] == _lib.MESH_DONE:
            assert np.array_equal(r.code, rec[16:16 + opt.code_len])
            assert np.array_equal(r.vertices, meshes[w][0]) and np.array_equal(r.faces, meshes[w][1])
    plain = opt.reconstruct_mono_batch(mono)
    assert [r.flipped for r in plain] == [r.flipped for r in res]


@pytest.mark.gpu
def test_schedules_give_identical_grids_meshes_and_words(golden_dir, cfg_kitti):
    objs, modes, gates = _stereo_keyframe()
    pairs = [-1] * len(objs)
    out = {}
    for schedule in ("launches", "persistent"):
        opt = _opt(golden_dir, _cfg(cfg_kitti, 5), "tc", schedule)
        out[schedule] = _check_call(opt.solver, objs, modes, gates, 32, pairs, want_sdf=True)
    a, b = out["launches"], out["persistent"]
    assert np.array_equal(a[0], b[0]) and a[2] == b[2]
    assert np.array_equal(a[3].view(np.uint32), b[3].view(np.uint32))
    for ma, mb in zip(a[1], b[1]):
        assert (ma is None) == (mb is None)
        if ma is not None:
            assert np.array_equal(ma[0], mb[0]) and np.array_equal(ma[1], mb[1])
    sdf = a[3]
    for i, w in enumerate(a[2]):
        assert np.isnan(sdf[i]).all() == (w != 1), i


@pytest.mark.gpu
@pytest.mark.parametrize("engine,schedule", [("simt", "launches"), ("tc", "persistent")])
def test_chunk_bound_at_dim_128(golden_dir, cfg_kitti, engine, schedule):
    """9 candidates of 128^3 rows: the walker puts the pair that would cross 2^24 rows into the next chunk."""
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, schedule)
    objs = [_new(760 + k, 120, 60, 20, "chairs" if k % 3 == 1 else "cars") for k in range(7)]
    d = _new(770)
    objs += [d, dict(d, t_cam_obj=_moved(d["t_cam_obj"], angle=np.pi))]
    pairs = [-1] * 7 + [8, 7]
    modes = [0] * 9
    got, meshes, words = _check_call(opt.solver, objs, modes, None, 128, pairs)
    for lo, hi in ((0, 7), (7, 9)):                                  # the same as the separate per-chunk calls
        pp = None if lo == 0 else [1, 0]
        out, m = opt.solver.keyframe(objs[lo:hi], modes[lo:hi], voxels_dim=128, pairs=pp)
        assert np.array_equal(_bits(out, hi - lo), got[lo:hi])
        for k in range(hi - lo):
            assert (m[k] is None) == (meshes[lo + k] is None)
            if m[k] is not None:
                assert np.array_equal(m[k][0], meshes[lo + k][0]) and np.array_equal(m[k][1], meshes[lo + k][1])


@pytest.mark.gpu
def test_more_than_1024_objects_with_gates_and_pairs(golden_dir, cfg_kitti):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), None, None)
    objs, modes, gates, pairs = [], [], [], []
    for i in range(1030):
        if i % 5 == 1:
            objs.append(_gated(2000 + i, dict(dx=3.0) if i % 10 == 1 else dict(), n_pts=64)); modes.append(1)
            gates.append(_gate_in(objs[-1]))
        elif i % 5 == 3:
            objs.append(_tracked(2000 + i, 64, outliers=4)); modes.append(1); gates.append(None)
        else:
            objs.append(_new(2000 + i, 64, 24, 8)); modes.append(0); gates.append(None)
    # pairs of new objects four apart (the objects between them are walked after the pair), one across the edge of
    # the first resident chunk (five objects take six slots: it ends near object 853)
    pairs = [-1] * len(objs)
    for i in (0, 850, 1020):
        assert modes[i] == 0 and modes[i + 4] == 0
        pairs[i], pairs[i + 4] = i + 4, i
    _check_call(opt.solver, objs, modes, gates, 8, pairs)


@pytest.mark.gpu
def test_misuse_leaves_the_resident_batch_untouched(golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), None, None)
    s = opt.solver
    objs, modes, gates = _stereo_keyframe()
    s.upload(objs[:4])
    s.run_modes(modes[:4])
    before = _bits(s.results_raw(), 4)
    n = len(objs)
    pose = modes.index(1)
    gated = next(i for i, g in enumerate(gates) if g is not None)
    joint = [i for i, m in enumerate(modes) if m == 0]
    bad = [dict(voxels_dim=1), dict(voxels_dim=129),
           dict(voxels_dim=8, pairs=[pose if i == joint[0] else (joint[0] if i == pose else -1) for i in range(n)]),
           dict(voxels_dim=8, pairs=[gated if i == joint[0] else (joint[0] if i == gated else -1) for i in range(n)]),
           dict(voxels_dim=8, pairs=[joint[1] if i == joint[0] else -1 for i in range(n)]),
           dict(voxels_dim=8, pairs=[joint[0] if i == joint[0] else -1 for i in range(n)]),
           dict(voxels_dim=8, pairs=[n if i == joint[0] else -1 for i in range(n)])]
    for kw in bad:
        with pytest.raises(_lib.DspgnError) as e:
            s.keyframe(objs, modes, gates, **kw)
        assert e.value.code == _lib.E_ARG, kw
    assert np.array_equal(_bits(s.results_raw(), 4), before)
    s.run_modes(modes[:4])
    assert np.array_equal(_bits(s.results_raw(), 4), before)


@pytest.mark.gpu
def test_optimizer_surfaces_carry_the_meshes(golden_dir, cfg_kitti):
    from dsp_slam_b200.optimizer import MeshExtractor
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), None, None)
    new = [_new(780), _new(781, cls="chairs")]
    res = opt.reconstruct_batch(new, voxels_dim=16)
    ref = opt.reconstruct_batch(new)
    ext = MeshExtractor(os.path.join(golden_dir, "decoder_cars.npz"), opt.code_len, 16)
    for r, w, o in zip(res, ref, new):
        assert r.is_good == w.is_good and r.loss == w.loss
        if r.is_good:
            assert np.array_equal(r.code, w.code)
            m = opt.solver.mesh(r.code[None], 16, [o["class_id"]])[0]
            assert np.array_equal(r.vertices, m[0]) and np.array_equal(r.faces, m[1])
            if o["class_id"] == 0:
                e = ext.extract_meshes([r.code])[0]
                assert np.array_equal(r.vertices, e.vertices) and np.array_equal(r.faces, e.faces)
    tracked = [_gated(790, dict(dx=3.0)), _gated(791, dict())]
    r1, T1, rej1 = opt.keyframe_batch(new, tracked, voxels_dim=16)
    r0, T0, rej0 = opt.keyframe_batch(new, tracked)
    assert [x.loss for x in r1] == [x.loss for x in r0]
    assert rej1[0] is not None and rej1[1] is None and rej0[1] is None
    if rej1[0].is_good:
        m = opt.solver.mesh(rej1[0].code[None], 16, [0])[0]
        assert np.array_equal(rej1[0].vertices, m[0]) and np.array_equal(rej1[0].faces, m[1])


# ---- C caller -----------------------------------------------------------------------------------------------------
def _build_caller(tmp):
    exe = os.path.join(tmp, "keyframe_mesh_caller")
    libd = os.path.join(ROOT, "dsp_slam_b200")
    subprocess.check_call(["gcc", "-O1", "-std=c11", "-Wall", "-Werror", f"-I{os.path.join(ROOT, 'include')}",
                           os.path.join(NATIVE, "keyframe_mesh_caller.c"), "-o", exe, f"-L{libd}", "-ldspgn",
                           f"-Wl,-rpath,{libd}"])
    return exe


def test_keyframe_mesh_caller_compiles_and_links(tmp_path):
    exe = _build_caller(str(tmp_path))
    assert subprocess.run([exe]).returncode == 2


def _read_call(raw, off, n):
    from dsp_slam_b200 import _lib
    rec = np.frombuffer(raw, np.uint32, n * _lib.RESULT_FLOATS, off).reshape(n, _lib.RESULT_FLOATS)
    off += rec.nbytes
    nv = np.frombuffer(raw, np.int32, n, off); off += 4 * n
    nf = np.frombuffer(raw, np.int32, n, off); off += 4 * n
    V = np.frombuffer(raw, np.float32, 3 * int(nv.sum()), off).reshape(-1, 3); off += V.nbytes
    F = np.frombuffer(raw, np.int32, 3 * int(nf.sum()), off).reshape(-1, 3); off += F.nbytes
    ov, of = np.concatenate([[0], np.cumsum(nv)]), np.concatenate([[0], np.cumsum(nf)])
    return rec, [(V[ov[i]:ov[i + 1]], F[of[i]:of[i + 1]]) for i in range(n)], off


@pytest.mark.gpu
def test_plain_c_keyframe_mesh_caller_matches_python(tmp_path, golden_dir, cfg_kitti):
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
    dets = [_gated(810, dict()), _gated(811, dict(dx=2.0)), _gated(812, dict(angle=2.5))]
    new = _new(813)
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
        for g, w_ in zip(got, want):
            if w_ is None:
                assert g[0].shape[0] == 0 and g[1].shape[0] == 0
            else:
                assert np.array_equal(g[0], w_[0]) and np.array_equal(g[1], w_[1])
    assert any(w_ is not None for w_ in want1)
    assert "meshes" in r.stdout


# ---- no GPU ---------------------------------------------------------------------------------------------------------
def test_meshed_misuse_returns_e_arg_before_touching_cuda():
    from dsp_slam_b200 import _lib
    lib = _lib.load()
    FP = C.POINTER(C.c_float)
    T = np.eye(4, dtype=np.float32)
    P = np.zeros((8, 3), np.float32)
    code = np.zeros(64, np.float32)
    ins = (_lib.ObjectIn * 3)()
    for o in ins:
        o.t_cam_obj = T.ctypes.data_as(FP); o.t_rs = 4; o.t_cs = 1
        o.pts = P.ctypes.data_as(FP); o.n_pts = 8; o.pts_rs = 3; o.pts_cs = 1
        o.code = code.ctypes.data_as(FP); o.scale = 1.0
    outs = (_lib.ObjectOut * 3)()
    nv, nf = (C.c_int32 * 3)(), (C.c_int32 * 3)()
    modes = (C.c_int32 * 3)(0, 0, 1)
    h = C.cast(C.create_string_buffer(64), C.c_void_p)

    def spec(dim=8, pair=None):
        s = _lib.MeshSpec()
        s.voxels_dim = dim
        s.pair = None if pair is None else (C.c_int32 * 3)(*pair)
        return C.byref(s)

    def call(sp, g=None, m=modes):
        return lib.dspgn_keyframe_batch_meshed(h, 3, ins, m, g, sp, outs, nv, nf)

    assert lib.dspgn_keyframe_batch_meshed(None, 3, ins, modes, None, spec(), outs, nv, nf) == -1
    assert lib.dspgn_keyframe_batch_meshed(h, 3, ins, modes, None, None, outs, nv, nf) == -1
    assert lib.dspgn_keyframe_batch_meshed(h, 3, ins, modes, None, spec(), outs, None, nf) == -1
    for dim in (1, 0, 129, -3):
        assert call(spec(dim)) == -1
        assert b"voxels_dim" in lib.dspgn_last_error()
    for pair in ([1, -1, -1], [0, -1, -1], [3, -1, -1], [-2, -1, -1], [1, 2, 0]):      # asymmetric, self, out of range
        assert call(spec(8, pair)) == -1, pair
        assert b"pair must be" in lib.dspgn_last_error()
    assert call(spec(8, [2, -1, 0])) == -1                                           # a pair with a pose-only object
    assert b"ungated joint" in lib.dspgn_last_error()
    g = (_lib.GateIn * 3)()
    g[2].t_cam_obj_map = T.ctypes.data_as(FP); g[2].map_rs = 4; g[2].map_cs = 1
    g[2].t_cam_obj_sim3 = T.ctypes.data_as(FP); g[2].sim3_rs = 4; g[2].sim3_cs = 1
    g[2].gate = 1
    both_pose = (C.c_int32 * 3)(0, 1, 1)
    assert call(spec(8, [-1, 2, 1]), g, both_pose) == -1                             # a pair with a gated object
    assert b"ungated joint" in lib.dspgn_last_error()
    assert call(spec(8), g, (C.c_int32 * 3)(0, 0, 0)) == -1                         # the gated call's checks still apply
    assert b"pose-only" in lib.dspgn_last_error()


def test_python_wrappers_check_their_arguments():
    from dsp_slam_b200 import _lib
    from dsp_slam_b200.optimizer import BatchSolver
    s = BatchSolver.__new__(BatchSolver)          # no device: every check below comes before the library call
    s.handle = None
    s.cfg = _lib.Config()
    objs = [dict(t_cam_obj=np.eye(4, dtype=np.float32), pts=np.zeros((4, 3), np.float32))] * 2
    with pytest.raises(ValueError, match="pairs only apply"):
        s.keyframe(objs, [0, 0], pairs=[1, 0])
    with pytest.raises(ValueError, match="pairs for"):
        s.keyframe(objs, [0, 0], voxels_dim=8, pairs=[-1])
    with pytest.raises(ValueError, match="modes for"):
        s.keyframe(objs, [0], voxels_dim=8)
    with pytest.raises(ValueError, match="gates for"):
        s.keyframe(objs, [0, 1], gates=[None], voxels_dim=8)


def test_mesh_word_is_the_first_pad_word_and_the_abi_matches_the_header():
    import re
    from dsp_slam_b200 import _lib
    o = _lib.ObjectOut()
    o.pad_[0] = 3
    assert o.mesh == 3 == _lib.MESH_LOST
    hdr = open(os.path.join(ROOT, "include", "dspgn.h")).read()
    for name, v in (("OFF", 0), ("DONE", 1), ("FAILED", 2), ("LOST", 3)):
        assert re.search(rf"#define DSPGN_MESH_{name} {v}\b", hdr)
        assert getattr(_lib, f"MESH_{name}") == v
    assert "int32_t mesh;" in hdr and "dspgn_keyframe_batch_meshed(" in hdr
    assert C.sizeof(_lib.MeshSpec) == 16 and _lib.MeshSpec.pair.offset == 8
    sym = {n: a for n, _, a in _lib.SYMBOLS}
    assert len(sym["dspgn_keyframe_batch_meshed"]) == 9
