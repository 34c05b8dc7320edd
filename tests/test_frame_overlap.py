"""A keyframe's detections built while the previous keyframe's objects run: the SM budget of the solver's grid-sized
launches (the persistent kernels, the per-iteration schedule's decoder launches) leaves DSPGN_FRAME_RESERVE_SMS SMs
free while a frame handle is alive, and the frame handles' streams have the greatest priority.

GPU: records and meshes are bit-identical at every budget (1, 2, 66 and all SMs, and the reserved budget); the budget
follows the live frame handles of the device, from any thread; a frame call returns while a long keyframe still runs,
with the standalone call's instances, and the keyframe then gives the blocking call's records; the plain-C caller does
the same through the C ABI.  CPU: the hook's prototype against the header, its argument checks without a device, and
the C caller compiles and links.
"""
import ctypes as C
import gc
import os
import re
import struct
import subprocess
import threading

import numpy as np
import pytest

from test_keyframe_async import _same, _stereo
from test_keyframe_batch import NATIVE, ROOT, _bits, _cfg, _new, _opt

LIDAR_CFG = dict(num_lidar_max=250, min_mask_area=1000, downsample_ratio=4.0)


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _budgets():
    from dsp_slam_b200 import _lib
    n = _num_sms()
    return [n, n - _lib.FRAME_RESERVE_SMS, 66, 2, 1]


def _forced(solver, budgets, run):
    """run() at every forced budget, then the automatic budget restored"""
    outs = []
    for k in budgets:
        assert solver.debug_sm_budget(k) == k
        outs.append(run())
    solver.debug_sm_budget(None)
    return outs


def _long_keyframe():
    """16 joint objects x 2048 points + 2048 foreground and 200 background rays with the render term: from cfg2_full's
    257 ms for 32 such objects, far longer than a frame call."""
    from dsp_slam_b200 import synth
    objs = synth.make_batch(16, 2048, 2048, 200, cls="cars", seed0=700)
    return [dict(t_cam_obj=o["t_cam_obj_init"], pts=o["pts"], rays=o["rays"], depth=o["depth"]) for o in objs]


def _same_lidar(got, want):
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert np.array_equal(a.surface_points, b.surface_points) and np.array_equal(a.T_cam_obj, b.T_cam_obj)
        assert (a.rays is None) == (b.rays is None)
        if b.rays is not None:
            assert np.array_equal(a.rays, b.rays) and np.array_equal(a.depth, b.depth)


# ---- GPU: results do not depend on the budget ------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("sdf_only", [True, False], ids=["sdf", "render"])
def test_persistent_records_are_the_same_at_every_budget(golden_dir, cfg_kitti, sdf_only):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), "tc", "persistent", sdf_only=sdf_only)
    objs = [_new(600 + k, cls="chairs" if k == 2 else "cars") for k in range(5)]
    outs = _forced(opt.solver, _budgets(), lambda: _bits(opt.solver.reconstruct(objs), len(objs)))
    for o in outs[1:]:
        assert np.array_equal(o, outs[0])


@pytest.mark.gpu
def test_gated_meshed_keyframe_is_the_same_at_every_budget(golden_dir, cfg_kitti):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), "tc", "persistent")
    s = opt.solver
    objs, modes, gates = _stereo()

    def run():
        s.keyframe_submit(objs, modes, gates, voxels_dim=32)
        return s.keyframe_wait()

    outs = _forced(s, _budgets(), run)
    assert any(m is not None for m in outs[0][1])
    for o in outs[1:]:
        _same(o, outs[0], len(objs), 32)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["simt", "tc"])
def test_per_iteration_schedule_is_the_same_at_two_budgets(golden_dir, cfg_kitti, engine):
    opt = _opt(golden_dir, _cfg(cfg_kitti, 5), engine, "launches")
    objs = [_new(620 + k) for k in range(3)]
    outs = _forced(opt.solver, [_num_sms(), 2], lambda: _bits(opt.solver.reconstruct(objs), len(objs)))
    assert np.array_equal(outs[0], outs[1])


# ---- GPU: the policy -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_budget_follows_the_live_frame_handles(golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib, synth
    from dsp_slam_b200.lidar_frame import LidarFrameBuilder
    from dsp_slam_b200.mono_frame import MonoFrameBuilder
    gc.collect()                                   # builders of earlier tests
    n, r = _num_sms(), _lib.FRAME_RESERVE_SMS
    s = _opt(golden_dir, _cfg(cfg_kitti, 5), None, None).solver
    assert s.debug_sm_budget() == n
    fr = synth.make_lidar_frame(5, 2000)
    made = []
    t = threading.Thread(target=lambda: made.append(LidarFrameBuilder(fr["K"], fr["T_cam_velo"], LIDAR_CFG, fr["img_hw"])))
    t.start()
    t.join()
    lidar = made.pop()
    assert s.debug_sm_budget() == n - r
    mf = synth.make_mono_frame(6, "redwood", 2, 10)
    mono = MonoFrameBuilder(mf["K"], mf["k1"], mf["k2"], dict(downsample_ratio=4.0), mf["img_hw"], 5)
    assert s.debug_sm_budget() == n - r
    assert s.debug_sm_budget(3) == 3                 # a forced budget wins over the automatic one
    assert s.debug_sm_budget(0) == n - r
    lidar.close()
    assert s.debug_sm_budget() == n - r
    mono.close()
    assert s.debug_sm_budget() == n
    for bad in (-1, n + 1):
        with pytest.raises(_lib.DspgnError) as e:
            s.debug_sm_budget(bad)
        assert e.value.code == _lib.E_ARG
    # in flight: E_BUSY, and the submitted call is left intact
    objs, modes, gates = _stereo()
    want = s.keyframe(objs, modes, gates)
    s.keyframe_submit(objs, modes, gates)
    cur = C.c_int32(-7)
    assert _lib.load().dspgn_debug_sm_budget(s.handle, 2, C.byref(cur)) == _lib.E_BUSY and cur.value == -7
    assert np.array_equal(_bits(s.keyframe_wait(), len(objs)), _bits(want, len(objs)))
    assert s.debug_sm_budget() == n


# ---- GPU: a frame call beside a running keyframe ---------------------------------------------------------------------
def _overlap(golden_dir, cfg_kitti, frame_call):
    """Warm the solver and the builder on the exact shapes, submit the long keyframe, run the frame call once, then
    collect.  Returns (frame call's result, keyframe still running when it returned, records, blocking records)."""
    from dsp_slam_b200.optimizer import Optimizer
    opt = Optimizer(os.path.join(golden_dir, "decoder_cars.npz"), cfg_kitti)
    s = opt.solver
    objs = _long_keyframe()
    modes = [0] * len(objs)
    frame_call()
    want = _bits(s.keyframe(objs, modes), len(objs))
    s.keyframe_submit(objs, modes)
    got = frame_call()
    running = not s.keyframe_query()
    rec = _bits(s.keyframe_wait(), len(objs))
    return got, running, rec, want


@pytest.mark.gpu
def test_lidar_frame_returns_while_the_keyframe_runs(golden_dir, cfg_kitti):
    from dsp_slam_b200 import synth
    from dsp_slam_b200.lidar_frame import LidarFrameBuilder
    fr = synth.make_lidar_frame(31, 127000)
    b = LidarFrameBuilder(fr["K"], fr["T_cam_velo"], LIDAR_CFG, fr["img_hw"])

    def call():
        return b.detections(fr["scan"], fr["dets"], fr["masks"], fr["bboxes"])

    alone = call()
    got, running, rec, want = _overlap(golden_dir, cfg_kitti, call)
    assert running, "the frame call waited for the keyframe"
    _same_lidar(got, alone)
    assert any(it.rays is not None for it in alone)
    assert np.array_equal(rec, want)
    b.close()


@pytest.mark.gpu
def test_mono_frame_returns_while_the_keyframe_runs(golden_dir, cfg_kitti):
    from dsp_slam_b200 import synth
    from dsp_slam_b200.mono_frame import MonoFrameBuilder
    f = synth.make_mono_frame(200, "freiburg", 12, 2000)
    b = MonoFrameBuilder(f["K"], f["k1"], f["k2"], dict(downsample_ratio=4.0), f["img_hw"], 15)

    def call():
        inst = b.detections(f["masks"], f["bboxes"], f["keypoints"])
        return [it.background_rays for it in inst], b.feature_points().copy()

    alone = call()
    (rays, feats), running, rec, want = _overlap(golden_dir, cfg_kitti, call)
    assert running, "the frame call waited for the keyframe"
    assert len(rays) == len(alone[0]) == 1 and np.array_equal(rays[0], alone[0][0])
    assert np.array_equal(feats, alone[1])
    assert np.array_equal(rec, want)
    b.close()


# ---- plain-C caller --------------------------------------------------------------------------------------------------
def _build_caller(tmp):
    exe = os.path.join(tmp, "overlap_caller")
    libd = os.path.join(ROOT, "dsp_slam_b200")
    subprocess.check_call(["gcc", "-O1", "-std=c11", "-Wall", "-Werror", f"-I{os.path.join(ROOT, 'include')}",
                           os.path.join(NATIVE, "overlap_caller.c"), "-o", exe, f"-L{libd}", "-ldspgn",
                           f"-Wl,-rpath,{libd}"])
    return exe


def test_overlap_caller_compiles_and_links(tmp_path):
    exe = _build_caller(str(tmp_path))
    assert subprocess.run([exe]).returncode == 2


@pytest.mark.gpu
def test_plain_c_overlap_caller_matches_python(tmp_path, golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib, synth
    from dsp_slam_b200.decoder import DecoderWeights
    from dsp_slam_b200.lidar_frame import LidarFrameBuilder, _box_matrices
    from dsp_slam_b200.optimizer import Optimizer
    exe = _build_caller(str(tmp_path))
    dec = os.path.join(golden_dir, "decoder_cars.npz")
    w = DecoderWeights.from_npz(dec)
    wp, fp, kp, op = (str(tmp_path / n) for n in ("w.bin", "frame.bin", "kf.bin", "out.bin"))
    with open(wp, "wb") as f:
        f.write(struct.pack("<3i", len(w.W), w.latent_size, w.latent_in_layer))
        for W, b in zip(w.W, w.b):
            f.write(struct.pack("<2i", *W.shape)); f.write(W.tobytes()); f.write(b.tobytes())
    fr = synth.make_lidar_frame(33, 127000)
    b = LidarFrameBuilder(fr["K"], fr["T_cam_velo"], LIDAR_CFG, fr["img_hw"])
    inst = b.detections(fr["scan"], fr["dets"], fr["masks"], fr["bboxes"])
    b.close()
    dets = fr["dets"][np.argsort(fr["dets"][:, 0]), :]
    boxes = (_lib.LidarBox * len(dets))()
    for n, d in enumerate(dets):
        _, Tov = _box_matrices(d)
        boxes[n].t_obj_velo[:] = Tov[:3].ravel().tolist()
        boxes[n].trans[:] = d[:3].tolist()
        boxes[n].size[:] = d[3:6].tolist()
        boxes[n].front = int(bool(inst[n].is_front))
    sp = _lib.LidarSpec(img_h=b.img_h, img_w=b.img_w, num_lidar_max=250, min_mask_area=1000, downsample_ratio=4)
    sp.k[:], sp.inv_k[:], sp.t_cam_velo[:] = b.K.ravel().tolist(), b.invK.ravel().tolist(), b.T_cam_velo.ravel().tolist()
    with open(fp, "wb") as f:
        f.write(bytes(sp))
        f.write(struct.pack("<3i", fr["scan"].shape[0], len(dets), fr["masks"].shape[0]))
        f.write(fr["scan"].tobytes()); f.write(bytes(boxes))
        f.write(fr["masks"].view(np.uint8).tobytes()); f.write(fr["bboxes"].astype(np.int32).tobytes())
    objs = _long_keyframe()
    with open(kp, "wb") as f:
        f.write(struct.pack("<i", len(objs)))
        for o in objs:
            f.write(struct.pack("<3i", o["pts"].shape[0], o["rays"].shape[0], o["depth"].shape[0]))
            for a in (o["t_cam_obj"], o["pts"], o["rays"], o["depth"]):
                f.write(np.ascontiguousarray(a, np.float32).tobytes())
    r = subprocess.run([exe, wp, fp, kp, op], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    raw = open(op, "rb").read()
    k = len(dets)
    budget, running = struct.unpack_from("<2i", raw, 0)
    assert budget == _num_sms() - _lib.FRAME_RESERVE_SMS
    hdr = np.frombuffer(raw, np.int32, 4 * k, 8).reshape(k, 4)
    assert [h[0] for h in hdr] == [it.num_surface_points for it in inst]
    assert [h[1] for h in hdr] == [-1 if it.rays is None else it.rays.shape[0] for it in inst]
    npts, nr = int(hdr[:, 0].sum()), int(np.maximum(hdr[:, 1], 0).sum())
    o = 8 + 16 * k
    pts = np.frombuffer(raw, np.float32, 3 * npts, o).reshape(-1, 3); o += 12 * npts
    depth = np.frombuffer(raw, np.float32, npts, o); o += 4 * npts
    rays = np.frombuffer(raw, np.float32, 3 * nr, o).reshape(-1, 3); o += 12 * nr
    assert np.array_equal(pts, np.concatenate([it.surface_points for it in inst]))
    assert np.array_equal(depth, pts[:, 2])
    assert np.array_equal(rays, np.concatenate([it.rays for it in inst if it.rays is not None]))
    rec = np.frombuffer(raw, np.uint32, len(objs) * _lib.RESULT_FLOATS, o).reshape(len(objs), -1)
    assert o + rec.nbytes == len(raw)
    opt = Optimizer(dec, cfg_kitti)
    want = _bits(opt.solver.keyframe(objs, [0] * len(objs)), len(objs))
    assert np.array_equal(rec, want)
    assert f"keyframe running when the frame returned: {running}" in r.stdout


# ---- no GPU ----------------------------------------------------------------------------------------------------------
def test_sm_budget_hook_prototype_and_argument_checks():
    from dsp_slam_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "dspgn.h")).read()
    m = re.search(r"int dspgn_debug_sm_budget\(([^)]*)\);", hdr)
    assert m and [a.strip() for a in m.group(1).split(",")] == ["DspgnSolver* s", "int n", "int32_t* current"]
    sym = {n: (r, a) for n, r, a in _lib.SYMBOLS}
    assert sym["dspgn_debug_sm_budget"] == (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int32)])
    d = re.search(r"#define DSPGN_FRAME_RESERVE_SMS (\d+)", hdr)
    assert d and int(d.group(1)) == _lib.FRAME_RESERVE_SMS and 1 <= _lib.FRAME_RESERVE_SMS < 66
    lib = _lib.load()
    cur = C.c_int32(-7)
    h = C.cast(C.create_string_buffer(64), C.c_void_p)      # never dereferenced: the arguments fail first
    assert lib.dspgn_debug_sm_budget(None, 0, C.byref(cur)) == _lib.E_ARG
    assert lib.dspgn_debug_sm_budget(None, 4, None) == _lib.E_ARG
    assert lib.dspgn_debug_sm_budget(h, -1, C.byref(cur)) == _lib.E_ARG
    assert cur.value == -7
