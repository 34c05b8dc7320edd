"""The fp32 SIMT engine (engine="simt") on the persistent schedule (k_simt_persistent) against its per-iteration schedule
(k_decoder_simt, k_ray_scan, k_solve launches): every record word (pose, code, loss, status, V, m, iterations, gate and
mesh words) and every mesh of the same call is bit-identical under schedule="persistent" and schedule="launches".  Covers
cars + chairs, the LayerNorm / xyz_in_all / use_tanh / two-latent_in variant, DeepSDF's 8 x 512 network and its 512-wide
LayerNorm variant (tests/wide_fixtures.py), a mixed-width solver, SDF-only and pose-only runs, gated and meshed
keyframes (blocking and submitted), a stop, D = 2 and D = 64 at 8192 rays, more than 1024 objects, forced SM budgets and
the row and launch counters.
"""
import copy
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import wide_fixtures as WF  # noqa: E402
from test_keyframe_batch import _bits, _cfg, _new, _tracked  # noqa: E402
from test_keyframe_mesh import _check_call, _stereo_keyframe  # noqa: E402

pytestmark = pytest.mark.gpu

SCHEDULES = ("persistent", "launches")
V_WORD, STATUS_WORD, ITERS_WORD, GATE_WORD, MESH_WORD = 82, 81, 84, 85, 86
_FILES = {}


@pytest.fixture(scope="module", autouse=True)
def _wide_files(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("wide_decoders"))
    for name in ("wide", "wide_variant"):
        _FILES[name] = WF.write(name, d)


def _path(golden_dir, name):
    return _FILES[name] if name in _FILES else os.path.join(golden_dir, f"decoder_{name}.npz")


def _opt(golden_dir, cfg, schedule, name="cars", extra=("chairs",), **kw):
    from dsp_slam_b200 import _lib
    from dsp_slam_b200.optimizer import Optimizer
    opt = Optimizer(_path(golden_dir, name), cfg, extra_decoders=[_path(golden_dir, e) for e in extra], engine="simt",
                    schedule=schedule, **kw)
    assert opt.solver.engine == _lib.ENGINE_SIMT
    return opt


def _both(make, call):
    """call(opt) under both schedules -> ({schedule: result}, {schedule: counters})"""
    out, ctr = {}, {}
    for sch in SCHEDULES:
        opt = make(sch)
        out[sch] = call(opt)
        ctr[sch] = opt.solver.counters()
        opt.solver.close()
    return out, ctr


def _same(got, what):
    a, b = got["persistent"], got["launches"]
    assert a.shape == b.shape, what
    assert np.array_equal(a, b), (what, np.argwhere(a != b)[:8])


def _ragged(cls=(0, 1)):
    """A ragged joint / pose-only batch over classes `cls` with the render soft failures: a new object without rays and
    one whose rays all miss it."""
    from dsp_slam_b200 import _lib
    c0, c1 = cls[0], cls[-1]
    no_rays = dict(_new(411), class_id=c1)
    no_rays["rays"] = np.zeros((0, 3), np.float32); no_rays["depth"] = np.zeros(0, np.float32)
    miss = dict(_new(412), class_id=c0)
    miss["rays"] = np.asfortranarray(np.tile(np.array([[3.0, 3.0, 1.0]], np.float32), (40, 1)))
    miss["depth"] = np.zeros(0, np.float32)
    objs = [dict(_tracked(401), class_id=c0), dict(_new(402), class_id=c0), dict(_tracked(403, 150), class_id=c1),
            dict(_new(404, 180, 90, 30), class_id=c1), dict(_new(405, 250, 250, 200), class_id=c0), no_rays, miss,
            dict(_tracked(406, 64, outliers=6), class_id=c1), dict(_new(407, 65, 64, 10), class_id=c0)]
    modes = [1, 0, 1, 0, 0, 0, 0, 1, 0]
    return objs, [_lib.MODE_POSE if m else _lib.MODE_JOINT for m in modes]


DECODERS = [("cars", ("chairs",)), ("variant", ()), ("wide", ()), ("wide_variant", ()), ("cars", ("wide",))]


@pytest.mark.parametrize("name,extra", DECODERS, ids=["cars+chairs", "variant", "wide", "wide_variant", "cars+wide"])
def test_joint_render_batch(golden_dir, cfg_kitti, name, extra):
    """Joint runs with the render term and pose-only runs in one ragged call: every record bit-identical; one launch of
    the persistent kernel (+ k_init and the readback's) serves every iteration."""
    from dsp_slam_b200 import _lib
    objs, modes = _ragged((0, 1) if extra else (0,))
    got, ctr = _both(lambda s: _opt(golden_dir, _cfg(cfg_kitti, 5), s, name, extra),
                     lambda opt: _bits(opt.solver.keyframe(objs, modes), len(objs)))
    _same(got, name)
    st = got["persistent"].view(np.int32)[:, STATUS_WORD]
    assert st[5] == _lib.ST_RENDER_FEW and st[6] == _lib.ST_RENDER_FEW, st
    assert (st == 0).sum() >= 5, st
    assert ctr["persistent"]["kernel_launches"] <= 3, ctr
    assert ctr["launches"]["kernel_launches"] > 10, ctr


@pytest.mark.parametrize("pose_iters", [5, 7])
@pytest.mark.parametrize("sdf_only", [False, True])
def test_sdf_only_and_pose_only(golden_dir, cfg_kitti, sdf_only, pose_iters):
    """SDF-only joint runs with pose-only ones, 5 and 7 pose-only iterations (7: the inlier cut of iteration 4 applies):
    bit-identical records; the SDF rows are counted alike."""
    objs, modes = _ragged()
    got, ctr = _both(lambda s: _opt(golden_dir, _cfg(cfg_kitti, pose_iters), s, sdf_only=sdf_only),
                     lambda opt: _bits(opt.solver.keyframe(objs, modes), len(objs)))
    _same(got, "sdf_only" if sdf_only else "pose-only")
    pose = [o for o, m in zip(objs, modes) if m]
    got_p, _ = _both(lambda s: _opt(golden_dir, _cfg(cfg_kitti, pose_iters), s),
                     lambda opt: _bits(opt.solver.estimate_pose(pose), len(pose)))
    _same(got_p, "estimate_pose")
    if sdf_only:
        p, l = ctr["persistent"], ctr["launches"]
        assert p["rows_fwd_bwd"] == l["rows_fwd_bwd"] and p["rows_fwd_only"] == l["rows_fwd_only"] == 0, (p, l)


def test_keyframe_batch_gated_meshed_and_async(golden_dir, cfg_kitti):
    """The gated, meshed stereo keyframe of test_keyframe_mesh (kept and rejected gated objects, meshes of the new
    ones): records, gate and mesh words and meshes bit-identical across the schedules, blocking and submitted; the
    persistent kernel wakes the rejected slots in its own launch, and the submit adds no host sync."""
    from dsp_slam_b200 import _lib
    objs, modes, gates = _stereo_keyframe()
    n, dim = len(objs), 16
    launches = {}

    def call(opt):
        got, meshes, words = _check_call(opt.solver, objs, modes, gates, dim)
        opt.solver.keyframe(objs, modes, gates)
        launches[opt.schedule_name] = opt.solver.counters()["kernel_launches"]
        opt.solver.keyframe_submit(objs, modes, gates, voxels_dim=dim)      # warm: the solver's buffers fit this call
        opt.solver.keyframe_wait()
        before = opt.solver.host_syncs()
        opt.solver.keyframe_submit(objs, modes, gates, voxels_dim=dim)
        assert opt.solver.host_syncs() == before
        sub, sub_meshes = opt.solver.keyframe_wait()
        assert np.array_equal(_bits(sub, n), got)
        flat = [got.ravel()]
        for m, s in zip(meshes, sub_meshes):
            assert (m is None) == (s is None)
            if m is not None:
                assert np.array_equal(m[0].view(np.uint32), s[0].view(np.uint32)) and np.array_equal(m[1], s[1])
                flat += [m[0].view(np.uint32).ravel(), m[1].view(np.uint32).ravel()]
        return np.concatenate(flat)

    def make(s):
        opt = _opt(golden_dir, _cfg(cfg_kitti, 5), s)
        opt.schedule_name = s
        return opt

    got, _ = _both(make, call)
    _same(got, "stereo keyframe")
    rec = got["persistent"][:n * _lib.RESULT_FLOATS].reshape(n, _lib.RESULT_FLOATS).view(np.int32)
    gw = rec[:, GATE_WORD]
    assert (gw == _lib.GATE_KEPT).sum() >= 1 and (gw == _lib.GATE_REJECTED).sum() >= 3, gw
    assert (rec[:, MESH_WORD] == _lib.MESH_DONE).any()
    assert launches["persistent"] <= 2 < launches["launches"], launches


def test_mono_pair_meshes(golden_dir, cfg_kitti):
    """reconstruct_mono_batch with flipped hypotheses: kept results, flags and meshes bit-identical."""
    from test_keyframe_gate import _moved
    objs = [_new(3100 + i, cls="cars" if i % 2 == 0 else "chairs") for i in range(4)]
    mono = [dict(o, t_cam_obj_flipped=_moved(o["t_cam_obj"], angle=np.pi)) if i < 3 else o for i, o in enumerate(objs)]
    cfg = copy.deepcopy(cfg_kitti)
    cfg["optimizer"]["joint_optim"]["num_iterations"] = 5

    def call(opt):
        flat = []
        for r in opt.reconstruct_mono_batch(mono, voxels_dim=16):
            flat.append(np.uint32([bool(r["flipped"]), bool(r.is_good)]))
            flat += [np.asarray(r.t_cam_obj, np.float32).view(np.uint32).ravel(),
                     np.asarray(r.code, np.float32).view(np.uint32).ravel(), np.float32([r.loss]).view(np.uint32)]
            if r.get("vertices") is not None:
                flat += [np.asarray(r["vertices"], np.float32).view(np.uint32).ravel(), np.asarray(r["faces"]).view(np.uint32).ravel()]
        return np.concatenate(flat)

    got, _ = _both(lambda s: _opt(golden_dir, cfg, s), call)
    _same(got, "mono pairs")


def test_stop_equals_the_shorter_call(golden_dir, cfg_kitti):
    """debug_stop_at(1, 3) on the persistent kernel: object 1 ends STOPPED after 4 iterations.  Every STOPPED record is,
    status word aside, the record of the unstopped call at num_iterations = its iterations; every other record is the
    unstopped call's.  (Other objects see the stop at their own next solve, wherever they are.)"""
    from dsp_slam_b200 import _lib
    objs, modes = [_new(961), _new(962), _tracked(963)], [_lib.MODE_JOINT, _lib.MODE_JOINT, _lib.MODE_POSE]
    runs = {}

    def run(iters, stop=False):
        if (iters, stop) not in runs:
            cfg = _cfg(cfg_kitti, 5)
            cfg["optimizer"]["joint_optim"]["num_iterations"] = iters
            opt = _opt(golden_dir, cfg, "persistent")
            if stop:
                opt.solver.debug_stop_at(1, 3)
            runs[iters, stop] = _bits(opt.solver.keyframe(objs, modes), len(objs))
            opt.solver.close()
        return runs[iters, stop]

    stopped, full = run(10, True), run(10, False)
    si = stopped.view(np.int32)
    assert si[1, STATUS_WORD] == _lib.ST_STOPPED and si[1, ITERS_WORD] == 4
    for i in range(len(objs)):
        if si[i, STATUS_WORD] != _lib.ST_STOPPED:
            assert np.array_equal(stopped[i], full[i]), (i, np.flatnonzero(stopped[i] != full[i])[:8])
            continue
        assert modes[i] == _lib.MODE_JOINT, i
        k = int(si[i, ITERS_WORD])
        a, b = stopped[i].copy(), run(k)[i].copy()
        a[STATUS_WORD] = b[STATUS_WORD] = 0
        assert np.array_equal(a, b), (i, k, np.flatnonzero(a != b)[:8])


@pytest.mark.parametrize("D,n_rays", [(2, 300), (64, 8192)])
def test_depth_samples_and_ray_count(golden_dir, cfg_kitti, D, n_rays):
    """D = 2, and D = 64 with 8192 rays (the most range words a ray-sample tile stages): records bit-identical."""
    from dsp_slam_b200 import synth
    cfg = copy.deepcopy(cfg_kitti)
    cfg["optimizer"]["num_depth_samples"] = D
    cfg["optimizer"]["joint_optim"]["num_iterations"] = 3
    n_fg = min(n_rays, 6000)
    o = synth.make_object(5100 + D, 300, n_fg, n_rays - n_fg)
    objs = [dict(t_cam_obj=o["t_cam_obj_init"], pts=o["pts"], rays=o["rays"], depth=o["depth"]), _new(5200)]
    assert len(objs[0]["rays"]) == n_rays
    got, ctr = _both(lambda s: _opt(golden_dir, cfg, s, extra=()),
                     lambda opt: _bits(opt.solver.reconstruct(objs), len(objs)))
    _same(got, f"D={D}")
    samples = 3 * sum(len(x["rays"]) for x in objs) * D
    assert ctr["launches"]["rows_fwd_only"] == samples
    # D = 2 samples only the two ends of each depth range, at or outside the unit sphere: none lies inside
    assert (D == 2 or ctr["persistent"]["rows_fwd_only"] > 0) and ctr["persistent"]["rows_fwd_only"] < samples, ctr


def test_more_than_1024_objects(golden_dir, cfg_kitti):
    """1030 objects (two resident chunks) with the render term: records bit-identical."""
    from dsp_slam_b200 import _lib
    objs = [_new(7000 + i, n_pts=40, n_fg=16, n_bg=8, cls="cars" if i % 2 else "chairs") if i % 3 else _tracked(7000 + i, 40, outliers=4)
            for i in range(1030)]
    modes = [_lib.MODE_POSE if i % 3 == 0 else _lib.MODE_JOINT for i in range(len(objs))]
    got, _ = _both(lambda s: _opt(golden_dir, _cfg(cfg_kitti, 5), s),
                   lambda opt: _bits(opt.solver.keyframe(objs, modes), len(objs)))
    _same(got, "1030 objects")


def test_forced_sm_budgets(golden_dir, cfg_kitti):
    """The persistent kernel on every SM, 64 and 5 SMs: the same records as the per-iteration schedule."""
    objs, modes = _ragged()
    ref = None
    for sch, budget in (("launches", 0), ("persistent", 0), ("persistent", 64), ("persistent", 5)):
        opt = _opt(golden_dir, _cfg(cfg_kitti, 7), sch)
        n_sms = opt.solver.debug_sm_budget(budget)
        assert n_sms == budget or budget == 0
        out = _bits(opt.solver.keyframe(objs, modes), len(objs))
        opt.solver.close()
        if ref is None:
            ref = out
        assert np.array_equal(out, ref), (sch, budget, np.argwhere(out != ref)[:8])


def test_row_counters(golden_dir, cfg_kitti):
    """One joint iteration with the render term: the persistent kernel decodes exactly the V samples inside the unit
    sphere (the records' V words), fewer than the n_rays x D the per-iteration schedule decodes; the SDF rows are counted
    alike in a pose-only run."""
    objs = [_new(8100 + i, cls="cars" if i % 2 else "chairs") for i in range(6)]
    cfg = copy.deepcopy(cfg_kitti)
    cfg["optimizer"]["joint_optim"]["num_iterations"] = 1
    got, ctr = _both(lambda s: _opt(golden_dir, cfg, s), lambda opt: _bits(opt.solver.reconstruct(objs), len(objs)))
    _same(got, "one iteration")
    V = got["persistent"].view(np.int32)[:, V_WORD].astype(np.int64)
    samples = sum(len(o["rays"]) for o in objs) * cfg["optimizer"]["num_depth_samples"]
    assert ctr["persistent"]["rows_fwd_only"] == V.sum() < samples, (ctr, V.sum(), samples)
    assert ctr["launches"]["rows_fwd_only"] == samples
    pose = [_tracked(8200 + i) for i in range(4)]
    _, ctr = _both(lambda s: _opt(golden_dir, _cfg(cfg_kitti, 5), s), lambda opt: opt.solver.estimate_pose(pose))
    assert ctr["persistent"]["rows_fwd_bwd"] == ctr["launches"]["rows_fwd_bwd"] == 5 * 200 * 4, ctr
    assert ctr["persistent"]["kernel_launches"] <= 3, ctr


def test_auto_schedule_runs_the_persistent_kernel(golden_dir, cfg_kitti):
    """engine="simt" with the default schedule: a joint call takes at most 3 launches, for 5 and for 10 iterations."""
    o = _new(990)
    for iters in (5, 10):
        cfg = copy.deepcopy(cfg_kitti)
        cfg["optimizer"]["joint_optim"]["num_iterations"] = iters
        opt = _opt(golden_dir, cfg, None)
        opt.solver.reconstruct([o])
        assert opt.solver.counters()["kernel_launches"] <= 3, iters
        opt.solver.close()
