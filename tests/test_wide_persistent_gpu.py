"""The wide tensor-core engine (engine="tc_wide") on the persistent schedule (k_wide_persistent) against its
per-iteration schedule (k_wide_wgmma, k_ray_scan, k_solve launches): every record word and every mesh of the same call
is bit-identical under schedule="persistent" and schedule="launches", on DeepSDF's own 8 x 512 decoder
(tests/wide_fixtures.py) with chairs as a second class.  Covers the single-object calls, a batch larger than the grid,
the gated, meshed stereo keyframe (blocking and submitted), the mono pair rule, a mixed-width solver, a stop, and that the
persistent kernel really runs (one launch for all iterations).
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
STATUS_WORD, ITERS_WORD = 81, 84
_WIDE = {}


@pytest.fixture(scope="module", autouse=True)
def _wide_files(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("wide_decoders"))
    _WIDE["wide"] = WF.write("wide", d)


def _path(golden_dir, name):
    return _WIDE[name] if name in _WIDE else os.path.join(golden_dir, f"decoder_{name}.npz")


def _opt(golden_dir, cfg, schedule, name="wide", extra=("chairs",), **kw):
    from dsp_slam_b200 import _lib
    from dsp_slam_b200.optimizer import Optimizer
    opt = Optimizer(_path(golden_dir, name), cfg, extra_decoders=[_path(golden_dir, e) for e in extra], engine="tc_wide",
                    schedule=schedule, **kw)
    assert opt.solver.engine == _lib.ENGINE_TC_WIDE
    return opt


def _both(make, call):
    """call(opt) under both schedules -> {schedule: result}"""
    out = {}
    for sch in SCHEDULES:
        opt = make(sch)
        out[sch] = call(opt)
        opt.solver.close()
    return out


def _same(got, what):
    a, b = got["persistent"], got["launches"]
    assert a.shape == b.shape, what
    assert np.array_equal(a, b), (what, np.argwhere(a != b)[:8])


def test_single_object_calls(golden_dir, cfg_kitti):
    """reconstruct_object on recon_wide.npz and estimate_pose_cam_obj on pose_only_wide.npz (10 pose-only iterations:
    the inlier cut at iteration 4 is taken) are bit-identical across the schedules."""
    d = np.load(os.path.join(golden_dir, "recon_wide.npz"))
    p = np.load(os.path.join(golden_dir, "pose_only_wide.npz"))
    cfg = copy.deepcopy(cfg_kitti)
    cfg["optimizer"]["pose_only_optim"]["num_iterations"] = 10

    def call(opt):
        r = opt.reconstruct_object(np.asfortranarray(d["in_t_cam_obj"]), np.asfortranarray(d["in_pts"]),
                                   np.asfortranarray(d["in_rays"]), d["in_depth"])
        T = opt.estimate_pose_cam_obj(p["in_t_co_se3"].copy(), float(p["in_scale"]), p["in_pts"], p["in_code"])
        return np.concatenate([np.asarray(r.t_cam_obj, np.float32).ravel(), np.asarray(r.code, np.float32).ravel(),
                               np.float32([r.loss, r.is_good]), np.asarray(T, np.float32).ravel()]).view(np.uint32)

    got = _both(lambda s: _opt(golden_dir, cfg, s, extra=()), call)
    _same(got, "single-object calls")


@pytest.mark.parametrize("sdf_only", [False, True])
def test_batch_larger_than_the_grid(golden_dir, cfg_kitti, sdf_only):
    """140 objects (more than the 132 CTAs of an H100) of 600 points each (10 tiles of 64 rows), cars and chairs, with
    and without the render term: every record bit-identical.  Row counters: the SDF rows are counted alike.  With the
    render term each schedule counts as the 128-row engine's do: the per-iteration schedule every ray sample it decodes
    (n_rays x D per iteration) and no band rows, the persistent kernel what the reference decodes, V samples inside the
    unit sphere (its ray tiles cover only those hulls) and the band rows (fwd + bwd)."""
    import torch
    n = torch.cuda.get_device_properties(0).multi_processor_count + 8
    objs = [_new(2000 + i, n_pts=600, cls="cars" if i % 3 else "chairs") for i in range(n)]
    cfg = copy.deepcopy(cfg_kitti)
    cfg["optimizer"]["joint_optim"]["num_iterations"] = 5
    got, ctr = {}, {}
    for sch in SCHEDULES:
        opt = _opt(golden_dir, cfg, sch, sdf_only=sdf_only)
        got[sch] = _bits(opt.solver.reconstruct(objs), n)
        ctr[sch] = opt.solver.counters()
        opt.solver.close()
    _same(got, "batch")
    assert (got["persistent"].view(np.int32)[:, STATUS_WORD] == 0).sum() >= n // 2
    p, l = ctr["persistent"], ctr["launches"]
    assert l["rows_fwd_bwd"] == 5 * 600 * n
    if sdf_only:
        assert p["rows_fwd_bwd"] == l["rows_fwd_bwd"] and p["rows_fwd_only"] == l["rows_fwd_only"] == 0, (p, l)
    else:
        samples = 5 * sum(len(o["rays"]) for o in objs) * cfg["optimizer"]["num_depth_samples"]
        assert l["rows_fwd_only"] == samples, (l, samples)
        assert 0 < p["rows_fwd_only"] < samples, (p, samples)           # V <= n_rays x D per iteration
        assert p["rows_fwd_bwd"] > l["rows_fwd_bwd"], (p, l)              # + the band rows of every iteration


def test_gated_meshed_stereo_keyframe(golden_dir, cfg_kitti):
    """The stereo keyframe of test_keyframe_mesh (kept and rejected gated objects, meshes of the new ones): records,
    gate and mesh words and meshes bit-identical across the schedules, blocking and submitted."""
    from dsp_slam_b200 import _lib
    objs, modes, gates = _stereo_keyframe()
    n, dim = len(objs), 16

    def call(opt):
        got, meshes, words = _check_call(opt.solver, objs, modes, gates, dim)
        opt.solver.keyframe_submit(objs, modes, gates, voxels_dim=dim)
        sub, sub_meshes = opt.solver.keyframe_wait()
        assert np.array_equal(_bits(sub, n), got)
        flat = [got.ravel()]
        for m, s in zip(meshes, sub_meshes):
            assert (m is None) == (s is None)
            if m is not None:
                assert np.array_equal(m[0].view(np.uint32), s[0].view(np.uint32)) and np.array_equal(m[1], s[1])
                flat += [m[0].view(np.uint32).ravel(), m[1].view(np.uint32).ravel()]
        return np.concatenate(flat)

    got = _both(lambda s: _opt(golden_dir, _cfg(cfg_kitti, 5), s), call)
    _same(got, "stereo keyframe")
    rec = got["persistent"][:n * _lib.RESULT_FLOATS].reshape(n, _lib.RESULT_FLOATS).view(np.int32)
    gw = rec[:, 85]
    assert (gw == _lib.GATE_KEPT).any() and (gw == _lib.GATE_REJECTED).any()


def test_mono_pairs(golden_dir, cfg_kitti):
    """reconstruct_mono_batch with flipped hypotheses: the kept results, flags and meshes are bit-identical."""
    from test_keyframe_gate import _moved
    objs = [_new(3100 + i, cls="cars" if i % 2 == 0 else "chairs") for i in range(4)]
    mono = [dict(o, t_cam_obj_flipped=_moved(o["t_cam_obj"], angle=np.pi)) if i < 3 else o for i, o in enumerate(objs)]
    cfg = copy.deepcopy(cfg_kitti)
    cfg["optimizer"]["joint_optim"]["num_iterations"] = 5

    def call(opt):
        res = opt.reconstruct_mono_batch(mono, voxels_dim=16)
        flat = []
        for r in res:
            flat.append(np.uint32([bool(r["flipped"]), bool(r.is_good)]))
            flat += [np.asarray(r.t_cam_obj, np.float32).view(np.uint32).ravel(), np.asarray(r.code, np.float32).view(np.uint32).ravel(),
                     np.float32([r.loss]).view(np.uint32)]
            if r.get("vertices") is not None:
                flat += [np.asarray(r["vertices"], np.float32).view(np.uint32).ravel(), np.asarray(r["faces"]).view(np.uint32).ravel()]
        return np.concatenate(flat)

    got = _both(lambda s: _opt(golden_dir, cfg, s), call)
    _same(got, "mono pairs")


def test_mixed_width_solver(golden_dir, cfg_kitti):
    """cars as class 0 and the wide decoder as class 1 on the one engine: records bit-identical across the schedules."""
    from dsp_slam_b200 import _lib
    objs = [_new(971), dict(_new(972), class_id=1), _tracked(973), dict(_tracked(974), class_id=1), dict(_new(975), class_id=1)]
    modes = [_lib.MODE_JOINT, _lib.MODE_JOINT, _lib.MODE_POSE, _lib.MODE_POSE, _lib.MODE_JOINT]
    got = _both(lambda s: _opt(golden_dir, _cfg(cfg_kitti, 5), s, "cars", extra=("wide",)),
                lambda opt: _bits(opt.solver.keyframe(objs, modes), len(objs)))
    _same(got, "mixed width")
    assert (got["persistent"].view(np.int32)[:, STATUS_WORD] == 0).sum() >= 4


def test_stop_at_iteration_3(golden_dir, cfg_kitti):
    """A stop raised by the device at iteration 3 of a joint object: its stopped record and every other record are
    bit-identical across the schedules."""
    from dsp_slam_b200 import _lib
    objs = [_new(961), _new(962), _tracked(963)]
    modes = [_lib.MODE_JOINT, _lib.MODE_JOINT, _lib.MODE_POSE]

    def call(opt):
        opt.solver.debug_stop_at(1, 3)
        return _bits(opt.solver.keyframe(objs, modes), len(objs))

    got = _both(lambda s: _opt(golden_dir, _cfg(cfg_kitti, 5), s), call)
    _same(got, "stopped call")
    gi = got["persistent"].view(np.int32)
    assert gi[1, STATUS_WORD] == _lib.ST_STOPPED and gi[1, ITERS_WORD] == 4


def test_one_launch_for_every_iteration(golden_dir, cfg_kitti):
    """The persistent schedule really runs k_wide_persistent: a joint run enqueues as many kernels for 10 iterations
    as for 5, while the per-iteration schedule's launches grow with the iteration count."""
    o = _new(990)
    launches = {}
    for sch in SCHEDULES:
        for iters in (5, 10):
            cfg = copy.deepcopy(cfg_kitti)
            cfg["optimizer"]["joint_optim"]["num_iterations"] = iters
            opt = _opt(golden_dir, cfg, sch)
            opt.solver.reconstruct([o])
            launches[sch, iters] = opt.solver.counters()["kernel_launches"]
            opt.solver.close()
    assert launches["persistent", 5] == launches["persistent", 10], launches
    assert launches["launches", 10] > launches["launches", 5], launches
