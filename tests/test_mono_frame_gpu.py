"""A monocular keyframe's detection built on the H100 (DspgnMonoFrame): bit for bit against the golden made with the
unmodified reference and cv2, against the numpy oracle on full-size seeded frames, through the drop-in MonoSequence,
on a caller's stream, and as the background rays of reconstruct_mono_batch."""
import ctypes as C
import os

import numpy as np
import pytest

from test_mono_frame_cpu import GOLDEN, golden_frames

pytestmark = pytest.mark.gpu


def builder(K, k1, k2, alpha, hw, e):
    from dsp_slam_b200.mono_frame import MonoFrameBuilder
    return MonoFrameBuilder(K, k1, k2, dict(downsample_ratio=float(alpha)), hw, e)


def test_device_equals_golden():
    for f in golden_frames(np.load(GOLDEN)):
        b = builder(f["K"], f["k1"], f["k2"], f["alpha"], f["hw"], f["erosion"])
        if f["raised"]:
            with pytest.raises(ValueError):
                b.detections(f["masks"], f["bboxes"], f["kp"])
            assert b.last.mask == f["mask_index"] and b.last.n_rays == -1
        else:
            got = b.detections(f["masks"], f["bboxes"], f["kp"])
            assert len(got) == f["n_inst"]
            if got:
                it = got[0]
                assert np.shares_memory(it.bbox, f["bboxes"]) and np.array_equal(it.bbox, f["bboxes"][f["mask_index"]])
                assert it.mask.dtype == np.float32 and np.array_equal(it.mask, f["masks"][f["mask_index"]] * np.float32(255))
                assert it.background_rays.dtype == np.float32
                assert np.array_equal(it.background_rays, f["background_rays"])
        if f["feature_idx"] is None:
            assert b.feature_points().size == 0
        else:
            assert np.array_equal(b.feature_points(), f["feature_idx"])


@pytest.mark.parametrize("seed,camera,n_masks,e", [(1, "redwood", 8, 5), (2, "redwood", 16, 15), (3, "freiburg", 12, 5),
                                                   (4, "freiburg", 16, 15)])
def test_device_equals_oracle_full_size(seed, camera, n_masks, e):
    from dsp_slam_b200 import synth
    from oracle import mono_frame as O
    f = synth.make_mono_frame(seed, camera, n_masks)
    invK = np.linalg.inv(f["K"])
    for alpha in (4, 1):
        b = builder(f["K"], f["k1"], f["k2"], alpha, f["img_hw"], e)
        want = O.detection(f["masks"], f["bboxes"], f["K"], invK, f["k1"], f["k2"], alpha, *f["img_hw"])
        want_fp = O.feature_points(f["masks"][want["mask_index"]], f["keypoints"], e)
        for _ in range(2):                                    # repeated runs are bit-identical
            got = b.detections(f["masks"], f["bboxes"], f["keypoints"])
            assert b.last.mask == want["mask_index"] and b.last.n_nonsurface == want["n_nonsurface"]
            assert np.array_equal(got[0].background_rays, want["background_rays"])
            assert np.array_equal(b.feature_points(), want_fp)
        assert want_fp.size >= 20 and want["background_rays"].shape[0] == 200


def test_set_stream():
    import torch
    from dsp_slam_b200 import synth
    f = synth.make_mono_frame(5, "freiburg", 10)
    b = builder(f["K"], f["k1"], f["k2"], 4, f["img_hw"], 10)
    a = b.detections(f["masks"], f["bboxes"], f["keypoints"])[0].background_rays
    fa = b.feature_points().copy()
    s = torch.cuda.Stream()
    b.set_stream(s.cuda_stream)
    g = b.detections(f["masks"], f["bboxes"], f["keypoints"])[0].background_rays
    assert np.array_equal(a, g) and np.array_equal(fa, b.feature_points())
    b.set_stream(0)
    g = b.detections(f["masks"], f["bboxes"], f["keypoints"])[0].background_rays
    assert np.array_equal(a, g)


def test_misuse_returns_e_arg_and_enqueues_nothing():
    from dsp_slam_b200 import _lib, synth
    lib = _lib.load()
    f = synth.make_mono_frame(6, "redwood", 8)
    b = builder(f["K"], f["k1"], f["k2"], 4, f["img_hw"], 5)
    ref = b.detections(f["masks"], f["bboxes"], f["keypoints"])[0].background_rays
    ref_fp = b.feature_points().copy()
    m8 = f["masks"].view(np.uint8)
    bb = f["bboxes"].astype(np.int32)
    kp = np.ascontiguousarray(f["keypoints"])
    mp, bp, kpp = m8.ctypes.data_as(C.POINTER(C.c_uint8)), bb.ctypes.data_as(C.POINTER(C.c_int32)), kp.ctypes.data_as(_lib._FP)
    out = _lib.MonoOut()
    H, W = f["img_hw"]
    bad = [(mp, bp, 65, kpp, 10), (mp, bp, -1, kpp, 10), (None, bp, 8, kpp, 10), (mp, None, 8, kpp, 10),
           (mp, bp, 8, None, 10), (mp, bp, 8, kpp, -1), (mp, bp, 8, kpp, (1 << 20) + 1)]
    for args in bad:
        assert lib.dspgn_mono_frame_run(b._h, *args, C.byref(out)) == _lib.E_ARG
    assert lib.dspgn_mono_frame_run(b._h, mp, bp, 8, kpp, 10, None) == _lib.E_ARG
    for row in ([50, 10, 40, 20], [0, 0, W + 1, 20], [0, 30, 10, 20], [-1, 0, 10, 10], [0, 0, 10, H + 1]):
        bb_bad = bb.copy()
        bb_bad[3] = row
        assert lib.dspgn_mono_frame_run(b._h, mp, bb_bad.ctypes.data_as(C.POINTER(C.c_int32)), 8, kpp, 10,
                                        C.byref(out)) == _lib.E_ARG
    for pt in ([-1.0, 5.0], [W, 5.0], [5.0, H + 0.5], [np.nan, 5.0], [5.0, -np.inf]):
        kb = kp.copy()
        kb[7] = pt
        assert lib.dspgn_mono_frame_run(b._h, mp, bp, 8, kb.ctypes.data_as(_lib._FP), kb.shape[0], C.byref(out)) == _lib.E_ARG
    # the last good run's results are untouched
    rays = np.empty_like(ref)
    fp = np.empty_like(ref_fp)
    assert lib.dspgn_mono_frame_results(b._h, rays.ctypes.data_as(_lib._FP), fp.ctypes.data_as(C.POINTER(C.c_int32))) == 0
    assert np.array_equal(rays, ref) and np.array_equal(fp, ref_fp)
    sp = _lib.MonoSpec(img_h=480, img_w=640, downsample_ratio=4, mask_erosion=5)
    sp.k[:] = f["K"].ravel().tolist()
    h = C.c_void_p()
    for k, v in (("downsample_ratio", 0), ("img_h", 4097), ("img_w", 0), ("mask_erosion", 64), ("mask_erosion", -1)):
        s2 = _lib.MonoSpec.from_buffer_copy(sp)
        setattr(s2, k, v)
        assert lib.dspgn_mono_frame_create(C.byref(s2), 0, C.byref(h)) == _lib.E_ARG
    with pytest.raises(TypeError):
        b.detections(f["masks"].astype(np.uint8), f["bboxes"])


def test_dropin_sequence_on_files(tmp_path, monkeypatch, capsys):
    cv2 = pytest.importorskip("cv2")
    import torch
    root = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
    monkeypatch.syspath_prepend(os.path.join(root, "integration"))
    from reconstruct.mono_sequence import MonoSequence
    fr = golden_frames(np.load(GOLDEN))
    for fi, f in enumerate(fr):
        d = tmp_path / f"seq{fi}"
        (d / "image_0").mkdir(parents=True)
        (d / "lbl2d").mkdir()
        (d / "cam.yaml").write_text(f["yaml"])
        H, W = f["hw"]
        cv2.imwrite(str(d / "image_0" / ("%06d.png" % fi)), np.zeros((H, W, 3), np.uint8))
        torch.save({"pred_boxes": f["bboxes"], "pred_masks": f["masks"]}, str(d / "lbl2d" / ("%06d.lbl" % fi)))
        seq = MonoSequence(str(d), dict(detect_online=False, data_type="Redwood", path_label_2d=str(d / "lbl2d"),
                                        slam_config_path=str(d / "cam.yaml"), downsample_ratio=float(f["alpha"])))
        assert seq.mask_erosion == f["erosion"]
        got = seq.get_frame_by_id(fi)
        assert seq.detections_in_current_frame is got
        assert len(got) == f["n_inst"]
        if got:
            assert np.array_equal(got[0].background_rays, f["background_rays"])
            assert np.array_equal(got[0].bbox, f["bboxes"][f["mask_index"]])
        if f["raised"]:
            assert seq.current_frame is None and "no detections" in capsys.readouterr().err


def test_device_rays_feed_reconstruct_mono_batch(golden_dir, cfg_redwood):
    from dsp_slam_b200 import synth
    from dsp_slam_b200.optimizer import Optimizer
    from oracle import lidar_frame as OL
    from oracle import mono_frame as O
    opt = Optimizer(os.path.join(golden_dir, "decoder_chairs.npz"), cfg_redwood)
    objs_dev, objs_host = [], []
    for seed in range(3):
        f = synth.make_mono_frame(20 + seed, "redwood", 10)
        invK = np.linalg.inv(f["K"])
        dev = builder(f["K"], f["k1"], f["k2"], 4, f["img_hw"], 5).detections(f["masks"], f["bboxes"])[0].background_rays
        host = O.detection(f["masks"], f["bboxes"], f["K"], invK, f["k1"], f["k2"], 4, *f["img_hw"])["background_rays"]
        o = synth.make_object(300 + seed, 300, 150, 0, cls="chairs")
        # foreground rays from the surface points' pixels, as the mono path builds them
        uv = (o["pts"][:150] @ f["K"].T)[:, :2] / o["pts"][:150, 2:3]
        fg = OL.rays_of(uv, invK)
        base = dict(t_cam_obj=o["t_cam_obj_init"], pts=o["pts"], depth=o["depth"])
        flip = o["t_cam_obj_init"] @ np.diag([-1.0, 1.0, -1.0, 1.0]).astype(np.float32)
        objs_dev.append(dict(base, rays=np.concatenate([fg, dev]), t_cam_obj_flipped=flip))
        objs_host.append(dict(base, rays=np.concatenate([fg, host]), t_cam_obj_flipped=flip))
    ra = opt.reconstruct_mono_batch(objs_dev)
    rb = opt.reconstruct_mono_batch(objs_host)
    assert any(r.is_good for r in ra)
    for x, y in zip(ra, rb):
        assert x.is_good == y.is_good and x.flipped == y.flipped and np.float32(x.loss) == np.float32(y.loss)
        if x.is_good:
            assert np.array_equal(x.t_cam_obj, y.t_cam_obj) and np.array_equal(x.code, y.code)
