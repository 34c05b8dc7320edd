"""The LiDAR keyframe's detections built on the H100 (DspgnLidarFrame): bit for bit against the golden made with the
unmodified reference, against the numpy oracle on full-size seeded frames, through the drop-in KITIISequence, and as
inputs of the keyframe call."""
import ctypes as C
import os
import sys
import types

import numpy as np
import pytest

from test_lidar_frame_cpu import GOLDEN, assert_instances_equal, golden_frames

pytestmark = pytest.mark.gpu


def as_dicts(inst, masks):
    """ResultDicts -> the oracle's dict form (mask_index from the view the instance holds)."""
    out = []
    for it in inst:
        d = dict(it)
        m = -1
        if "mask" in it:
            m = (it.mask.__array_interface__["data"][0] - masks.__array_interface__["data"][0]) // masks.strides[0]
            assert it.mask.base is not None and np.shares_memory(it.mask, masks)
        d["mask_index"] = m
        out.append(d)
    return out


def builder(K, Tcv, cfg, hw):
    from dsp_slam_b200.lidar_frame import LidarFrameBuilder
    return LidarFrameBuilder(K, Tcv, cfg, hw)


def test_device_equals_golden():
    g = np.load(GOLDEN)
    hw = tuple(int(v) for v in g["img_hw"])
    for inp, cfg, want in golden_frames(g):
        b = builder(g["K"], g["T_cam_velo"], cfg, hw)
        got = b.detections(inp["velo"], inp["dets"], inp["masks"], inp["bboxes"])
        assert_instances_equal(as_dicts(got, inp["masks"]), want)
        for it, w in zip(got, want):
            if w["mask_index"] >= 0:
                assert np.array_equal(it.bbox, inp["bboxes"][w["mask_index"]])


@pytest.mark.parametrize("seed,n_points", [(1, 120000), (2, 190000), (3, 260000)])
def test_device_equals_oracle_full_size(seed, n_points):
    from dsp_slam_b200 import synth
    from oracle import lidar_frame as O
    f = synth.make_lidar_frame(seed, n_points)
    K, Tcv = f["K"], f["T_cam_velo"]
    for cfg in (dict(num_lidar_max=250, min_mask_area=1000, downsample_ratio=4.0),
                dict(num_lidar_max=4096, min_mask_area=100, downsample_ratio=1.0)):
        want = O.detections(f["scan"], f["dets"], f["masks"], f["bboxes"], K, np.linalg.inv(K).astype(np.float32), Tcv,
                            cfg["num_lidar_max"], cfg["min_mask_area"], cfg["downsample_ratio"], *f["img_hw"])
        b = builder(K, Tcv, cfg, f["img_hw"])
        got = b.detections(f["scan"], f["dets"], f["masks"], f["bboxes"])
        assert_instances_equal(as_dicts(got, f["masks"]), want)
        again = b.detections(f["scan"], f["dets"], f["masks"], f["bboxes"])   # two runs are bit-identical
        assert_instances_equal(as_dicts(again, f["masks"]), want)
        assert sum(d["rays"] is not None for d in want) >= 3


def test_torch_inputs():
    import torch
    from dsp_slam_b200 import synth
    f = synth.make_lidar_frame(4, 130000)
    cfg = dict(num_lidar_max=250, min_mask_area=1000, downsample_ratio=4.0)
    b = builder(f["K"], f["T_cam_velo"], cfg, f["img_hw"])
    a = b.detections(f["scan"], f["dets"], f["masks"], f["bboxes"])
    t = b.detections(torch.from_numpy(f["scan"]), torch.from_numpy(f["dets"]), torch.from_numpy(f["masks"]),
                     torch.from_numpy(f["bboxes"]))
    assert_instances_equal(as_dicts(t, f["masks"]), as_dicts(a, f["masks"]))


def test_misuse_returns_e_arg_and_enqueues_nothing():
    from dsp_slam_b200 import _lib, synth
    lib = _lib.load()
    f = synth.make_lidar_frame(5, 120000)
    cfg = dict(num_lidar_max=250, min_mask_area=1000, downsample_ratio=4.0)
    b = builder(f["K"], f["T_cam_velo"], cfg, f["img_hw"])
    ref = b.detections(f["scan"], f["dets"], f["masks"], f["bboxes"])
    n_pts = sum(it.num_surface_points for it in ref)
    scan = np.ascontiguousarray(f["scan"])
    m8 = f["masks"].view(np.uint8)
    bb = f["bboxes"].astype(np.int32)
    box = (_lib.LidarBox * 257)()
    out = (_lib.LidarBoxOut * 257)()
    fp = scan.ctypes.data_as(_lib._FP)
    mp = m8.ctypes.data_as(C.POINTER(C.c_uint8))
    bp = bb.ctypes.data_as(C.POINTER(C.c_int32))
    bad = [(fp, (1 << 22) + 1, box, 1, mp, bp, 10), (fp, 100, box, 257, mp, bp, 10), (fp, 100, box, 1, mp, bp, 65),
           (None, 100, box, 1, mp, bp, 10), (fp, 100, None, 1, mp, bp, 10), (fp, 100, box, 1, None, bp, 10),
           (fp, 100, box, 1, mp, None, 10), (fp, -1, box, 1, mp, bp, 10)]
    for args in bad:
        assert lib.dspgn_lidar_frame_run(b._h, *args, out) == _lib.E_ARG
    bb_bad = bb.copy()
    bb_bad[3] = [50, 10, 40, 20]                           # l > r
    assert lib.dspgn_lidar_frame_run(b._h, fp, 100, box, 1, mp, bb_bad.ctypes.data_as(C.POINTER(C.c_int32)), 10, out) == _lib.E_ARG
    bb_bad[3] = [0, 0, 1243, 20]                           # r > img_w
    assert lib.dspgn_lidar_frame_run(b._h, fp, 100, box, 1, mp, bb_bad.ctypes.data_as(C.POINTER(C.c_int32)), 10, out) == _lib.E_ARG
    # the last good run's results are untouched
    pts = np.empty((n_pts, 3), np.float32)
    assert lib.dspgn_lidar_frame_results(b._h, pts.ctypes.data_as(_lib._FP), None, None) == 0
    assert np.array_equal(pts, np.concatenate([it.surface_points for it in ref]))
    sp = _lib.LidarSpec(img_h=375, img_w=1242, num_lidar_max=250, downsample_ratio=4)
    h = C.c_void_p()
    for k, v in (("num_lidar_max", 0), ("num_lidar_max", 4097), ("downsample_ratio", 0), ("img_h", 4097), ("img_w", 0)):
        s2 = _lib.LidarSpec.from_buffer_copy(sp)
        setattr(s2, k, v)
        assert lib.dspgn_lidar_frame_create(C.byref(s2), 0, C.byref(h)) == _lib.E_ARG
    with pytest.raises(TypeError):
        b.detections(f["scan"], f["dets"], f["masks"].astype(np.uint8), f["bboxes"])


def write_golden_sequence(root, g, fi):
    import torch
    p = f"f{fi}_"
    for sub in ("image_2", "velodyne", "lbl2d", "lbl3d"):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
    open(os.path.join(root, "calib.txt"), "w").write(str(g["calib"]))
    with open(os.path.join(root, "image_2", "%06d.png" % fi), "wb") as f:
        np.save(f, g[p + "img"])
    g[p + "scan"].tofile(os.path.join(root, "velodyne", "%06d.bin" % fi))
    torch.save(g[p + "dets"], os.path.join(root, "lbl3d", "%06d.lbl" % fi))
    torch.save({"pred_boxes": g[p + "bboxes"], "pred_masks": g[p + "masks"]}, os.path.join(root, "lbl2d", "%06d.lbl" % fi))


def test_dropin_sequence_equals_golden(tmp_path, monkeypatch):
    cv2 = types.ModuleType("cv2")           # image files of the golden are .npy bytes under the .png name
    cv2.COLOR_BGR2RGB = 4
    cv2.imread = lambda path, *a: np.load(path)
    cv2.cvtColor = lambda img, code: np.ascontiguousarray(img[..., ::-1])
    monkeypatch.setitem(sys.modules, "cv2", cv2)
    root = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
    monkeypatch.syspath_prepend(os.path.join(root, "integration"))
    from reconstruct.kitti_sequence import KITIISequence
    g = np.load(GOLDEN)
    for fi, (inp, cfg, want) in enumerate(golden_frames(g)):
        d = str(tmp_path / f"seq{fi}")
        write_golden_sequence(d, g, fi)
        seq = KITIISequence(d, dict(cfg, detect_online=False, path_label_2d=os.path.join(d, "lbl2d"),
                                    path_label_3d=os.path.join(d, "lbl3d")))
        got = seq.get_frame_by_id(fi)
        masks = seq.current_frame is not None and got and next((it.mask.base for it in got if "mask" in it), None)
        dicts = []
        for it in got:
            dd = dict(it)
            dd["mask_index"] = -1 if "mask" not in it else \
                (it.mask.__array_interface__["data"][0] - masks.__array_interface__["data"][0]) // masks.strides[0]
            dicts.append(dd)
        assert_instances_equal(dicts, want)
        assert seq.detections_in_current_frame is got


def test_detections_feed_the_keyframe_call(golden_dir, cfg_kitti):
    from dsp_slam_b200 import synth
    from dsp_slam_b200.optimizer import Optimizer
    from oracle import lidar_frame as O
    f = synth.make_lidar_frame(6, 150000)
    K, Tcv = f["K"], f["T_cam_velo"]
    cfg = dict(num_lidar_max=250, min_mask_area=1000, downsample_ratio=4.0)
    dev = builder(K, Tcv, cfg, f["img_hw"]).detections(f["scan"], f["dets"], f["masks"], f["bboxes"])
    ora = O.detections(f["scan"], f["dets"], f["masks"], f["bboxes"], K, np.linalg.inv(K).astype(np.float32), Tcv,
                       250, 1000, 4.0, *f["img_hw"])
    opt = Optimizer(os.path.join(golden_dir, "decoder_cars.npz"), cfg_kitti)

    def objs(ds):
        return [dict(t_cam_obj=d["T_cam_obj"], pts=d["surface_points"], rays=d["rays"], depth=d["depth"])
                for d in ds if d["rays"] is not None]

    a, b = objs(dev), objs(ora)
    assert len(a) >= 3
    ra, _ = opt.keyframe_batch(a, [])
    rb, _ = opt.keyframe_batch(b, [])
    assert any(r.is_good for r in ra)
    for x, y in zip(ra, rb):
        assert x.is_good == y.is_good and np.float32(x.loss) == np.float32(y.loss)
        if x.is_good:
            assert np.array_equal(x.t_cam_obj, y.t_cam_obj) and np.array_equal(x.code, y.code)
