"""tests/native/lidar_frame_caller.c: plain C in the Tracking thread's order -- build a LiDAR keyframe's detections on
the device, then reconstruct the detections with rays in one dspgn_reconstruct_batch call.  CPU: it compiles and
links.  GPU: its detections and records equal the Python path's bit for bit."""
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _build(tmp):
    exe = os.path.join(tmp, "lidar_frame_caller")
    libd = os.path.join(ROOT, "dsp_slam_b200")
    subprocess.check_call(["gcc", "-O1", "-std=c11", f"-I{os.path.join(ROOT, 'include')}",
                           os.path.join(ROOT, "tests", "native", "lidar_frame_caller.c"), "-o", exe, f"-L{libd}", "-ldspgn",
                           f"-Wl,-rpath,{libd}"])
    return exe


def test_lidar_frame_caller_compiles_and_links(tmp_path):
    exe = _build(str(tmp_path))
    assert subprocess.run([exe]).returncode == 2


@pytest.mark.gpu
def test_lidar_frame_caller_matches_python(tmp_path, golden_dir, cfg_kitti):
    from dsp_slam_b200 import _lib, synth
    from dsp_slam_b200.decoder import DecoderWeights
    from dsp_slam_b200.lidar_frame import LidarFrameBuilder, _box_matrices
    from dsp_slam_b200.optimizer import Optimizer
    exe = _build(str(tmp_path))
    dec = os.path.join(golden_dir, "decoder_cars.npz")
    w = DecoderWeights.from_npz(dec)
    wp, fp, op = str(tmp_path / "w.bin"), str(tmp_path / "frame.bin"), str(tmp_path / "out.bin")
    with open(wp, "wb") as f:
        f.write(struct.pack("<3i", len(w.W), w.latent_size, w.latent_in_layer))
        for W, b in zip(w.W, w.b):
            f.write(struct.pack("<2i", *W.shape)); f.write(W.tobytes()); f.write(b.tobytes())
    fr = synth.make_lidar_frame(11, 140000)
    cfg = dict(num_lidar_max=250, min_mask_area=1000, downsample_ratio=4.0)
    b = LidarFrameBuilder(fr["K"], fr["T_cam_velo"], cfg, fr["img_hw"])
    inst = b.detections(fr["scan"], fr["dets"], fr["masks"], fr["bboxes"])
    # the C caller gets the same per-box host matrices in the same depth order
    dets = fr["dets"][np.argsort(fr["dets"][:, 0]), :]
    boxes = (_lib.LidarBox * len(dets))()
    tco = np.stack([it.T_cam_obj for it in inst]).astype(np.float32)
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
        f.write(fr["scan"].tobytes()); f.write(bytes(boxes)); f.write(tco.tobytes())
        f.write(fr["masks"].view(np.uint8).tobytes()); f.write(fr["bboxes"].astype(np.int32).tobytes())
    r = subprocess.run([exe, wp, fp, op], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    raw = open(op, "rb").read()
    k = len(dets)
    hdr = np.frombuffer(raw, np.int32, 4 * k).reshape(k, 4)
    assert [h[0] for h in hdr] == [it.num_surface_points for it in inst]
    assert [h[1] for h in hdr] == [-1 if it.rays is None else it.rays.shape[0] for it in inst]
    npts, nr = int(hdr[:, 0].sum()), int(np.maximum(hdr[:, 1], 0).sum())
    o = 16 * k
    pts = np.frombuffer(raw, np.float32, 3 * npts, o).reshape(-1, 3); o += 12 * npts
    depth = np.frombuffer(raw, np.float32, npts, o); o += 4 * npts
    rays = np.frombuffer(raw, np.float32, 3 * nr, o).reshape(-1, 3); o += 12 * nr
    assert np.array_equal(pts, np.concatenate([it.surface_points for it in inst]))
    assert np.array_equal(depth, pts[:, 2])
    assert np.array_equal(rays, np.concatenate([it.rays for it in inst if it.rays is not None]))
    objs = [dict(t_cam_obj=it.T_cam_obj, pts=it.surface_points, rays=it.rays, depth=it.depth) for it in inst if it.rays is not None]
    ref = Optimizer(dec, cfg_kitti).reconstruct_batch(objs)
    rec = np.frombuffer(raw, np.float32, 82 * len(objs), o).reshape(-1, 82)
    for i, rr in enumerate(ref):
        assert (int(rec[i].view(np.int32)[0]) == 0) == rr.is_good
        if rr.is_good:
            assert np.array_equal(rec[i, 1:17].reshape(4, 4), rr.t_cam_obj) and np.array_equal(rec[i, 17:81], rr.code)
        assert rec[i, 81] == np.float32(rr.loss)
    assert any(rr.is_good for rr in ref)
