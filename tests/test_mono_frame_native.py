"""tests/native/mono_frame_caller.c: plain C in the Tracking thread's order -- build a monocular keyframe's detection
and its keypoint test on the device.  CPU: it compiles and links.  GPU: its output equals the Python path's bit for
bit."""
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _build(tmp):
    exe = os.path.join(tmp, "mono_frame_caller")
    libd = os.path.join(ROOT, "dsp_slam_b200")
    subprocess.check_call(["gcc", "-O1", "-std=c11", f"-I{os.path.join(ROOT, 'include')}",
                           os.path.join(ROOT, "tests", "native", "mono_frame_caller.c"), "-o", exe, f"-L{libd}", "-ldspgn",
                           f"-Wl,-rpath,{libd}"])
    return exe


def test_mono_frame_caller_compiles_and_links(tmp_path):
    exe = _build(str(tmp_path))
    assert subprocess.run([exe]).returncode == 2


@pytest.mark.gpu
@pytest.mark.parametrize("camera,e", [("redwood", 5), ("freiburg", 15)])
def test_mono_frame_caller_matches_python(tmp_path, camera, e):
    from dsp_slam_b200 import _lib, synth
    from dsp_slam_b200.mono_frame import MonoFrameBuilder
    exe = _build(str(tmp_path))
    fr = synth.make_mono_frame(31, camera, 12)
    b = MonoFrameBuilder(fr["K"], fr["k1"], fr["k2"], dict(downsample_ratio=4.0), fr["img_hw"], e)
    inst = b.detections(fr["masks"], fr["bboxes"], fr["keypoints"])
    feats = b.feature_points()
    sp = _lib.MonoSpec(img_h=b.img_h, img_w=b.img_w, downsample_ratio=4, mask_erosion=e, k1=b.k1, k2=b.k2)
    sp.k[:], sp.inv_k[:] = b.K.ravel().tolist(), b.invK.ravel().tolist()
    fp, op = str(tmp_path / "frame.bin"), str(tmp_path / "out.bin")
    with open(fp, "wb") as f:
        f.write(bytes(sp))
        f.write(struct.pack("<2i", fr["masks"].shape[0], fr["keypoints"].shape[0]))
        f.write(fr["masks"].view(np.uint8).tobytes()); f.write(fr["bboxes"].astype(np.int32).tobytes())
        f.write(np.ascontiguousarray(fr["keypoints"]).tobytes())
    r = subprocess.run([exe, fp, op], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    raw = open(op, "rb").read()
    mask, n_ns, n_rays, n_feat, good = np.frombuffer(raw, np.int32, 5)
    assert (mask, n_ns, n_rays, n_feat) == (b.last.mask, b.last.n_nonsurface, b.last.n_rays, b.last.n_feature)
    assert bool(good) == (feats.size >= 20) and good
    rays = np.frombuffer(raw, np.float32, 3 * n_rays, 20).reshape(-1, 3)
    assert np.array_equal(rays, inst[0].background_rays)
    assert np.array_equal(np.frombuffer(raw, np.int32, n_feat, 20 + 12 * n_rays), feats)
