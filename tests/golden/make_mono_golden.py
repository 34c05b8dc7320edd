"""Golden frames of the monocular loader: tests/golden/mono_frames.npz.

Runs the UNMODIFIED reference MonoSequence(...).get_frame_by_id (reconstruct/mono_sequence.py) through
tools/ref_harness.py with the real cv2, on synthetic frames written as real files: the ORB-SLAM yaml
(read by cv2.FileStorage), the image (cv2.imwrite png) and the stored labels (.lbl, torch.save).  Two shims: np.bool8 =
np.bool_ (gone from numpy >= 1.24) and torch.load with weights_only=False (the labels are pickled numpy arrays).
The keypoint test of Tracking::GetObjectDetectionsMono (src/Tracking_util.cc:176-201) is C++ and is not built here;
its result is computed as that code does it, with cv2.getStructuringElement + cv2.erode on the float mask and the
(int) read of at<float>(pt.y, pt.x).  CPU only; needs the reference checkout.
`python tests/golden/make_mono_golden.py` rewrites the npz.

The frames cover: a tie for the largest mask; bboxes at each image border (all four clamp branches); crops narrower
than alpha (linspace num 0 and 1); 0, 1 and 2 background pixels (the first two raise in the reference); fewer and
more than 200 background pixels; the Redwood and Freiburg intrinsics, and a strongly distorted camera whose border
pixels take OpenCV's icdist < 0 branch (the shipped intrinsics never do); a frame without masks; erosion 0, 5, 10 and
15 with keypoints on mask edges, on the image border and at fractional coordinates.
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
OUT = os.path.join(ROOT, "tests", "golden", "mono_frames.npz")

# name: (fx, fy, cx, cy, k1, k2, H, W)
CAMERAS = {"redwood": (538.204343, 538.204343, 320.0, 240.0, 0.023896, -0.067078, 480, 640),
           "freiburg": (984.697, 984.697, 480.0, 270.0, -0.133543, -0.15436, 540, 960),
           "strong": (500.0, 500.0, 320.0, 240.0, -0.9, -0.6, 480, 640)}


def rect(H, W, l, t, r, b):
    m = np.zeros((H, W), bool)
    m[t:b, l:r] = True
    return m


def ellipse(H, W, cu, cv, au, av):
    v, u = np.mgrid[0:H, 0:W]
    return ((u - cu) / au) ** 2 + ((v - cv) / av) ** 2 <= 1.0


def keypoints(rng, H, W, mask, n=400):
    """Random, fractional, on the mask's edges and on the image border."""
    kp = [np.stack([rng.uniform(-0.99, W - 0.01, n), rng.uniform(-0.99, H - 0.01, n)], -1)]
    vv, uu = np.nonzero(mask)
    if vv.size:
        edge = mask & ~np.pad(mask, 1)[2:, 1:-1] | mask & ~np.pad(mask, 1)[:-2, 1:-1] | \
            mask & ~np.pad(mask, 1)[1:-1, 2:] | mask & ~np.pad(mask, 1)[1:-1, :-2]
        ev, eu = np.nonzero(edge)
        pick = rng.integers(0, ev.size, 150)
        kp.append(np.stack([eu[pick] + rng.choice([0.0, 0.5, 0.999], 150), ev[pick] + rng.choice([0.0, 0.25, 0.75], 150)], -1))
        pick = rng.integers(0, vv.size, 150)
        kp.append(np.stack([uu[pick] + rng.random(150), vv[pick] + rng.random(150)], -1))
    kp.append(np.array([[0.0, 0.0], [W - 1.0, H - 1.0], [W - 0.5, 0.5], [-0.5, H - 0.25], [0.25, -0.75],
                        [W - 0.01, H / 2], [W / 2, H - 0.01]]))
    return np.concatenate(kp, 0).astype(np.float32)


def frames():
    """(camera, alpha, erosion, masks, bboxes) per frame."""
    rng = np.random.default_rng(20261016)
    out = []
    H, W = 480, 640
    # F0 Redwood: a tie for the largest mask (1 and 2), > 200 background pixels, erosion 5
    m = [rect(H, W, 300, 200, 340, 260), ellipse(H, W, 320, 250, 120, 150), ellipse(H, W, 100, 100, 120, 150)]
    m[2] = np.roll(m[1], (-150, -220), (0, 1))
    bb = [[295.3, 198.7, 341.9, 262.2], [199.5, 99.2, 440.8, 400.6], [0.0, 0.0, 220.0, 250.0]]
    out.append(("redwood", 4, 5, np.array(m), np.array(bb, np.float32)))
    # F1 Freiburg: bbox at the left and top borders (both clamp to 0), erosion 15
    H, W = 540, 960
    m = [ellipse(H, W, 120, 110, 115, 105), rect(H, W, 600, 300, 640, 330)]
    bb = [[3.7, 4.2, 240.1, 220.9], [598.0, 299.0, 641.0, 331.0]]
    out.append(("freiburg", 4, 15, np.array(m), np.array(bb, np.float32)))
    # F2 Freiburg: bbox at the right and bottom borders, erosion 10, fewer than 200 background pixels (alpha 16)
    m = [rect(H, W, 700, 350, 957, 538), ellipse(H, W, 830, 440, 130, 95)]
    bb = [[697.2, 347.9, 958.4, 539.0], [699.0, 344.0, 960.0, 540.0]]
    out.append(("freiburg", 16, 10, np.array(m), np.array(bb, np.float32)))
    H, W = 480, 640
    # F3 Redwood, alpha 16: crop narrower than alpha (linspace num 0) -> no background pixel (the reference raises)
    m = [rect(H, W, 100, 100, 104, 104)]
    out.append(("redwood", 16, 0, np.array(m), np.array([[102.0, 102.0, 102.9, 102.5]], np.float32)))
    # F4: one background pixel (num 1 x num 1, outside the mask; the reference raises)
    m = [rect(H, W, 200, 200, 260, 260)]
    out.append(("redwood", 16, 5, np.array(m), np.array([[190.0, 190.0, 201.0, 201.0]], np.float32)))
    # F5: two background pixels (num 2 x num 1)
    m = [rect(H, W, 200, 200, 260, 260)]
    out.append(("redwood", 8, 5, np.array(m), np.array([[190.0, 190.0, 192.0, 200.0]], np.float32)))
    # F6: no masks
    out.append(("redwood", 4, 5, np.zeros((0, H, W), bool), np.zeros((0, 4), np.float32)))
    # F7: strong distortion (icdist < 0 near the border), a crop covering the whole image, erosion 0, alpha 2
    m = [ellipse(H, W, 320, 240, 200, 170), rect(H, W, 10, 10, 30, 30)]
    out.append(("strong", 2, 0, np.array(m), np.array([[0.0, 0.0, 640.0, 480.0], [9.5, 9.5, 30.5, 30.5]], np.float32)))
    # F8 Redwood: 20 random masks, erosion 10, alpha 1
    ms, bbs = [], []
    for _ in range(20):
        cu, cv = rng.uniform(60, W - 60), rng.uniform(60, H - 60)
        au, av = rng.uniform(20, 150), rng.uniform(20, 150)
        mk = ellipse(H, W, cu, cv, au, av)
        vv, uu = np.nonzero(mk)
        ms.append(mk)
        bbs.append([uu.min() - rng.uniform(0, 3), vv.min() - rng.uniform(0, 3), uu.max() + rng.uniform(0, 3), vv.max() + rng.uniform(0, 3)])
    out.append(("redwood", 1, 10, np.array(ms), np.clip(np.array(bbs), 0, [W, H, W, H]).astype(np.float32)))
    return out


def yaml_text(cam, erosion):
    fx, fy, cx, cy, k1, k2, H, W = cam
    return ("%YAML:1.0\n" + "".join(f"Camera.{k}: {v!r}\n" for k, v in
                                    (("fx", fx), ("fy", fy), ("cx", cx), ("cy", cy), ("k1", k1), ("k2", k2))) +
            f"Camera.width: {W}\nCamera.height: {H}\nObjects.maskErrosion: {erosion}\n")


def cv2_feature_points(cv2, mask_f32, kp, e):
    """Tracking_util.cc:181-195: erode a copy of the float mask with the ellipse, read (int) at<float>(pt.y, pt.x)."""
    kernel = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (2 * e + 1, 2 * e + 1), (e, e))
    er = cv2.erode(mask_f32, kernel)
    return np.array([i for i, (x, y) in enumerate(kp) if int(er[int(y), int(x)]) > 0], np.int32)


def main():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import cv2
    import ref_harness
    import torch
    ref_harness.install_shims()
    np.bool8 = np.bool_
    load0 = torch.load
    torch.load = lambda *a, **k: load0(*a, **dict(k, weights_only=False))
    ms = __import__("reconstruct.mono_sequence", fromlist=["MonoSequence"])
    rng = np.random.default_rng(11)
    arrs = {"numpy_version": np.array(np.__version__), "cv2_version": np.array(cv2.__version__)}
    fr = frames()
    arrs["n_frames"] = np.array(len(fr))
    for fi, (cam_name, alpha, e, masks, boxes) in enumerate(fr):
        cam = CAMERAS[cam_name]
        H, W = cam[6], cam[7]
        img = rng.integers(0, 255, (H, W, 3), dtype=np.uint8)
        with tempfile.TemporaryDirectory() as root:
            os.makedirs(os.path.join(root, "image_0"))
            os.makedirs(os.path.join(root, "lbl2d"))
            yp = os.path.join(root, "cam.yaml")
            with open(yp, "w") as f:
                f.write(yaml_text(cam, e))
            cv2.imwrite(os.path.join(root, "image_0", "%06d.png" % fi), img)
            torch.save({"pred_boxes": boxes, "pred_masks": masks}, os.path.join(root, "lbl2d", "%06d.lbl" % fi))
            cfg = ref_harness._AttrDict(detect_online=False, data_type="Redwood" if cam_name != "freiburg" else "Freiburg",
                                        path_label_2d=os.path.join(root, "lbl2d"), slam_config_path=yp,
                                        min_mask_area=1000, downsample_ratio=float(alpha))
            seq = ms.MonoSequence(root, cfg)
            p = f"f{fi}_"
            arrs[p + "K"], arrs[p + "invK"] = seq.K_cam, seq.invK_cam
            arrs[p + "dist"] = np.array([seq.k1, seq.k2])
            try:
                inst = seq.get_frame_by_id(fi)
                raised = ""
            except Exception as ex:          # noqa: BLE001 -- the reference's failure is part of the fixture
                inst, raised = None, type(ex).__name__
        kp = keypoints(rng, H, W, masks[int(np.argmax(masks.sum(-1).sum(-1)))] if masks.shape[0] else np.zeros((H, W), bool))
        arrs.update({p + "masks": masks, p + "bboxes": boxes, p + "cfg": np.array([alpha, e, H, W]), p + "kp": kp,
                     p + "raised": np.array(raised), p + "yaml": np.array(yaml_text(cam, e))})
        m = -1
        if inst:
            it = inst[0]
            full = it.bbox.base
            m = (it.bbox.__array_interface__["data"][0] - full.__array_interface__["data"][0]) // full.strides[0]
            assert np.array_equal(it.bbox, boxes[m]) and np.array_equal(it.mask, masks[m].astype(np.float32) * 255.)
            arrs[p + "background_rays"] = it.background_rays
        elif raised:
            m = int(np.argmax(masks.sum(-1).sum(-1)))       # the mask the reference chose before it raised
        arrs[p + "n_inst"] = np.array(0 if not inst else len(inst))
        arrs[p + "mask_index"] = np.array(m)
        if m >= 0:
            arrs[p + "feature_idx"] = cv2_feature_points(cv2, masks[m].astype(np.float32) * 255., kp, e)
        print(f"frame {fi} {cam_name} alpha {alpha} e {e}: mask {m} raised {raised or '-'} "
              f"rays {None if not inst else inst[0].background_rays.shape} "
              f"features {None if m < 0 else arrs[p + 'feature_idx'].size}/{kp.shape[0]}")
    np.savez_compressed(OUT, **arrs)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
