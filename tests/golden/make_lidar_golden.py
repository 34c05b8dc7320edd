"""Golden frames of the KITTI LiDAR loader: tests/golden/lidar_frames.npz.

Runs the UNMODIFIED reference KITIISequence(...).get_frame_by_id (reconstruct/kitti_sequence.py) through
tools/ref_harness.py on synthetic frames written as real files (calib.txt, velodyne .bin, stored .lbl labels), with
three shims: a cv2 stand-in (imread loads the frame's image, stored as .npy bytes under the .png name; cvtColor flips
the channels), torch.load with weights_only=False (the labels are pickled numpy arrays), and the harness's own.
CPU only; needs the reference checkout.  `python tests/golden/make_lidar_golden.py` rewrites the npz.

The frames cover: boxes with more and fewer than num_lidar_max points and an empty box; a box behind the camera;
a front box matching no mask, and a matched mask at or below min_mask_area; more and fewer than 200 background
pixels; a bbox at the image border and crops narrower than alpha (linspace num 0 and 1); surface points projecting
outside the image and from behind the camera; two boxes matching one mask and a vote tie; a frame without masks.
"""
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
OUT = os.path.join(ROOT, "tests", "golden", "lidar_frames.npz")

H, W = 96, 320
P2 = np.array([[120.0, 0.0, 160.0, 44.857], [0.0, 121.5, 48.0, 0.2163], [0.0, 0.0, 1.0, 0.0027]])
TR = np.array([[0.0004, -0.9999, -0.0092, -0.0119], [0.0104, 0.0092, -0.9999, -0.0732], [0.9999, 0.0005, 0.0104, -0.2711]])
CFGS = {"A": (250, 300, 4.0), "B": (250, 50, 16.0), "C": (64, 300, 2.0)}


def calib_text():
    p2 = " ".join("%.12e" % v for v in P2.ravel())
    tr = " ".join("%.12e" % v for v in TR.ravel())
    p0 = " ".join("%.12e" % v for v in np.hstack([P2[:, :3], np.zeros((3, 1))]).ravel())
    return f"P0: {p0}\nP1: {p0}\nP2: {p2}\nP3: {p2}\nTr: {tr}\n"


def cam_of(pv):
    """velodyne -> camera (float64, for placing masks only)."""
    T = np.eye(4); T[:3] = TR
    S = np.eye(4); S[0, 3] = P2[0, 3] / P2[0, 0]
    M = S @ T
    return pv @ M[:3, :3].T + M[:3, 3]


def project(pc):
    h = pc @ P2[:, :3].T
    return h[:, :2] / h[:, 2:3]


def box_points(rng, det, n, shrink=0.9):
    x, y, z, w, l, h, th = det
    o = (rng.random((n, 3)) - 0.5) * np.array([w, h, l]) * shrink
    c, s = np.cos(th), np.sin(th)
    R = np.array([[c, 0, -s], [-s, 0, -c], [0, 1, 0]])
    return o @ R.T + np.array([x, y, z + h / 2])


def scan_with(rng, boxes_pts, n_bg=5000):
    bg = np.stack([rng.uniform(-20, 40, n_bg), rng.uniform(-15, 15, n_bg), rng.uniform(-2.5, 1.0, n_bg)], -1)
    pts = np.concatenate([bg] + boxes_pts, axis=0)
    pts = pts[rng.permutation(pts.shape[0])]
    refl = rng.random((pts.shape[0], 1))
    return np.concatenate([pts, refl], -1).astype(np.float32)


def rect_mask(u0, v0, u1, v1):
    m = np.zeros((H, W), bool)
    m[max(int(v0), 0):max(int(v1), 0), max(int(u0), 0):max(int(u1), 0)] = True
    return m


def proj_rect(pv, pad=2.0):
    uv = project(cam_of(pv))
    return uv[:, 0].min() - pad, uv[:, 1].min() - pad, uv[:, 0].max() + pad, uv[:, 1].max() + pad


def frames():
    rng = np.random.default_rng(20261015)
    out = []
    # F0: dense / sparse / empty / behind / small mask / border bbox / unmatched
    d = [(10.0, 0.0, -1.6, 1.6, 3.9, 1.5, 0.3), (14.0, 3.5, -1.6, 1.7, 4.2, 1.5, -0.4), (30.0, 12.0, 3.0, 1.6, 3.9, 1.5, 0.0),
         (-8.0, 1.0, -1.6, 1.6, 3.9, 1.5, 0.1), (20.0, -4.0, -1.6, 1.6, 3.9, 1.5, 1.2), (7.0, 7.5, -1.6, 1.6, 3.9, 1.5, 0.7),
         (18.0, -1.0, -1.6, 1.6, 3.9, 1.5, 2.0), (25.0, -9.0, -1.6, 1.6, 3.9, 1.5, 0.4)]
    npts = [600, 120, 0, 300, 200, 180, 90, 80]
    bp = [box_points(rng, np.array(b), n) for b, n in zip(d, npts)]
    r0, r1, r4, r5 = proj_rect(bp[0]), proj_rect(bp[1]), proj_rect(bp[4]), proj_rect(bp[5])
    masks = [rect_mask(*r0), rect_mask(r1[0] - 1, r1[1] - 1, r1[2] + 1, r1[3] + 1),
             rect_mask(r4[0] + 4, r4[1] + 2, r4[0] + 16, r4[1] + 14), rect_mask(*r5)]
    boxes = [np.array([r0[0] - 25, r0[1] - 12, r0[2] + 25, r0[3] + 12]), np.array(r1),
             np.array([r4[0], r4[1], r4[2], r4[3]]), np.array([2.7, r5[1], r5[2], r5[3]])]
    out.append(("A", scan_with(rng, bp), np.array(d, np.float32), np.array(masks), np.clip(np.array(boxes), 0, W).astype(np.float32)))
    # F1: two boxes in one mask, a vote tie, a box half outside the image, a box with points behind the camera plane
    d = [(12.0, 1.2, -1.6, 1.6, 3.9, 1.5, 0.0), (12.5, -1.2, -1.6, 1.6, 3.9, 1.5, 0.1), (16.0, 5.0, -1.6, 1.6, 3.9, 1.5, -0.3),
         (9.0, -9.0, -1.6, 1.6, 3.9, 1.5, 0.5), (1.0, 0.8, -0.9, 1.6, 4.0, 1.5, np.pi / 2)]
    npts = [260, 240, 150, 200, 300]
    bp = [box_points(rng, np.array(b), n) for b, n in zip(d, npts)]
    rab = proj_rect(np.concatenate([bp[0], bp[1]]))
    r2, r3 = proj_rect(bp[2]), proj_rect(bp[3])
    uvb = project(cam_of(bp[4]))
    inb = (uvb[:, 0] > 0) & (uvb[:, 0] < W) & (uvb[:, 1] > 0) & (uvb[:, 1] < H)
    r4 = (uvb[inb, 0].min() - 1, uvb[inb, 1].min() - 1, uvb[inb, 0].max() + 1, uvb[inb, 1].max() + 1) if inb.any() else (0, 0, 1, 1)
    masks = [rect_mask(*rab), rect_mask(*r2), rect_mask(*r2), rect_mask(*r3), rect_mask(*r4)]
    boxes = [np.array(rab), np.array(r2), np.array(r2) + 1, np.array([r3[0], r3[1], W - 1.5, r3[3]]), np.array(r4)]
    out.append(("A", scan_with(rng, bp), np.array(d, np.float32), np.array(masks), np.clip(np.array(boxes), 0, W).astype(np.float32)))
    # F2 (alpha 16): bboxes whose crops are narrower than alpha -> linspace num 0 and num 1
    d = [(10.0, 2.0, -1.6, 1.6, 3.9, 1.5, 0.2), (11.0, -3.0, -1.6, 1.6, 3.9, 1.5, -0.2), (13.0, 0.0, -1.6, 1.6, 3.9, 1.5, 0.0)]
    bp = [box_points(rng, np.array(b), 200) for b in d]
    rr = [proj_rect(p) for p in bp]
    masks = [rect_mask(*r) for r in rr]
    cu = [(r[0] + r[2]) / 2 for r in rr]
    cv = [(r[1] + r[3]) / 2 for r in rr]
    boxes = [np.array([cu[0], cv[0], cu[0] + 0.4, cv[0] + 0.3]), np.array([rr[1][0] - 3, rr[1][1] - 3, rr[1][0] + 17, rr[1][1] + 7]),
             np.array(rr[2])]
    out.append(("B", scan_with(rng, bp), np.array(d, np.float32), np.array(masks), np.clip(np.array(boxes), 0, W).astype(np.float32)))
    # F3: no masks at all (the detector's empty result)
    d = [(10.0, 0.0, -1.6, 1.6, 3.9, 1.5, 0.3), (15.0, 2.0, -1.6, 1.6, 3.9, 1.5, 0.0)]
    bp = [box_points(rng, np.array(b), 100) for b in d]
    out.append(("A", scan_with(rng, bp), np.array(d, np.float32), np.zeros((0, 0, 0), bool), np.zeros((0, 4), np.float32)))
    # F4 (num_lidar_max 64, alpha 2): N just above and far above the maximum, many background pixels
    d = [(9.0, 1.0, -1.6, 1.6, 3.9, 1.5, 0.4), (12.0, -2.5, -1.6, 1.6, 3.9, 1.5, -0.1), (17.0, 4.0, -1.6, 1.6, 3.9, 1.5, 0.9)]
    npts = [65, 900, 40]
    bp = [box_points(rng, np.array(b), n, shrink=0.8) for b, n in zip(d, npts)]
    rr = [proj_rect(p) for p in bp]
    masks = [rect_mask(*rr[0]), rect_mask(*rr[1]), rect_mask(*rr[2])]
    boxes = [np.array([rr[0][0] - 30, rr[0][1] - 20, rr[0][2] + 30, rr[0][3] + 20]), np.array(rr[1]), np.array(rr[2])]
    out.append(("C", scan_with(rng, bp), np.array(d, np.float32), np.array(masks), np.clip(np.array(boxes), 0, W).astype(np.float32)))
    return out


def install_cv2_stub():
    cv2 = types.ModuleType("cv2")
    cv2.COLOR_BGR2RGB = 4
    cv2.imread = lambda path, *a: np.load(path)
    cv2.cvtColor = lambda img, code: np.ascontiguousarray(img[..., ::-1])
    sys.modules["cv2"] = cv2


def write_sequence(root, fid, img, scan, dets, masks, boxes):
    import torch
    for sub in ("image_2", "velodyne", "lbl2d", "lbl3d"):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
    with open(os.path.join(root, "calib.txt"), "w") as f:
        f.write(calib_text())
    with open(os.path.join(root, "image_2", "%06d.png" % fid), "wb") as f:
        np.save(f, img)
    scan.tofile(os.path.join(root, "velodyne", "%06d.bin" % fid))
    torch.save(dets, os.path.join(root, "lbl3d", "%06d.lbl" % fid))
    torch.save({"pred_boxes": boxes, "pred_masks": masks}, os.path.join(root, "lbl2d", "%06d.lbl" % fid))


def main():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import ref_harness
    import torch
    ref_harness.install_shims()
    install_cv2_stub()
    load0 = torch.load
    torch.load = lambda *a, **k: load0(*a, **dict(k, weights_only=False))
    ks = __import__("reconstruct.kitti_sequence", fromlist=["KITIISequence"])
    rng = np.random.default_rng(7)
    arrs = {"numpy_version": np.array(np.__version__), "calib": np.array(calib_text()), "img_hw": np.array([H, W])}
    fr = frames()
    arrs["n_frames"] = np.array(len(fr))
    for fi, (cfg_name, scan, dets, masks, boxes) in enumerate(fr):
        nmax, marea, alpha = CFGS[cfg_name]
        img = rng.integers(0, 255, (H, W, 3), dtype=np.uint8)
        with tempfile.TemporaryDirectory() as root:
            write_sequence(root, fi, img, scan, dets, masks, boxes)
            cfg = ref_harness._AttrDict(detect_online=False, data_type="KITTI", path_label_2d=os.path.join(root, "lbl2d"),
                                        path_label_3d=os.path.join(root, "lbl3d"), num_lidar_max=nmax, num_lidar_min=10,
                                        min_mask_area=marea, downsample_ratio=alpha)
            seq = ks.KITIISequence(root, cfg)
            inst = seq.get_frame_by_id(fi)
            if fi == 0:
                arrs["K"], arrs["invK"], arrs["T_cam_velo"] = seq.K_cam, seq.invK_cam, seq.T_cam_velo
        p = f"f{fi}_"
        arrs.update({p + "scan": scan, p + "dets": dets, p + "masks": masks, p + "bboxes": boxes, p + "img": img,
                     p + "cfg": np.array([nmax, marea, alpha]), p + "n_inst": np.array(len(inst))})
        for i, it in enumerate(inst):
            q = f"{p}i{i}_"
            arrs[q + "T_cam_obj"] = it.T_cam_obj
            arrs[q + "scale"] = it.scale
            arrs[q + "surface_points"] = it.surface_points
            arrs[q + "num_surface_points"] = np.array(it.num_surface_points)
            arrs[q + "is_front"] = np.array(it.is_front)
            m = -1
            if "mask" in it:
                full = it.mask.base              # the loaded label's mask stack; instance.mask is a view of one entry
                m = (it.mask.__array_interface__["data"][0] - full.__array_interface__["data"][0]) // full.strides[0]
                assert np.array_equal(it.bbox, boxes[m])
            arrs[q + "mask_index"] = np.array(m)
            if it.rays is not None:
                arrs[q + "rays"] = it.rays
                arrs[q + "depth"] = it.depth
        summary = [(int(it.num_surface_points), bool(it.is_front), int(arrs[f"{p}i{i}_mask_index"]),
                    None if it.rays is None else it.rays.shape[0]) for i, it in enumerate(inst)]
        print(f"frame {fi} cfg {cfg_name}: {summary}")
    np.savez_compressed(OUT, **arrs)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
