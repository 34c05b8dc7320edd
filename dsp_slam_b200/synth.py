"""Seeded synthetic detections with the shapes DSP-SLAM's sequence loaders hand to the optimiser.

Mirrors what reconstruct/kitti_sequence.py:114-216 produces per detection (T_cam_obj initial guess,
surface points in the camera frame, foreground rays + depths, background rays) for an analytic
latent-conditioned ellipsoid -- the shape family the fixture decoders in tests/golden/ are fitted
to (tools/fit_fixture_decoder.py).  numpy only; no CUDA, no torch.  SURVEY.md section 8(d).
"""
import numpy as np

F32 = np.float32

CLASS_RADII = {"cars": (0.30, 0.25, 0.60), "chairs": (0.35, 0.45, 0.35)}


def _rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def make_object(seed, n_pts, n_fg_rays=None, n_bg_rays=0, cls="cars", code_scale=0.1,
                noise=0.01, trans_jitter=0.15, yaw_jitter=0.1, init_code_frac=None):
    """One synthetic detection.

    Returns dict with (all float32, Fortran-ordered like pybind11's Eigen casters deliver them,
    src/LocalMapping_util.cc:179-180):
      t_cam_obj_init (4,4)  initial Sim(3) object->camera guess
      t_cam_obj_gt   (4,4)  ground truth
      pts   (n_pts,3)       surface points, camera frame
      rays  (n_fg+n_bg,3)   ray directions (z = 1), foreground first
      depth (n_fg,)         observed depth of the foreground rays
      code_gt (64,), code_init (64,) or None
    """
    rng = np.random.default_rng(10_000 + seed)
    radii0 = np.array(CLASS_RADII[cls])
    z_gt = code_scale * rng.standard_normal(64)
    radii = radii0 * (1.0 + z_gt[:3])
    s = rng.uniform(1.5, 2.5)
    yaw = rng.uniform(-np.pi, np.pi)
    t = np.array([rng.uniform(-5, 5), rng.uniform(0.5, 1.5), rng.uniform(6, 25)])
    flip = np.diag([1.0, -1.0, -1.0])          # camera y down / object y up
    R = _rot_y(yaw) @ flip
    T_gt = np.eye(4)
    T_gt[:3, :3] = s * R
    T_gt[:3, 3] = t

    def surface(n):
        d = rng.standard_normal((n, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        p_obj = d * radii
        # keep the camera-facing one of each antipodal pair (proxy for visibility)
        pa = (p_obj @ (s * R).T) + t
        pb = ((-p_obj) @ (s * R).T) + t
        p = np.where((np.linalg.norm(pa, axis=1) <= np.linalg.norm(pb, axis=1))[:, None], pa, pb)
        return p + noise * rng.standard_normal((n, 3))

    pts = surface(n_pts)
    out = dict(t_cam_obj_gt=T_gt, pts=pts, code_gt=z_gt)

    if n_fg_rays is None:
        n_fg_rays = n_pts
    if n_fg_rays or n_bg_rays:
        fg_src = pts[:n_fg_rays] if n_fg_rays <= n_pts else surface(n_fg_rays)
        fg = fg_src / fg_src[:, 2:3]
        depth = fg_src[:, 2].copy()
        bg = np.zeros((0, 3))
        if n_bg_rays:
            centre = t / t[2]
            half = 1.0 * s / t[2]
            Rinv = R.T / s
            got = []
            while sum(len(g) for g in got) < n_bg_rays:
                uv = centre[:2] + rng.uniform(-half, half, size=(4 * n_bg_rays, 2))
                r = np.concatenate([uv, np.ones((len(uv), 1))], axis=1)
                # ray/ellipsoid test in the radii-normalised object frame (inflated 15 %)
                o = (Rinv @ (-t)) / (1.15 * radii)
                dirs = (r @ Rinv.T) / (1.15 * radii)
                a = (dirs * dirs).sum(1)
                b = (dirs * o).sum(1)
                c = (o * o).sum() - 1.0
                miss = (b * b - a * c) < 0
                got.append(r[miss])
            bg = np.concatenate(got)[:n_bg_rays]
        out["rays"] = np.concatenate([fg, bg], axis=0)
        out["depth"] = depth

    # initial guess: translation + yaw jitter (SURVEY.md 8d)
    dyaw = yaw_jitter * rng.standard_normal()
    dt = trans_jitter * rng.standard_normal(3)
    T0 = np.eye(4)
    T0[:3, :3] = s * (_rot_y(yaw + dyaw) @ flip)
    T0[:3, 3] = t + dt
    out["t_cam_obj_init"] = T0
    out["code_init"] = None if init_code_frac is None else init_code_frac * z_gt

    for k, v in list(out.items()):
        if isinstance(v, np.ndarray):
            out[k] = np.asfortranarray(v.astype(F32))
    return out


def make_batch(n_obj, n_pts, n_fg_rays=None, n_bg_rays=0, cls="cars", seed0=0, **kw):
    clss = cls if isinstance(cls, (list, tuple)) else [cls] * n_obj
    return [make_object(seed0 + i, n_pts, n_fg_rays, n_bg_rays, cls=clss[i], **kw)
            for i in range(n_obj)]


KITTI_K = np.array([[721.5377, 0.0, 609.5593], [0.0, 721.5377, 172.854], [0.0, 0.0, 1.0]], F32)
KITTI_T_CAM_VELO = np.array([[0.000427, -0.999967, -0.008084, 0.048489], [-0.007211, 0.008081, -0.999941, -0.073220],
                             [0.999974, 0.000485, -0.007206, -0.333997], [0.0, 0.0, 0.0, 1.0]], F32)


def make_lidar_frame(seed, n_points=127000, n_boxes=20, n_masks=10, img_hw=(375, 1242)):
    """A KITTI-sized LiDAR keyframe as FrameWithLiDAR.get_detections receives it (kitti_sequence.py:99-216):
    scan (n, 4) f32 with dense clusters inside the boxes, boxes (k, 7) f32 (x, y, z, w, l, h, theta, velodyne frame),
    masks (m, H, W) bool over the projections of the nearest front boxes (one pair shares a mask, one mask misses),
    bboxes (m, 4) f32 clipped to the image."""
    rng = np.random.default_rng(seed)
    H, W = img_hw
    x = rng.uniform(-15, 45, n_boxes)
    y = rng.uniform(-12, 12, n_boxes)
    size = np.stack([rng.uniform(1.4, 2.0, n_boxes), rng.uniform(3.4, 4.8, n_boxes), rng.uniform(1.3, 1.8, n_boxes)], -1)
    th = rng.uniform(-np.pi, np.pi, n_boxes)
    dets = np.concatenate([np.stack([x, y, np.full(n_boxes, -1.7)], -1), size, th[:, None]], -1)
    cl, per_box = [], []
    n_dense = int(n_points * 0.25)
    counts = rng.multinomial(n_dense, rng.dirichlet(np.ones(n_boxes)))
    for b in range(n_boxes):
        o = (rng.random((counts[b], 3)) - 0.5) * np.array([size[b, 0], size[b, 2], size[b, 1]]) * 1.05
        c, s = np.cos(th[b]), np.sin(th[b])
        R = np.array([[c, 0, -s], [-s, 0, -c], [0, 1, 0]])
        p = o @ R.T + np.array([x[b], y[b], -1.7 + size[b, 2] / 2])
        cl.append(p)
        per_box.append(p)
    n_bg = n_points - n_dense
    bg = np.stack([rng.uniform(-40, 60, n_bg), rng.uniform(-30, 30, n_bg), rng.uniform(-2.5, 1.0, n_bg)], -1)
    pts = np.concatenate([bg] + cl, 0)
    pts = pts[rng.permutation(pts.shape[0])]
    scan = np.concatenate([pts, rng.random((pts.shape[0], 1))], -1).astype(F32)
    # masks over the projected clusters of the front boxes, nearest first
    T = KITTI_T_CAM_VELO.astype(np.float64)
    K = KITTI_K.astype(np.float64)
    rects = []
    for b in np.argsort(x):
        pc = per_box[b] @ T[:3, :3].T + T[:3, 3]
        pc = pc[pc[:, 2] > 0.5]
        if pc.shape[0] < 10:
            continue
        uv = (pc @ K.T)[:, :2] / (pc @ K.T)[:, 2:3]
        u0, v0 = np.clip(uv.min(0), 0, [W, H])
        u1, v1 = np.clip(uv.max(0), 0, [W, H])
        if u1 - u0 > 2 and v1 - v0 > 2:
            rects.append((u0, v0, u1, v1))
    masks = np.zeros((n_masks, H, W), bool)
    bboxes = np.zeros((n_masks, 4), F32)
    for m in range(n_masks):
        if m < len(rects) and m != n_masks - 1:
            u0, v0, u1, v1 = rects[m]
            if m == 1 and len(rects) > 2:          # one mask covering two boxes
                u0, v0 = min(u0, rects[2][0]), min(v0, rects[2][1])
                u1, v1 = max(u1, rects[2][2]), max(v1, rects[2][3])
        else:                                      # a mask where no box projects
            u0, v0 = rng.uniform(0, W - 60), rng.uniform(0, H - 40)
            u1, v1 = u0 + 50, v0 + 30
        masks[m, int(v0):int(np.ceil(v1)), int(u0):int(np.ceil(u1))] = True
        bboxes[m] = np.clip([u0 - rng.uniform(0, 30), v0 - rng.uniform(0, 15), u1 + rng.uniform(0, 30), v1 + rng.uniform(0, 15)],
                            0, [W, H, W, H])
    return dict(scan=scan, dets=dets.astype(F32), masks=masks, bboxes=bboxes, K=KITTI_K, T_cam_velo=KITTI_T_CAM_VELO,
                img_hw=(H, W))


# Redwood 01053 and Freiburg 002 cameras (Camera.fx, fy, cx, cy, k1, k2 of their ORB-SLAM yamls) and image sizes
MONO_CAMERAS = {"redwood": ((538.204343, 538.204343, 320.0, 240.0), 0.023896, -0.067078, (480, 640)),
                "freiburg": ((984.697, 984.697, 480.0, 270.0), -0.133543, -0.15436, (540, 960))}


def make_mono_frame(seed, camera="redwood", n_masks=12, n_kp=2000):
    """A full-size monocular keyframe as Frame.get_detections and GetObjectDetectionsMono receive it
    (mono_sequence.py:75-114, Tracking_util.cc:176-201): masks (m, H, W) bool (ellipses with ragged edges, one large
    object in the middle), bboxes (m, 4) f32 around them, keypoints (n, 2) f32 (pt.x, pt.y; a third on the largest
    mask, fractional, some on the image border), K (3, 3) f64, k1, k2."""
    rng = np.random.default_rng(seed)
    (fx, fy, cx, cy), k1, k2, (H, W) = MONO_CAMERAS[camera]
    v, u = np.mgrid[0:H, 0:W]
    masks = np.zeros((n_masks, H, W), bool)
    bboxes = np.zeros((n_masks, 4), F32)
    for m in range(n_masks):
        big = m == n_masks // 2
        cu = W / 2 + rng.uniform(-30, 30) if big else rng.uniform(0, W)
        cv = H / 2 + rng.uniform(-20, 20) if big else rng.uniform(0, H)
        au = rng.uniform(0.2, 0.3) * W if big else rng.uniform(10, 0.15 * W)
        av = rng.uniform(0.25, 0.35) * H if big else rng.uniform(10, 0.15 * H)
        r = ((u - cu) / au) ** 2 + ((v - cv) / av) ** 2
        mk = r <= 1.0 + 0.08 * rng.standard_normal((H, W))
        masks[m] = mk
        vv, uu = np.nonzero(mk)
        if vv.size == 0:
            continue
        bboxes[m] = np.clip([uu.min() - rng.uniform(0, 4), vv.min() - rng.uniform(0, 4), uu.max() + rng.uniform(0, 4),
                             vv.max() + rng.uniform(0, 4)], 0, [W, H, W, H])
    big = masks[int(np.argmax(masks.sum(-1).sum(-1)))]
    vv, uu = np.nonzero(big)
    n_in = n_kp // 3
    pick = rng.integers(0, vv.size, n_in)
    kp = np.concatenate([np.stack([uu[pick] + rng.random(n_in), vv[pick] + rng.random(n_in)], -1),
                         np.stack([rng.uniform(-0.99, W - 0.01, n_kp - n_in - 4), rng.uniform(-0.99, H - 0.01, n_kp - n_in - 4)], -1),
                         [[0.0, 0.0], [W - 0.5, H - 0.5], [-0.5, H / 2], [W / 2, H - 0.01]]]).astype(F32)
    K = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])
    return dict(masks=masks, bboxes=bboxes, keypoints=kp, K=K, k1=k1, k2=k2, img_hw=(H, W))
