"""numpy restatement of a KITTI LiDAR keyframe's detection geometry (the reference's
FrameWithLiDAR.get_detections, reconstruct/kitti_sequence.py:99-216), written from its semantics.

Test infrastructure only: the product (dsp_slam_b200/lidar_frame.py + the CUDA path) never imports it.
Every array it returns is what the reference computes bit for bit under numpy 2 (NEP 50 promotion); the
device path is checked against it on seeded full-size frames and both are checked against the golden made
by running the unmodified reference (tests/golden/make_lidar_golden.py).
"""
import numpy as np

NEAR_R = 3.0          # the +-3 m cube around a box centre
N_BACKGROUND = 200    # background pixels kept per box
EXPAND = 5            # the sampler's crop expansion


def box_matrices(det):
    """(T_velo_obj, T_obj_velo) of one 3D box row (x, y, z, w, l, h, theta), float32 as the loader builds them."""
    trans, size, theta = det[:3], det[3:6], det[6]
    c, s = np.cos(theta), np.sin(theta)
    T_velo_obj = np.array([[c, 0, -s, trans[0]],
                           [-s, 0, -c, trans[1]],
                           [0, 1, 0, trans[2] + size[2] / 2],
                           [0, 0, 0, 1]]).astype(np.float32)
    return T_velo_obj, np.linalg.inv(T_velo_obj)


def transform3(p, T):
    """(p[:, None, :3] * T[:3, :3]).sum(-1) + T[:3, 3] in p's float type: ((p0 r0 + p1 r1) + p2 r2) + t."""
    R, t = T[:3, :3], T[:3, 3]
    return (p[:, None, :3] * R).sum(-1) + t


def box_points(velo, trans, size, T_obj_velo, num_max):
    """The scan points of one box in scan order, subsampled to num_max ranks (velodyne frame, n x 4)."""
    x, y, z = list(trans)
    near = ((velo[:, 0] > x - NEAR_R) & (velo[:, 0] < x + NEAR_R) &
            (velo[:, 1] > y - NEAR_R) & (velo[:, 1] < y + NEAR_R) &
            (velo[:, 2] > z - NEAR_R) & (velo[:, 2] < z + NEAR_R))
    pn = velo[near]
    po = transform3(pn, T_obj_velo)
    hw, hl, hh = list(size / 2)
    hw *= 1.1
    hl *= 1.1
    inside = ((po[:, 0] > -hw) & (po[:, 0] < hw) & (po[:, 1] > -hh) & (po[:, 1] < hh) &
              (po[:, 2] > -hl) & (po[:, 2] < hl))
    ps = pn[inside]
    if ps.shape[0] > num_max:
        ps = ps[np.linspace(0, ps.shape[0] - 1, num_max).astype(np.int32)]
    return ps, hl


def sample_background(bbox, mask, alpha, img_h, img_w):
    """(u, v) int32 pixels of the expanded-crop grid that lie outside the mask, row-major."""
    max_w, max_h = img_w - 1, img_h - 1
    l, t, r, b = [int(v) for v in bbox.astype(np.int32)]
    l = l - EXPAND if l > EXPAND else 0
    t = t - EXPAND if t > EXPAND else 0
    r = r + EXPAND if r < max_w - EXPAND else max_w
    b = b + EXPAND if b < max_h - EXPAND else max_h
    hh = np.linspace(t, b, int((b - t + 1) / alpha)).astype(np.int32)
    ww = np.linspace(l, r, int((r - l + 1) / alpha)).astype(np.int32)
    vv = np.repeat(hh, ww.shape[0])
    uu = np.tile(ww, hh.shape[0])
    keep = ~mask[vv, uu]
    return np.stack([uu[keep], vv[keep]], axis=-1)


def rays_of(pixels, inv_k):
    """inv_k [u, v, 1] in float64, ((u k0 + v k1) + k2), cast to float32."""
    uh = np.concatenate([pixels.astype(np.float64), np.ones((pixels.shape[0], 1))], axis=-1)
    return (uh[:, None, :] * inv_k).sum(-1).astype(np.float32)


def detections(velo, dets, masks, bboxes, K, inv_k, T_cam_velo, num_lidar_max, min_mask_area, downsample_ratio,
               img_h, img_w):
    """The frame's instances in depth order: dicts with T_cam_obj, scale, surface_points, num_surface_points,
    is_front, rays (None or (n, 3) f32), and, when matched, mask_index (plus depth when rays is not None)."""
    dets = dets[np.argsort(dets[:, 0]), :]
    alpha = int(downsample_ratio)
    out = []
    for n in range(dets.shape[0]):
        d = dets[n, :]
        trans, size = d[:3], d[3:6]
        T_velo_obj, T_obj_velo = box_matrices(d)
        ps, hl = box_points(velo, trans, size, T_obj_velo, num_lidar_max)
        pc = transform3(ps, T_cam_velo).astype(np.float32)
        T_cam_obj = T_cam_velo @ T_velo_obj
        T_cam_obj[:3, :3] *= hl
        out.append(dict(T_cam_obj=T_cam_obj, scale=size, surface_points=pc, num_surface_points=pc.shape[0],
                        is_front=T_cam_obj[2, 3] > 0.0, rays=None, mask_index=-1))
    if masks.shape[0] == 0:
        return out
    for inst in out:
        if not inst["is_front"]:
            continue
        sp = inst["surface_points"]
        ph = (sp[:, None, :] * K).sum(-1)
        uv = ph[:, :2] / ph[:, 2, None]
        fov = (uv[:, 0] > 0) & (uv[:, 0] < img_w) & (uv[:, 1] > 0) & (uv[:, 1] < img_h)
        pix = uv[fov].astype(np.int32)
        votes = np.array([int(np.count_nonzero(masks[m, pix[:, 1], pix[:, 0]])) for m in range(masks.shape[0])])
        if votes.max() > pix.shape[0] * 0.5:
            m = int(np.argmax(votes))
            inst["mask_index"] = m
            if int(np.count_nonzero(masks[m])) > min_mask_area:
                bg = sample_background(bboxes[m], masks[m], alpha, img_h, img_w)
                if bg.shape[0] > N_BACKGROUND:
                    bg = bg[np.linspace(0, bg.shape[0] - 1, N_BACKGROUND).astype(np.int32)]
                inst["rays"] = rays_of(np.concatenate([uv, bg], axis=0), inv_k)
                inst["depth"] = sp[:, 2].astype(np.float32)
    return out
