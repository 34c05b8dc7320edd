"""numpy restatement of a monocular keyframe's detection (the reference's mono_sequence.Frame.get_detections,
reconstruct/mono_sequence.py:75-114) and of its keypoint test (Tracking::GetObjectDetectionsMono,
src/Tracking_util.cc:176-201), written from their semantics.

Test infrastructure only: the product (dsp_slam_b200/mono_frame.py + the CUDA path) never imports it, and it needs
no OpenCV: cv2.undistortPoints is restated as OpenCV's fp64 loop for distortion (k1, k2, 0, 0, 0) and P = K, and
cv2.erode with an ellipse is restated as a per-keypoint minimum over the element's footprint.  It is checked against
the golden made by running the unmodified reference with the real cv2 (tests/golden/make_mono_golden.py).
"""
import numpy as np

from oracle.lidar_frame import N_BACKGROUND, rays_of, sample_background

UNDISTORT_ITERS = 5   # cv2.undistortPoints' default TermCriteria(COUNT, 5, 0.01)


def largest_mask(masks):
    """np.argmax(masks.sum(-1).sum(-1)): the first mask with the most set pixels."""
    return int(np.argmax(masks.sum(axis=-1).sum(axis=-1)))


def undistort(pixels, K, k1, k2):
    """cv2.undistortPoints(pixels as float32, K, (k1, k2, 0, 0, 0), P=K) as (n, 2) float32: OpenCV's per-point loop in
    fp64.  The numerator of icdist is exactly 1 and the tangential terms exactly 0 for these coefficients."""
    K = np.asarray(K, np.float64)
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    ifx, ify = 1.0 / fx, 1.0 / fy
    u = pixels[:, 0].astype(np.float32).astype(np.float64)
    v = pixels[:, 1].astype(np.float32).astype(np.float64)
    x = (u - cx) * ifx
    y = (v - cy) * ify
    x0, y0 = x.copy(), y.copy()
    live = np.ones(x.shape, bool)
    for _ in range(UNDISTORT_ITERS):
        r2 = x * x + y * y
        icdist = 1.0 / (1.0 + (k2 * r2 + k1) * r2)
        neg = live & (icdist < 0)
        x[neg] = ((u - cx) * ifx)[neg]       # OpenCV falls back to the distorted point and stops iterating
        y[neg] = ((v - cy) * ify)[neg]
        live &= ~neg
        x = np.where(live, x0 * icdist, x)
        y = np.where(live, y0 * icdist, y)
    xx = (K[0, 0] * x + K[0, 1] * y) + K[0, 2]
    yy = (K[1, 0] * x + K[1, 1] * y) + K[1, 2]
    ww = 1.0 / ((K[2, 0] * x + K[2, 1] * y) + K[2, 2])
    return np.stack([xx * ww, yy * ww], -1).astype(np.float32)


def detection(masks, bboxes, K, inv_k, k1, k2, downsample_ratio, img_h, img_w):
    """None for a frame without masks, else dict(mask_index, n_nonsurface, background_rays): background_rays is None
    when fewer than 2 background pixels remain (the reference raises there), else (n, 3) float32."""
    if masks.shape[0] == 0:
        return None
    m = largest_mask(masks)
    bg = sample_background(bboxes[m], masks[m].astype(bool), int(downsample_ratio), img_h, img_w)
    n = bg.shape[0]
    if n > N_BACKGROUND:
        bg = bg[np.linspace(0, n - 1, N_BACKGROUND).astype(np.int32)]
    rays = None
    if bg.shape[0] >= 2:
        rays = rays_of(undistort(bg, K, k1, k2), np.asarray(inv_k, np.float64))
    return dict(mask_index=m, n_nonsurface=n, background_rays=rays)


def ellipse_rows(e):
    """Half-width per row dy = -e..e of getStructuringElement(MORPH_ELLIPSE, (2e+1, 2e+1), (e, e))."""
    if e == 0:
        return np.zeros(1, np.int64)
    inv_r2 = 1.0 / (float(e) * e)
    dy = np.arange(-e, e + 1)
    # cvRound: round half to even, as np.rint
    return np.rint(e * np.sqrt((e * e - dy * dy) * inv_r2)).astype(np.int64)


def feature_points(mask, keypoints, e):
    """Ascending indices of the keypoints ((int)y, (int)x) inside the mask eroded by the (2e+1)^2 ellipse, pixels
    outside the image ignored."""
    mask = np.asarray(mask).astype(bool)
    H, W = mask.shape
    half = ellipse_rows(e)
    kp = np.asarray(keypoints, np.float32)
    out = []
    for i, (x, y) in enumerate(kp):
        px, py = int(x), int(y)
        ok = True
        for r, dx in enumerate(half):
            yy = py + r - e
            if 0 <= yy < H and not mask[yy, max(px - dx, 0):min(px + dx, W - 1) + 1].all():
                ok = False
                break
        if ok:
            out.append(i)
    return np.array(out, np.int32)
