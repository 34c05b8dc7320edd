"""Python model of dspgn_mono.cuh's scalar formulas, one rounding per step as the device takes them.

Python floats are IEEE fp64 with round-to-nearest like the __d*_rn intrinsics, and round() on a float rounds half to
even like __double2int_rn.  tests/test_mono_frame_cpu.py checks this model against the installed cv2; the device is
then checked bit for bit against the numpy oracle and the golden.
"""
import math

import numpy as np

F = np.float32


def undistort(K, k1, k2, u, v, iters=5):
    """mono_undistort: (u, v) float32 pixel -> the float32 point cv2.undistortPoints(.., K, (k1, k2, 0, 0, 0), P=K)
    returns."""
    fx, fy, cx, cy = float(K[0][0]), float(K[1][1]), float(K[0][2]), float(K[1][2])
    ifx, ify = 1.0 / fx, 1.0 / fy
    u, v = float(F(u)), float(F(v))
    x, y = (u - cx) * ifx, (v - cy) * ify
    x0, y0 = x, y
    for _ in range(iters):
        r2 = x * x + y * y
        icdist = 1.0 / (1.0 + (k2 * r2 + k1) * r2)
        if icdist < 0:
            x, y = (u - cx) * ifx, (v - cy) * ify
            break
        x, y = x0 * icdist, y0 * icdist
    P = [[float(c) for c in row] for row in K]
    xx = (P[0][0] * x + P[0][1] * y) + P[0][2]
    yy = (P[1][0] * x + P[1][1] * y) + P[1][2]
    ww = 1.0 / ((P[2][0] * x + P[2][1] * y) + P[2][2])
    return F(xx * ww), F(yy * ww)


def icdist_negative(K, k1, k2, u, v, iters=5):
    """Whether OpenCV's loop takes its icdist < 0 exit for this pixel."""
    fx, fy, cx, cy = float(K[0][0]), float(K[1][1]), float(K[0][2]), float(K[1][2])
    x = (float(u) - cx) * (1.0 / fx)
    y = (float(v) - cy) * (1.0 / fy)
    x0, y0 = x, y
    for _ in range(iters):
        r2 = x * x + y * y
        icdist = 1.0 / (1.0 + (k2 * r2 + k1) * r2)
        if icdist < 0:
            return True
        x, y = x0 * icdist, y0 * icdist
    return False


def ellipse_half_width(e, dy):
    """mono_inside_eroded's row span: cvRound(e * sqrt((e*e - dy*dy) * (1./(e*e)))), 0 for e = 0."""
    if e == 0:
        return 0
    inv_r2 = 1.0 / float(e * e)
    return int(round(float(e) * math.sqrt(float(e * e - dy * dy) * inv_r2)))


def element(e):
    """The (2e+1)^2 structuring element as mono_inside_eroded reads it, as a uint8 array."""
    k = np.zeros((2 * e + 1, 2 * e + 1), np.uint8)
    for dy in range(-e, e + 1):
        dx = ellipse_half_width(e, dy)
        k[dy + e, e - dx:e + dx + 1] = 1
    return k


def inside_eroded(mask, e, x, y):
    """mono_inside_eroded for keypoint (pt.x, pt.y): every in-image mask pixel of the footprint is set."""
    H, W = mask.shape
    px, py = int(F(x)), int(F(y))
    for dy in range(-e, e + 1):
        yy = py + dy
        if yy < 0 or yy >= H:
            continue
        dx = ellipse_half_width(e, dy)
        if not mask[yy, max(px - dx, 0):min(px + dx, W - 1) + 1].all():
            return False
    return True
