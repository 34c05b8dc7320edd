"""Python model of dspgn_frame.cuh's scalar formulas, one rounding per step as the device takes them.

np.float32 scalar arithmetic rounds every operation to float32 (no FMA) like __fmul_rn / __fadd_rn / __fdiv_rn, and
Python floats are IEEE fp64 with round-to-nearest like the __d*_rn intrinsics.  tests/test_lidar_frame_cpu.py checks
this model against numpy on random inputs; the device is then checked bit for bit against the numpy oracle.
"""
import math

import numpy as np

F = np.float32


def f3dot(a, r):
    """(a0 r0 + a1 r1) + a2 r2 in float32."""
    return F(F(F(a[0] * r[0]) + F(a[1] * r[1])) + F(a[2] * r[2]))


def transform(p, T):
    """rows 0..2 of T (3x4 float32) applied to p: f3dot + t."""
    return [F(f3dot(p, T[j, :3]) + T[j, 3]) for j in range(3)]


def selects(box, p):
    """k_frame_select's test of one point: trans / size / T_obj_velo as the device receives them."""
    x, y, z = (F(v) for v in box["trans"])
    if not (p[0] > F(x - F(3)) and p[0] < F(x + F(3)) and p[1] > F(y - F(3)) and p[1] < F(y + F(3))
            and p[2] > F(z - F(3)) and p[2] < F(z + F(3))):
        return False
    s = [F(v) for v in box["size"]]
    hw, hl, hh = F(F(s[0] * F(0.5)) * F(1.1)), F(F(s[1] * F(0.5)) * F(1.1)), F(s[2] * F(0.5))
    o = transform(p, box["T_obj_velo"])
    return bool(-hw < o[0] < hw and -hh < o[1] < hh and -hl < o[2] < hl)


def linspace(start, stop, num, i):
    """np.linspace(start, stop, num)[i] for integer start / stop (np_linspace)."""
    delta = float(stop) - float(start)
    div = num - 1
    y = float(i)
    if div > 0:
        step = delta / div
        y = (y / div) * delta if step == 0.0 else y * step
    else:
        y = y * delta
    y = y + float(start)
    if num > 1 and i == num - 1:
        y = float(stop)
    return y


def subsample_slot(r, n, m):
    """np_subsample_slot: the slot of rank r in np.linspace(0, n-1, m).astype(int32), or -1 (n > m >= 1)."""
    if m == 1:
        return 0 if r == 0 else -1
    step = float(n - 1) / float(m - 1)
    c = math.ceil(float(r) / step)
    for i in range(max(c - 1, 0), min(c + 1, m - 1) + 1):
        if int(linspace(0, n - 1, m, i)) == r:
            return i
    return -1


def project(K, q):
    h = [f3dot(q, K[j]) for j in range(3)]
    return F(h[0] / h[2]), F(h[1] / h[2])


def ray(inv_k, u, v):
    """inv_k [u, v, 1] in fp64, ((u k0 + v k1) + k2), cast to float32."""
    return [F((float(u) * float(inv_k[j, 0]) + float(v) * float(inv_k[j, 1])) + float(inv_k[j, 2])) for j in range(3)]
