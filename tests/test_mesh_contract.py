"""The ordering contract the device marching tetrahedra (csrc/dspgn_mesh.cuh) relies on, pinned on the host reference
dsp_slam_b200.mesh.marching_tetrahedra; and the mesh entry points' argument checks, which need no GPU."""
import ctypes as C

import numpy as np
import pytest

from dsp_slam_b200.mesh import marching_tetrahedra

# the 7 positive Kuhn edge offsets (dx, dy, dz), k = 4 dx + 2 dy + dz - 1: increasing flat offset
_OFFS = [((k + 1) >> 2 & 1, (k + 1) >> 1 & 1, (k + 1) & 1) for k in range(7)]


def _edge_scan(vol, h):
    """Vertices as the kernel numbers them: lattice vertices in row order, then their crossed edges by k; an edge counts
    when at least one cube that contains it has no NaN corner."""
    n = vol.shape
    m = [s - 1 for s in n]
    corners = np.stack([vol[dx:dx + m[0], dy:dy + m[1], dz:dz + m[2]]
                        for dx in (0, 1) for dy in (0, 1) for dz in (0, 1)])
    cube_ok = ~np.isnan(corners).any(axis=0)
    out = []
    for x in range(n[0]):
        for y in range(n[1]):
            for z in range(n[2]):
                for d in _OFFS:
                    hi = (x + d[0], y + d[1], z + d[2])
                    if any(hi[a] >= n[a] for a in range(3)):
                        continue
                    va, vb = float(vol[x, y, z]), float(vol[hi])
                    if (va < 0) == (vb < 0):
                        continue
                    rng = [range(c, c + 1) if dd else range(c - 1, c + 1) for c, dd in zip((x, y, z), d)]
                    if not any(0 <= cx < m[0] and 0 <= cy < m[1] and 0 <= cz < m[2] and cube_ok[cx, cy, cz]
                               for cx in rng[0] for cy in rng[1] for cz in rng[2]):
                        continue
                    t = (0.0 - va) / (vb - va)
                    pa = np.array([x, y, z], np.float64) * h
                    pb = np.array(hi, np.float64) * h
                    out.append(pa + t * (pb - pa))
    return np.array(out, np.float64).reshape(-1, 3).astype(np.float32)


@pytest.mark.parametrize("shape,nans", [((9, 8, 7), 0), ((6, 6, 6), 0), ((8, 8, 8), 1), ((7, 9, 8), 3)])
def test_vertices_are_the_scan_of_crossed_kuhn_edges(shape, nans):
    rng = np.random.default_rng(sum(shape) + nans)
    vol = rng.standard_normal(shape).astype(np.float32)
    for _ in range(nans):
        vol[tuple(rng.integers(1, s - 1) for s in shape)] = np.nan
    h = 2.0 / (shape[0] - 1)
    v, f = marching_tetrahedra(vol, 0.0, (h, h, h))
    e = _edge_scan(vol, h)
    assert v.shape == e.shape and np.array_equal(v, e)


def test_mesh_entry_points_reject_misuse_without_a_gpu():
    from dsp_slam_b200 import _lib
    from dsp_slam_b200.optimizer import BatchSolver
    lib = _lib.load()
    i32 = C.POINTER(C.c_int32)
    nv, nf = (C.c_int32 * 2)(), (C.c_int32 * 2)()
    codes = np.zeros((2, 64), np.float32)
    cp = codes.ctypes.data_as(C.POINTER(C.c_float))
    assert lib.dspgn_mesh_batch(None, 2, cp, 64, None, 32, nv, nf) == _lib.E_ARG
    assert lib.dspgn_mesh_batch(None, 2, None, 64, None, 32, nv, nf) == _lib.E_ARG
    assert lib.dspgn_mesh_batch(None, 0, cp, 64, None, 32, nv, nf) == _lib.E_ARG
    assert lib.dspgn_mesh_batch(None, 2, cp, 64, None, 1, nv, nf) == _lib.E_ARG
    assert lib.dspgn_mesh_results(None, None, C.cast(None, i32), None) == _lib.E_ARG
    assert lib.dspgn_debug_mesh_grid(None, 1, 8, None, nv, nf) == _lib.E_ARG
    bs = BatchSolver.__new__(BatchSolver)
    bs.handle = None
    with pytest.raises(ValueError):
        bs.mesh(np.zeros(64, np.float32), 32)            # one code must still be (1, code_len)
