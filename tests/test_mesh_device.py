"""Meshes on the device (dspgn_mesh_batch, csrc/dspgn_mesh.cuh) against the host reference marching_tetrahedra
(dsp_slam_b200/mesh.py): same vertex bytes and order, same faces, on given grids and on decoded ones."""
import os

import numpy as np
import pytest

from dsp_slam_b200.mesh import marching_tetrahedra

pytestmark = pytest.mark.gpu

ENGINES = ["simt", "tc"]


def _host_mesh(grid):
    """extract_mesh_from_code's host fallback on one grid: marching tetrahedra, vertices shifted by -1."""
    dim = grid.shape[0]
    v, f = marching_tetrahedra(grid, 0.0, [2.0 / (dim - 1)] * 3)
    return (v + np.array([-1.0, -1.0, -1.0])).astype(np.float32), f.astype(np.int32)


def _same(dev, host):
    (v, f), (hv, hf) = dev, host
    assert v.dtype == np.float32 and f.dtype == np.int32
    assert v.shape == hv.shape and f.shape == hf.shape
    assert v.tobytes() == hv.tobytes()
    assert np.array_equal(f, hf)


@pytest.fixture(scope="module")
def golden():
    return os.path.join(os.path.dirname(__file__), "golden")


def _extractor(golden, dim, engine="simt", name="cars", **kw):
    from dsp_slam_b200.optimizer import MeshExtractor
    from dsp_slam_b200._lib import DspgnError
    try:
        return MeshExtractor(os.path.join(golden, f"decoder_{name}.npz"), 64, dim, engine=engine, **kw)
    except DspgnError:
        if engine == "tc":
            pytest.skip("tensor-core engine not available")
        raise


def _sphere(n, r=0.6, c=(0.03, -0.02, 0.05)):
    ax = np.linspace(-1, 1, n)
    X, Y, Z = np.meshgrid(ax, ax, ax, indexing="ij")
    return (np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r).astype(np.float32)


def _grids():
    rng = np.random.default_rng(7)
    out = {f"sphere{d}": _sphere(d, 0.6 if d > 3 else 0.9) for d in (2, 3, 16, 33, 64)}
    ax = np.arange(12, dtype=np.float32)
    X, Y, Z = np.meshgrid(ax, ax, ax, indexing="ij")
    out["plane_through_lattice"] = (X + Y - 2 * Z + 3).astype(np.float32)     # exact zeros on lattice vertices
    out["noise24"] = rng.standard_normal((24, 24, 24)).astype(np.float32)
    g = rng.standard_normal((12, 12, 12)).astype(np.float32)
    g[3, 4, 5] = np.nan
    g[0, 0, 0] = np.nan
    g[11, 6, 2] = np.nan
    out["noise_nan"] = g
    s = _sphere(20)
    s[10, 10, 4] = np.nan
    s[:, 0, :] = np.nan
    out["sphere_nan"] = s
    out["all_positive"] = np.abs(_sphere(10)) + 0.1
    out["all_negative"] = -np.abs(_sphere(10)) - 0.1
    return out


@pytest.mark.parametrize("name", list(_grids()))
def test_given_grids_match_marching_tetrahedra(name, golden):
    grid = _grids()[name]
    mx = _extractor(golden, 8)
    dev = mx.solver.debug_mesh_grid(grid[None])[0]
    host = _host_mesh(grid)
    _same(dev, host)
    if name.startswith("all_"):
        assert dev[0].shape == (0, 3) and dev[1].shape == (0, 3)
    if name == "plane_through_lattice":
        assert (grid == 0).any() and dev[1].shape[0] > 0            # collapsed triangles dropped, the rest kept


def _codes(golden):
    d = np.load(os.path.join(golden, "recon_kitti250.npz"))
    v = np.load(os.path.join(golden, "voxel.npz"))
    return {"zero": np.zeros(64, np.float32), "golden": v["z"].astype(np.float32),
            "gt": d["gt_code"].astype(np.float32), "reconstructed": d["code"].astype(np.float32)}


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", ["cars", "chairs"])
@pytest.mark.parametrize("dim", [8, 16, 32, 64])
def test_decoded_grids_and_meshes(engine, name, dim, golden):
    mx = _extractor(golden, dim, engine, name)
    codes = _codes(golden)
    meshes, sdf = mx.solver.mesh(np.stack(list(codes.values())), dim, want_sdf=True)
    c = mx.solver.counters()
    assert c["rows_fwd_only"] == len(codes) * dim ** 3 and c["kernel_launches"] > 0
    for i, code in enumerate(codes.values()):
        grid = mx.sdf_grid(code)
        assert sdf[i].tobytes() == grid.tobytes()
        _same(meshes[i], _host_mesh(grid))


def test_batch_equals_single_calls(golden):
    mx = _extractor(golden, 32)
    rng = np.random.default_rng(3)
    codes = (0.3 * rng.standard_normal((5, 64))).astype(np.float32)
    codes[0] = _codes(golden)["reconstructed"]
    batch = mx.extract_meshes(codes)
    for i in range(len(codes)):
        one = mx.extract_meshes(codes[i:i + 1])[0]
        _same((batch[i].vertices, batch[i].faces), (one.vertices, one.faces))


def test_mixed_classes_on_a_two_class_solver(golden):
    from dsp_slam_b200.optimizer import BatchSolver
    mc = _extractor(golden, 16, name="cars")
    mh = _extractor(golden, 16, name="chairs")
    two = BatchSolver([mc._dd, mh._dd], mc.solver.cfg, 0)
    code = _codes(golden)["reconstructed"]
    cls = [0, 1, 1, 0]
    meshes, sdf = two.mesh(np.stack([code] * 4), 16, class_ids=cls, want_sdf=True)
    for i, c in enumerate(cls):
        grid = (mc if c == 0 else mh).sdf_grid(code)
        assert sdf[i].tobytes() == grid.tobytes()
        _same(meshes[i], _host_mesh(grid))
    assert not np.array_equal(sdf[0], sdf[1])


def test_batch_across_the_chunk_bound_and_nan_code(golden):
    # 2^24 grid rows per chunk: 64 objects of 64^3, so 66 codes take two chunks
    mx = _extractor(golden, 64, "tc")
    rng = np.random.default_rng(5)
    codes = (0.2 * rng.standard_normal((66, 64))).astype(np.float32)
    codes[63] = np.nan
    meshes, sdf = mx.solver.mesh(codes, 64, want_sdf=True)
    assert meshes[63][0].shape == (0, 3) and meshes[63][1].shape == (0, 3)
    for i in (0, 62, 64, 65):
        grid = mx.sdf_grid(codes[i])
        assert sdf[i].tobytes() == grid.tobytes()
        _same(meshes[i], _host_mesh(grid))
    # the neighbours of the NaN object are what they are without it
    alone = mx.solver.mesh(codes[[62, 64]], 64)
    _same(meshes[62], alone[0])
    _same(meshes[64], alone[1])


def test_extract_mesh_from_code_without_scikit_image_is_the_old_host_path(golden):
    try:
        import skimage  # noqa: F401
        pytest.skip("scikit-image installed: extract_mesh_from_code uses it")
    except ImportError:
        pass
    mx = _extractor(golden, 32)
    for code in _codes(golden).values():
        m = mx.extract_mesh_from_code(code)
        _same((m.vertices, m.faces), _host_mesh(mx.sdf_grid(code)))
