"""The LiDAR frame's detection geometry on the CPU: the numpy oracle against the golden made with the unmodified
reference, a model of the device's scalar formulas against numpy, and the ctypes mirror of the C structs."""
import os
import subprocess

import numpy as np
import pytest

import lidar_frame_model as M

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lidar_frames.npz")


def golden_frames(g):
    """Each frame of the golden: (inputs, config, instances) in the oracle's dict form."""
    out = []
    for fi in range(int(g["n_frames"])):
        p = f"f{fi}_"
        nmax, marea, alpha = g[p + "cfg"]
        inp = dict(velo=g[p + "scan"], dets=g[p + "dets"], masks=g[p + "masks"], bboxes=g[p + "bboxes"])
        cfg = dict(num_lidar_max=int(nmax), min_mask_area=int(marea), downsample_ratio=float(alpha))
        inst = []
        for i in range(int(g[p + "n_inst"])):
            q = f"{p}i{i}_"
            d = {k: g[q + k] for k in ("T_cam_obj", "scale", "surface_points")}
            d["is_front"], d["mask_index"] = bool(g[q + "is_front"]), int(g[q + "mask_index"])
            d["num_surface_points"] = int(g[q + "num_surface_points"])
            d["rays"] = g[q + "rays"] if q + "rays" in g else None
            if d["rays"] is not None:
                d["depth"] = g[q + "depth"]
            inst.append(d)
        out.append((inp, cfg, inst))
    return out


def assert_instances_equal(got, want):
    assert len(got) == len(want)
    for a, b in zip(got, want):
        for k in ("T_cam_obj", "scale", "surface_points"):
            assert np.asarray(a[k]).dtype == b[k].dtype, k
            assert np.array_equal(a[k], b[k]), k
        assert a["num_surface_points"] == b["num_surface_points"]
        assert bool(a["is_front"]) == bool(b["is_front"])
        assert int(a["mask_index"]) == int(b["mask_index"])
        assert (a["rays"] is None) == (b["rays"] is None)
        if b["rays"] is not None:
            assert a["rays"].dtype == np.float32 and np.array_equal(a["rays"], b["rays"])
            assert np.array_equal(a["depth"], b["depth"])


def test_oracle_equals_golden():
    from oracle import lidar_frame as O
    g = np.load(GOLDEN)
    hw = g["img_hw"]
    for inp, cfg, want in golden_frames(g):
        got = O.detections(inp["velo"], inp["dets"], inp["masks"], inp["bboxes"], g["K"], g["invK"], g["T_cam_velo"],
                           cfg["num_lidar_max"], cfg["min_mask_area"], cfg["downsample_ratio"], int(hw[0]), int(hw[1]))
        assert_instances_equal(got, want)


def test_golden_covers_the_cases():
    g = np.load(GOLDEN)
    fr = golden_frames(g)
    inst = [(cfg, d) for _, cfg, ds in fr for d in ds]
    n = [d["num_surface_points"] for _, d in inst]
    assert any(cfg["num_lidar_max"] == k for cfg, d in inst for k in [d["num_surface_points"]])   # subsampled boxes
    assert 0 in n and any(0 < k < 250 for k in n)
    assert any(not d["is_front"] for _, d in inst)
    assert any(d["is_front"] and d["mask_index"] < 0 and d["num_surface_points"] > 0 for _, d in inst)
    assert any(d["mask_index"] >= 0 and d["rays"] is None for _, d in inst)
    bg = [d["rays"].shape[0] - d["num_surface_points"] for _, d in inst if d["rays"] is not None]
    assert 200 in bg and any(0 < k < 200 for k in bg) and 0 in bg and 1 in bg
    for _, _, ds in fr:
        m = [d["mask_index"] for d in ds if d["mask_index"] >= 0]
        if len(m) != len(set(m)):
            break
    else:
        pytest.fail("no two boxes match one mask")
    assert any(inp["masks"].shape[0] == 0 for inp, _, _ in fr)
    assert str(g["numpy_version"]).startswith("2.")


def test_device_formulas_match_numpy():
    rng = np.random.default_rng(3)
    # the float32 3-term transforms (scan -> object, scan -> camera, camera -> pixels)
    T = rng.normal(size=(3, 4)).astype(np.float32)
    p = (rng.normal(size=(400, 4)) * 20).astype(np.float32)
    ref = (p[:, None, :3] * T[:, :3]).sum(-1) + T[:, 3]
    got = np.array([M.transform(q, T) for q in p], np.float32)
    assert np.array_equal(got, ref)
    K = np.array([[721.5377, 0, 609.5593], [0, 721.5377, 172.854], [0, 0, 1]], np.float32)
    ph = (ref[:, None, :] * K).sum(-1)
    uv = ph[:, :2] / ph[:, 2, None]
    assert np.array_equal(np.array([M.project(K, q) for q in ref], np.float32), uv)
    # the fp64 rays of float32 pixels and of int32 pixels
    ik = np.linalg.inv(K).astype(np.float32)
    pix = np.concatenate([uv, rng.integers(0, 1242, (50, 2)).astype(np.int32)], 0)
    uh = np.concatenate([pix, np.ones((pix.shape[0], 1))], -1)
    want = (uh[:, None, :] * ik).sum(-1).astype(np.float32)
    assert np.array_equal(np.array([M.ray(ik, u, v) for u, v in pix], np.float32), want)
    # the box test against the oracle's statement of it
    from oracle import lidar_frame as O
    for _ in range(20):
        det = np.concatenate([rng.normal(size=3) * 4, rng.uniform(0.5, 5, 3), rng.uniform(-3.2, 3.2, 1)]).astype(np.float32)
        _, Tov = O.box_matrices(det)
        pts = np.concatenate([det[:3] + rng.normal(size=(300, 3)) * 2.5, rng.random((300, 1))], -1).astype(np.float32)
        sel, _ = O.box_points(pts, det[:3], det[3:6], Tov, 10 ** 9)
        box = dict(trans=det[:3], size=det[3:6], T_obj_velo=Tov[:3])
        mine = pts[[M.selects(box, q) for q in pts]]
        assert np.array_equal(mine, sel)


def test_linspace_branches():
    for start, stop, num in [(0, 10, 0), (3, 9, 1), (5, 5, 7), (0, 1, 2), (12, 311, 74), (7, 200, 33), (0, 99, 100),
                             (0, 123456, 250), (4, 4, 1), (-3, 17, 6)]:
        ref = np.linspace(start, stop, num)
        got = np.array([M.linspace(start, stop, num, i) for i in range(num)], np.float64)
        assert np.array_equal(got, ref), (start, stop, num)
        assert np.array_equal(got.astype(np.int32), ref.astype(np.int32))


def test_subsample_rank_inversion():
    rng = np.random.default_rng(5)
    cases = [(2, 1), (251, 250), (252, 250), (1000, 250), (4097, 4096), (201, 200), (100000, 200), (65, 64)]
    cases += [(int(n), int(m)) for m, n in zip(rng.integers(1, 300, 30), rng.integers(301, 5000, 30))]
    for n, m in cases:
        idx = np.linspace(0, n - 1, m).astype(np.int32)
        slot = np.full(n, -1)
        slot[idx] = np.arange(m)
        got = np.array([M.subsample_slot(r, n, m) for r in range(n)])
        assert np.array_equal(got, slot), (n, m)


def test_ctypes_structs_match_gcc(tmp_path):
    from dsp_slam_b200 import _lib
    src = tmp_path / "layout.c"
    fields = {"DspgnLidarSpec": ["k", "inv_k", "t_cam_velo", "img_h", "img_w", "num_lidar_max", "min_mask_area",
                                "downsample_ratio", "reserved_"],
              "DspgnLidarBox": ["t_obj_velo", "trans", "size", "front"],
              "DspgnLidarBoxOut": ["n_pts", "n_rays", "mask", "n_selected"]}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "dspgn.h"', "int main(void) {"]
    for s, fs in fields.items():
        lines.append(f'  printf("%zu\\n", sizeof({s}));')
        lines += [f'  printf("%zu\\n", offsetof({s}, {f}));' for f in fs]
    lines.append("  return 0;\n}")
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c11", f"-I{os.path.join(ROOT, 'include')}", str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = []
    for s, cls in (("DspgnLidarSpec", _lib.LidarSpec), ("DspgnLidarBox", _lib.LidarBox), ("DspgnLidarBoxOut", _lib.LidarBoxOut)):
        want.append(__import__("ctypes").sizeof(cls))
        want += [getattr(cls, f).offset for f in fields[s]]
    assert got == want


def test_builder_rejects_integer_masks_before_the_device(monkeypatch):
    from dsp_slam_b200 import lidar_frame as LF
    b = LF.LidarFrameBuilder.__new__(LF.LidarFrameBuilder)
    b.img_h, b.img_w = 4, 5
    with pytest.raises(TypeError):
        b.detections(np.zeros((3, 4), np.float32), np.zeros((1, 7), np.float32), np.zeros((1, 4, 5), np.uint8),
                     np.zeros((1, 4), np.float32))


def test_sequence_never_raises(tmp_path, capsys):
    from dsp_slam_b200 import lidar_frame as LF
    (tmp_path / "image_2").mkdir()
    g = np.load(GOLDEN)
    (tmp_path / "calib.txt").write_text(str(g["calib"]))
    seq = LF.KITIISequence(str(tmp_path), dict(detect_online=False, path_label_2d=str(tmp_path), path_label_3d=str(tmp_path),
                                               num_lidar_max=250, min_mask_area=1000, downsample_ratio=4.0))
    assert np.array_equal(seq.K_cam, g["K"]) and np.array_equal(seq.invK_cam, g["invK"])
    assert np.array_equal(seq.T_cam_velo, g["T_cam_velo"])
    assert seq.get_frame_by_id(0) == [] and seq.current_frame is None
