"""The monocular frame's detection on the CPU: the numpy oracle against the golden made with the unmodified reference
and the real cv2, a model of the device's scalar formulas against the installed cv2, the ctypes mirror of the C
structs, and the product's independence from the oracle."""
import os
import subprocess
import sys

import numpy as np
import pytest

import mono_frame_model as M

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "mono_frames.npz")


def golden_frames(g):
    """Each frame of the golden: dict(K, invK, k1, k2, alpha, erosion, hw, masks, bboxes, kp, mask_index, raised,
    background_rays (None unless an instance), feature_idx (None without masks), yaml)."""
    out = []
    for fi in range(int(g["n_frames"])):
        p = f"f{fi}_"
        alpha, e, H, W = (int(v) for v in g[p + "cfg"])
        k1, k2 = (float(v) for v in g[p + "dist"])
        out.append(dict(K=g[p + "K"], invK=g[p + "invK"], k1=k1, k2=k2, alpha=alpha, erosion=e, hw=(H, W),
                        masks=g[p + "masks"], bboxes=g[p + "bboxes"], kp=g[p + "kp"], mask_index=int(g[p + "mask_index"]),
                        raised=str(g[p + "raised"]), n_inst=int(g[p + "n_inst"]),
                        background_rays=g[p + "background_rays"] if p + "background_rays" in g else None,
                        feature_idx=g[p + "feature_idx"] if p + "feature_idx" in g else None, yaml=str(g[p + "yaml"])))
    return out


def test_oracle_equals_golden():
    from oracle import mono_frame as O
    for f in golden_frames(np.load(GOLDEN)):
        d = O.detection(f["masks"], f["bboxes"], f["K"], f["invK"], f["k1"], f["k2"], f["alpha"], *f["hw"])
        if f["mask_index"] < 0:
            assert d is None and f["n_inst"] == 0
            continue
        assert d["mask_index"] == f["mask_index"]
        if f["raised"]:
            assert d["background_rays"] is None and d["n_nonsurface"] < 2 and f["n_inst"] == 0
        else:
            assert f["n_inst"] == 1
            assert d["background_rays"].dtype == np.float32
            assert np.array_equal(d["background_rays"], f["background_rays"])
        m = f["masks"][f["mask_index"]]
        assert np.array_equal(O.feature_points(m, f["kp"], f["erosion"]), f["feature_idx"])


def test_golden_covers_the_cases():
    g = np.load(GOLDEN)
    fr = golden_frames(g)
    from oracle import mono_frame as O
    areas = [f["masks"].sum(-1).sum(-1) for f in fr if f["masks"].shape[0]]
    assert any((a == a.max()).sum() > 1 for a in areas)                         # a tie for the largest mask
    n_bg = [O.detection(f["masks"], f["bboxes"], f["K"], f["invK"], f["k1"], f["k2"], f["alpha"], *f["hw"])["n_nonsurface"]
            for f in fr if f["masks"].shape[0]]
    assert {0, 1, 2} <= set(n_bg) and any(2 < n < 200 for n in n_bg) and any(n > 200 for n in n_bg)
    assert sorted(f["raised"] for f in fr if f["raised"]) == ["ValueError", "error"]   # get_rays; cv2.error
    assert any(f["masks"].shape[0] == 0 for f in fr)
    assert {0, 5, 10, 15} <= {f["erosion"] for f in fr}
    # all four clamp branches of the expanded crop
    lo, hi = set(), set()
    for f in fr:
        if f["mask_index"] < 0:
            continue
        H, W = f["hw"]
        l, t, r, b = f["bboxes"][f["mask_index"]].astype(np.int32)
        lo |= {("l", l <= 5), ("t", t <= 5)}
        hi |= {("r", r >= W - 1 - 5), ("b", b >= H - 1 - 5)}
    assert {("l", True), ("l", False), ("t", True), ("t", False)} <= lo
    assert {("r", True), ("r", False), ("b", True), ("b", False)} <= hi
    # Freiburg's negative k1, Redwood's, and a camera whose border pixels take the icdist < 0 exit
    assert any(f["k1"] < -0.1 for f in fr) and any(f["k1"] > 0 for f in fr)
    neg = [f for f in fr if f["raised"] == "" and f["mask_index"] >= 0 and f["background_rays"] is not None
           and any(M.icdist_negative(f["K"], f["k1"], f["k2"], u, v) for u, v in [(0, 0), (639, 479)])]
    assert neg
    assert str(g["numpy_version"]).startswith("2.") and str(g["cv2_version"]).startswith("4.")


def test_model_undistort_equals_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(8)
    cams = [((538.204343, 538.204343, 320.0, 240.0), 0.023896, -0.067078, (480, 640)),
            ((984.697, 984.697, 480.0, 270.0), -0.133543, -0.15436, (540, 960)),
            ((952.186, 951.0, 478.5, 268.25), -0.13743, -0.127286, (540, 960)),
            ((500.0, 500.0, 320.0, 240.0), -0.9, -0.6, (480, 640)),
            ((525.0, 525.0, 319.5, 239.5), 0.0, 0.0, (480, 640))]
    n_neg = 0
    for (fx, fy, cx, cy), k1, k2, (H, W) in cams:
        K = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])
        pix = np.concatenate([rng.integers(0, [W, H], (600, 2)), [[0, 0], [W - 1, H - 1], [0, H - 1], [W - 1, 0]]]).astype(np.float32)
        want = cv2.undistortPoints(pix.reshape(1, -1, 2), K, np.array([k1, k2, 0.0, 0.0, 0.0]), P=K).reshape(-1, 2)
        got = np.array([M.undistort(K, k1, k2, u, v) for u, v in pix], np.float32)
        assert np.array_equal(got, want), (k1, k2)
        from oracle import mono_frame as O
        assert np.array_equal(O.undistort(pix, K, k1, k2), want)
        n_neg += sum(M.icdist_negative(K, k1, k2, u, v) for u, v in pix)
    assert n_neg > 0


@pytest.mark.parametrize("e", list(range(32)))
def test_model_erosion_equals_cv2(e):
    cv2 = pytest.importorskip("cv2")
    k = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (2 * e + 1, 2 * e + 1), (e, e))
    assert np.array_equal(M.element(e), k)
    rng = np.random.default_rng(100 + e)
    H, W = 90, 120
    v, u = np.mgrid[0:H, 0:W]
    mask = ((u - rng.uniform(20, 100)) / rng.uniform(15, 60)) ** 2 + ((v - rng.uniform(15, 75)) / rng.uniform(15, 50)) ** 2 <= 1
    mask[rng.integers(0, H, 5), rng.integers(0, W, 5)] ^= True
    mask[:, :3] = True                                 # set along the border: the outside is ignored
    er = cv2.erode(mask.astype(np.float32) * 255., k)
    kp = np.concatenate([np.stack([rng.uniform(-0.99, W - 0.01, 300), rng.uniform(-0.99, H - 0.01, 300)], -1),
                         [[0, 0], [W - 0.5, H - 0.5], [0.9, 45.2], [-0.5, 10.0]]]).astype(np.float32)
    want = [int(er[int(y), int(x)]) > 0 for x, y in kp]
    got = [M.inside_eroded(mask, e, x, y) for x, y in kp]
    assert got == want
    from oracle import mono_frame as O
    assert np.array_equal(O.feature_points(mask, kp, e), np.nonzero(want)[0])


def test_ctypes_structs_match_gcc(tmp_path):
    from dsp_slam_b200 import _lib
    src = tmp_path / "layout.c"
    fields = {"DspgnMonoSpec": ["k", "inv_k", "k1", "k2", "img_h", "img_w", "downsample_ratio", "mask_erosion"],
              "DspgnMonoOut": ["mask", "n_nonsurface", "n_rays", "n_feature"]}
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
    for s, cls in (("DspgnMonoSpec", _lib.MonoSpec), ("DspgnMonoOut", _lib.MonoOut)):
        want.append(__import__("ctypes").sizeof(cls))
        want += [getattr(cls, f).offset for f in fields[s]]
    assert got == want


def test_product_never_imports_the_oracle():
    code = ("import sys; import dsp_slam_b200.mono_frame, dsp_slam_b200._lib; "
            "sys.exit(any(m == 'oracle' or m.startswith('oracle.') for m in sys.modules))")
    assert subprocess.run([sys.executable, "-c", code], cwd=ROOT).returncode == 0


def test_builder_rejects_integer_masks_before_the_device():
    from dsp_slam_b200 import mono_frame as MF
    b = MF.MonoFrameBuilder.__new__(MF.MonoFrameBuilder)
    b.img_h, b.img_w = 4, 5
    with pytest.raises(TypeError):
        b.detections(np.zeros((1, 4, 5), np.uint8), np.zeros((1, 4), np.float32))


def test_sequence_reads_the_yaml_and_never_raises(tmp_path):
    pytest.importorskip("cv2")
    from dsp_slam_b200 import mono_frame as MF
    f = golden_frames(np.load(GOLDEN))[1]
    (tmp_path / "image_0").mkdir()
    (tmp_path / "cam.yaml").write_text(f["yaml"])
    seq = MF.MonoSequence(str(tmp_path), dict(detect_online=False, data_type="Freiburg", path_label_2d=str(tmp_path),
                                              slam_config_path=str(tmp_path / "cam.yaml"), downsample_ratio=4.0))
    assert np.array_equal(seq.K_cam, f["K"]) and np.array_equal(seq.invK_cam, f["invK"])
    assert (seq.k1, seq.k2, seq.mask_erosion) == (f["k1"], f["k2"], f["erosion"])
    assert seq.get_frame_by_id(0) == [] and seq.current_frame is None
