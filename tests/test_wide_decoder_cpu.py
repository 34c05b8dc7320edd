"""Decoders with layers wider than 256, without a GPU: the numpy oracle against the reference's goldens of DeepSDF's own
8 x 512 network and of a 512-wide LayerNorm + xyz_in_all variant (both built by tests/wide_fixtures.py), at the levels
of test_oracle_vs_golden.py; the width limit of the C ABI's spec check; and tc_pack_decoder declining a 512-wide
decoder.
"""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import teacher_states as TS  # noqa: E402
import test_oracle_vs_golden as OVG  # noqa: E402
import wide_fixtures as WF  # noqa: E402

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
WIDE_RUN = ("states_wide", "recon_wide", "wide", "kitti", 10, False, False)


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.fixture(scope="module")
def wide_files(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("wide_decoders"))
    return {n: WF.write(n, d) for n in WF.BUILDERS}


@pytest.fixture(scope="module")
def wide(oracle, wide_files):
    return {n: oracle.DecoderWeights.from_npz(p) for n, p in wide_files.items()}


@pytest.mark.parametrize("name,golden", [("wide", "wide_stages"), ("wide_variant", "wide_variant")])
def test_fixture_weights_are_those_of_the_goldens(name, golden, golden_dir):
    """The construction gives, bit for bit, the weights the reference's goldens were made from."""
    assert WF.digest(WF.BUILDERS[name]()[1]) == str(np.load(os.path.join(golden_dir, golden + ".npz"))["weights_sha256"])


def test_wide_fixture_is_deepsdf_8x512(wide, wide_files):
    dw = wide["wide"]
    assert dw.num_linear == 9 and dw.latent_in == (4,) and dw.latent_size == 64
    assert [w.shape for w in dw.W] == [(512, 67)] + [(512, 512)] * 2 + [(445, 512)] + [(512, 512)] * 4 + [(1, 512)]
    assert all(w.dtype == np.float32 for w in dw.W)
    from dsp_slam_b200.decoder import DecoderWeights
    pw = DecoderWeights.from_npz(wide_files["wide"])     # the product's own ingest
    assert pw.latent_in == (4,) and all(np.array_equal(a, b) for a, b in zip(pw.W + pw.b, dw.W + dw.b))
    v = wide["wide_variant"]
    assert v.xyz_in_all and sum(x is not None for x in v.ln) == 2 and max(max(w.shape) for w in v.W) == 512


@pytest.mark.parametrize("name,golden,tol", [("wide", "wide_stages", (2e-7, 2e-6, 2e-6, 2e-5)),
                                             ("wide_variant", "wide_variant", (2e-6, 5e-6, 1e-5, 2e-5))])
def test_stages_vs_reference(oracle, wide, golden_dir, name, golden, tol):
    """Forward, input Jacobian, SDF-term rows and render band rows at one state, against the reference's."""
    st = np.load(os.path.join(golden_dir, golden + ".npz"))
    dw = wide[name]
    t_y, t_g, t_J, t_rJ = tol
    np.testing.assert_allclose(oracle.decoder_forward(dw, st["dec_in"]), st["dec_y"], rtol=0, atol=max(t_y, 2e-7))
    y, g = oracle.decoder_value_and_input_grad(dw, st["dec_in"])
    np.testing.assert_allclose(y, st["jac_y"], rtol=0, atol=max(t_y, 2e-7))
    assert rel(g, st["jac_g"]) < t_g
    J, res = oracle.sdf_term(dw, st["sdf_pts"], st["sdf_t_obj_cam"], st["sdf_z"])
    assert rel(J, st["sdf_J"]) < t_J
    np.testing.assert_allclose(res, st["sdf_res"], rtol=0, atol=3e-6)
    r = oracle.render_term(dw, st["rnd_rays"], st["rnd_depth_obs"], st["sdf_t_obj_cam"], st["rnd_depths"], st["sdf_z"], 0.01)
    assert r is not None
    J, res, _ = r
    assert J.shape == st["rnd_J"].shape and J.shape[0] > 0     # same band rows kept, same order
    assert rel(J, st["rnd_J"]) < t_rJ
    np.testing.assert_allclose(res, st["rnd_res"], rtol=0, atol=1e-5)


def test_whole_joint_run(oracle, wide, cfg_kitti, cfg_redwood, golden_dir):
    """recon_wide.npz (KITTI hyper-parameters, render term, 10 iterations) at the levels of recon_kitti250."""
    OVG.test_whole_runs(oracle, wide, cfg_kitti, cfg_redwood, golden_dir, "recon_wide", "wide", "kitti", 10, False, False,
                        3e-2, 1.5e-2)


def test_pose_only_run(oracle, wide, cfg_kitti, golden_dir):
    d = np.load(os.path.join(golden_dir, "pose_only_wide.npz"))
    cfg = oracle.GNConfig.from_json_dict(cfg_kitti)
    T = oracle.estimate_pose_cam_obj(wide["wide"], cfg, d["in_t_co_se3"], float(d["in_scale"]), d["in_pts"], d["in_code"])
    np.testing.assert_allclose(T, d["t_cam_obj"], rtol=0, atol=2e-5)


def test_teacher_forced_states(oracle, wide, cfg_kitti, cfg_redwood, monkeypatch):
    """One oracle iteration from every state of the reference's wide joint run (states_wide.npz), as
    test_oracle_vs_golden.test_teacher_forced_states_vs_reference does for the 256-wide runs."""
    monkeypatch.setattr(TS, "STATE_RUNS", TS.STATE_RUNS + [WIDE_RUN])
    OVG.test_teacher_forced_states_vs_reference(oracle, wide, cfg_kitti, cfg_redwood, "states_wide")


def _spec(width):
    from dsp_slam_b200 import _lib
    spec = _lib.DecoderSpec()
    spec.latent_size = 64; spec.num_linear = 3; spec.latent_in_layer = -1
    dims = [(67, width), (width, width), (width, 1)]
    for k, (i, o) in enumerate(dims):
        spec.in_dim[k], spec.out_dim[k] = i, o
    W = [np.zeros((o, i), np.float32) for i, o in dims]
    b = [np.zeros(o, np.float32) for _, o in dims]
    return spec, W, b


def test_spec_check_accepts_512_and_rejects_513():
    """Layers up to 512 wide pass the spec check (then, without a device, creation stops at DSPGN_E_NOGPU); 513 is
    DSPGN_E_ARG with the limit in the message."""
    from dsp_slam_b200 import _lib
    lib = _lib.load()
    FP = C.POINTER(C.c_float)
    for width, want in ((512, None), (513, -1)):
        spec, W, b = _spec(width)
        Wp = (FP * 3)(*[w.ctypes.data_as(FP) for w in W]); bp = (FP * 3)(*[x.ctypes.data_as(FP) for x in b])
        h = C.c_void_p()
        rc = lib.dspgn_decoder_create(C.byref(spec), Wp, bp, 0, C.byref(h))
        if want is None:
            assert rc != -1, lib.dspgn_last_error()
            if rc == 0:
                lib.dspgn_decoder_destroy(h)
        else:
            assert rc == want and b"[1,512]" in lib.dspgn_last_error()


@pytest.mark.skipif(shutil.which(os.environ.get("NVCC", "nvcc")) is None, reason="needs nvcc")
def test_tc_pack_declines_wide_decoders(tmp_path):
    """tc_pack_decoder leaves a 512-wide (and a 257-wide) plain decoder to the SIMT engine: no truncated wgmma images."""
    exe = str(tmp_path / "tc_pack_wide")
    subprocess.check_call([os.environ.get("NVCC", "nvcc"), "-gencode", "arch=compute_90a,code=compute_90a", "-std=c++17",
                           "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "dsp_slam_b200", "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "native", "tc_pack_wide.cu")])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "declined", out.stdout
