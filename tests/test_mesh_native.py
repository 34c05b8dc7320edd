"""tests/native/mesh_caller.c: CreateNewMapObjects with the mesh step batched, in plain C against include/dspgn.h.
CPU: it compiles and links.  GPU: its meshes are bit-identical to MeshExtractor.extract_meshes of the same codes."""
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
NATIVE = os.path.join(ROOT, "tests", "native")


def _build(tmp):
    exe = os.path.join(tmp, "mesh_caller")
    libd = os.path.join(ROOT, "dsp_slam_b200")
    subprocess.check_call(["gcc", "-O1", "-std=c11", f"-I{os.path.join(ROOT, 'include')}", os.path.join(NATIVE, "mesh_caller.c"),
                           "-o", exe, f"-L{libd}", "-ldspgn", f"-Wl,-rpath,{libd}"])
    return exe


def test_mesh_caller_compiles_and_links(tmp_path):
    exe = _build(str(tmp_path))
    assert subprocess.run([exe]).returncode == 2           # usage


@pytest.mark.gpu
def test_mesh_caller_matches_extract_meshes(tmp_path, golden_dir):
    from dsp_slam_b200.decoder import DecoderWeights
    from dsp_slam_b200.optimizer import MeshExtractor
    exe = _build(str(tmp_path))
    d = np.load(os.path.join(golden_dir, "recon_kitti250.npz"))
    dec = os.path.join(golden_dir, "decoder_cars.npz")
    w = DecoderWeights.from_npz(dec)
    wp, inp, outp = str(tmp_path / "w.bin"), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(wp, "wb") as f:
        f.write(struct.pack("<3i", len(w.W), w.latent_size, w.latent_in_layer))
        for W, b in zip(w.W, w.b):
            f.write(struct.pack("<2i", *W.shape)); f.write(W.tobytes()); f.write(b.tobytes())
    with open(inp, "wb") as f:
        P = np.asarray(d["in_pts"], np.float32)
        R = np.asarray(d["in_rays"], np.float32)
        dep = np.asarray(d["in_depth"], np.float32)
        f.write(struct.pack("<3i", P.shape[0], R.shape[0], dep.shape[0]))
        for a in (np.asarray(d["in_t_cam_obj"], np.float32), P, R):
            f.write(a.tobytes(order="F"))
        f.write(dep.tobytes())
    r = subprocess.run([exe, wp, inp, "32", outp], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    raw = open(outp, "rb").read()
    n, = struct.unpack_from("<i", raw, 0)
    assert n >= 1
    off = 4 + 4 * n
    codes = np.frombuffer(raw, np.float32, 64 * n, off).reshape(n, 64); off += 256 * n
    nv = np.frombuffer(raw, np.int32, n, off); off += 4 * n
    nf = np.frombuffer(raw, np.int32, n, off); off += 4 * n
    V = np.frombuffer(raw, np.float32, 3 * int(nv.sum()), off).reshape(-1, 3); off += 12 * int(nv.sum())
    F = np.frombuffer(raw, np.int32, 3 * int(nf.sum()), off).reshape(-1, 3)
    ref = MeshExtractor(dec, 64, 32).extract_meshes(codes)
    ov, of = np.concatenate([[0], np.cumsum(nv)]), np.concatenate([[0], np.cumsum(nf)])
    for i in range(n):
        assert V[ov[i]:ov[i + 1]].tobytes() == ref[i].vertices.tobytes()
        assert np.array_equal(F[of[i]:of[i + 1]], ref[i].faces)
    assert nf.sum() > 100
