"""The wide tensor-core engine (DSPGN_ENGINE_TC_WIDE) without a GPU: its step plan and weight images against a numpy
model of the 64B-swizzled K-major fp16 hi / lo images, and the machine code of its kernel k_wide_wgmma in the built
library (cuobjdump).
"""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
NVCC = os.environ.get("NVCC", "nvcc")
# the decoder of tests/native/tc_wide_pack.cu: latent 64, latent_in = 2
IN_DIM, OUT_DIM, LATENT_IN, IN0 = [67, 320, 320, 512, 200], [320, 253, 512, 200, 1], 2, 67
TK_FWD_HIDDEN, TK_FWD_PENULT, TK_BWD_MID, TK_BWD_FIRST = 0, 1, 2, 3


def _model(W):
    """(plan rows, blob) as the engine must build them: forward steps k = 0 .. nl-2 (A = layer input, B = W_k),
    backward steps k = nl-2 .. 0 (A = gradient, B = W_k^T), N padded to 256 or 512 rows, K to whole 64-wide chunks; per
    chunk the images hi[k 0..31], hi[k 32..63], lo[k 0..31], lo[k 32..63], row n's 16-byte groups xor-ed with (n >> 1) & 3."""
    nl = len(W)
    steps, blob = [], bytearray()

    def images(B, n_img, k_steps):
        K = 16 * k_steps
        P = np.zeros((n_img, K), np.float32)
        P[:B.shape[0], :B.shape[1]] = B
        hi = P.astype(np.float16)
        lo = (P - hi.astype(np.float32)).astype(np.float16)
        n = np.arange(n_img)[:, None]
        e = np.arange(32)[None, :]
        dest = (((e >> 3) ^ ((n >> 1) & 3)) << 3) | (e & 7)
        out = bytearray()
        for c in range(k_steps // 4):
            for img, half in ((hi, 0), (hi, 1), (lo, 0), (lo, 1)):
                src = img[:, 64 * c + 32 * half:64 * c + 32 * half + 32]
                sw = np.zeros_like(src)
                np.put_along_axis(sw, np.broadcast_to(dest, src.shape).copy(), src, axis=1)
                out += sw.tobytes()
        return bytes(out)

    def step(kind, k, nout_img, nk, B, cat_off, mask_layer):
        n_mma = 256 if nout_img <= 256 else 512
        k_steps = (-(-nk // 16) + 3) // 4 * 4
        steps.append([kind, n_mma, k_steps, len(blob), k, nout_img, cat_off, mask_layer])
        blob.extend(images(B, n_mma, k_steps))

    for k in range(nl - 1):
        step(TK_FWD_PENULT if k == nl - 2 else TK_FWD_HIDDEN, k, OUT_DIM[k], IN_DIM[k], W[k],
             OUT_DIM[k] if k + 1 == LATENT_IN else -1, -1)
    for k in range(nl - 2, -1, -1):
        step(TK_BWD_FIRST if k == 0 else TK_BWD_MID, k, IN_DIM[k], OUT_DIM[k], W[k].T,
             IN_DIM[k] - IN0 if k == LATENT_IN else -1, k - 1 if k > 0 else -1)
    return steps, bytes(blob)


@pytest.mark.skipif(shutil.which(NVCC) is None, reason="needs nvcc")
def test_wide_packing_matches_the_numpy_model(tmp_path):
    """tcw_plan_decoder (host code, no device) gives exactly the model's plan and bytes; tc_pack_decoder declines the
    same decoder (the 256-wide engine keeps its limit)."""
    rng = np.random.default_rng(7)
    # magnitudes that exercise the lo halves: fp16 hi rounds, lo carries the remainder
    W = [(rng.standard_normal((o, i)) * 0.3).astype(np.float32) for i, o in zip(IN_DIM, OUT_DIM)]
    wpath, opath, exe = str(tmp_path / "w.bin"), str(tmp_path / "out.bin"), str(tmp_path / "tc_wide_pack")
    with open(wpath, "wb") as f:
        for w in W:
            f.write(np.ascontiguousarray(w).tobytes())
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=compute_90a", "-std=c++17",
                           "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "dsp_slam_b200", "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "native", "tc_wide_pack.cu")])
    out = subprocess.run([exe, wpath, opath], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "packed", (out.returncode, out.stdout)
    raw = open(opath, "rb").read()
    n_steps, n_fwd = np.frombuffer(raw[:8], np.int32)
    plan = np.frombuffer(raw[8:8 + 32 * n_steps], np.int32).reshape(n_steps, 8).tolist()
    nbytes = int(np.frombuffer(raw[8 + 32 * n_steps:16 + 32 * n_steps], np.int64)[0])
    blob = raw[16 + 32 * n_steps:]
    want_plan, want_blob = _model(W)
    assert (n_steps, n_fwd) == (8, 4)
    assert plan == want_plan
    assert nbytes == len(blob) == len(want_blob)
    assert blob == want_blob


def _sass(kernel):
    from dsp_slam_b200 import _lib
    if shutil.which("cuobjdump") is None or not os.path.isfile(_lib.LIB_PATH):
        pytest.skip("cuobjdump or the built library is not available")
    out = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    per_kernel, kern = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            kern = m.group(1)
            per_kernel[kern] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", line)
        if m and kern:
            per_kernel[kern].append(m.group(1))
    names = [k for k in per_kernel if kernel in k]
    assert len(names) == 1, sorted(per_kernel)
    return per_kernel[names[0]]


def test_wide_kernel_is_wgmma_with_bulk_copies():
    """k_wide_wgmma issues wgmma (HGMMA, WARPGROUP fences / waits), streams its weights with cp.async.bulk (UBLKCP) and
    has no mma.sync (HMMA)."""
    ops = _sass("k_wide_wgmma")
    assert any(o.startswith("HGMMA") for o in ops)
    assert any(o.startswith("WARPGROUP") for o in ops)
    assert any(o.startswith("UBLKCP") for o in ops)
    assert not any(o.startswith("HMMA") for o in ops)


def test_wide_kernel_has_no_local_memory_traffic():
    """No LDL / STL anywhere in k_wide_wgmma: the accumulator, the epilogue passes and the tile loop live in registers
    and shared memory (ptxas: no spills, no stack frame), not only the span of its MMA issue."""
    ops = _sass("k_wide_wgmma")
    local = [o for o in ops if o.split(".")[0] in ("LDL", "STL")]
    assert not local, len(local)
