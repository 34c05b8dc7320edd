"""The wgmma issue sequence of the production tensor-core kernels, read from the built library (cuobjdump, no GPU).

Between the first and the last HGMMA of k_gn_persistent, k_gn_persistent_render and k_decoder_tc:
  * at most one WARPGROUP.DEPBAR per four HGMMAs: the MMAs of a K chunk are issued back to back and retired in groups
    (wgmma.wait_group 1 behind every second ring stage), not one wait per MMA;
  * no local-memory traffic (LDL / STL): the consumer warpgroups hold the accumulator and the register A fragment in
    registers (setmaxnreg), so no spill sits between two MMAs.  k_gn_persistent (SDF tiles only, the flagship
    workload) meets this.  The render-term kernel and the per-iteration kernel carry more per-tile state through the
    step loop and still reload a few scalars (an address, a loop bound) from local memory there: strict xfail.
"""
import os
import re
import shutil
import subprocess

import pytest

KERNELS = ("k_gn_persistent_render", "k_gn_persistentENS", "k_decoder_tc")


def _hgmma_span(kernel):
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
    ops = per_kernel[names[0]]
    idx = [i for i, o in enumerate(ops) if o.startswith("HGMMA")]
    assert idx, names[0]
    return ops[idx[0]:idx[-1] + 1], len(idx)


@pytest.mark.parametrize("kernel", KERNELS)
def test_hgmma_waits_are_batched(kernel):
    span, n_mma = _hgmma_span(kernel)
    depbar = sum(o.startswith("WARPGROUP.DEPBAR") for o in span)
    assert 4 * depbar <= n_mma, (kernel, depbar, n_mma)


@pytest.mark.parametrize("kernel", [
    pytest.param("k_gn_persistent_render", marks=pytest.mark.xfail(strict=True, reason="6 LDL/STL left in the span")),
    "k_gn_persistentENS",
    pytest.param("k_decoder_tc", marks=pytest.mark.xfail(strict=True, reason="4 LDL/STL left in the span")),
])
def test_hgmma_span_has_no_local_memory_traffic(kernel):
    span, _ = _hgmma_span(kernel)
    local = [o for o in span if o.split(".")[0] in ("LDL", "STL")]
    assert not local, (kernel, len(local))
