"""The machine code of the three kernels built from the tensor-core tile body (tc_body in dspgn_tc.cuh), read from the
built library (cuobjdump, no GPU).  k_decoder_tc runs the per-iteration schedule and the mesh grid decode,
k_gn_persistent the SDF-only and pose-only persistent runs, k_gn_persistent_render the joint runs with the render term.

  * the MMAs of a K chunk are issued back to back and retired in groups (wgmma.wait_group 1 behind every second ring
    stage), not one wait per MMA: at most one WARPGROUP.DEPBAR per four HGMMAs between the first and the last HGMMA;
  * no local-memory traffic (LDL / STL) between the first and the last HGMMA: the consumer warpgroups hold the
    accumulator and the register A fragment in registers (setmaxnreg), so no spill sits between two MMAs;
  * the lo half of every next operand is written with stmatrix (STSM), not with scalar shared-memory stores;
  * the fp32 -> fp16 hi / lo split is one F2FP pack for hi and one for lo per element pair, 64 pairs per operand, at
    each of the four places an operand is built;
  * no step epilogue has a branch region per fragment element, and ptxas keeps the consumer tile loop in registers:
    the branch regions (BSSY) and local-memory accesses of each kernel stay within the counts below.  The general
    per-element epilogue loops these kernels used to run had 755 BSSY in k_gn_persistent alone.
"""
import collections
import os
import re
import shutil
import subprocess

import pytest

F2FP = 4 * 64 * 2
# kernel: (BSSY, LDL + STL) ceilings of the whole kernel
LIMITS = {
    "k_decoder_tc": (111, 47 + 33),
    "k_gn_persistent": (373, 33 + 36),
    "k_gn_persistent_render": (638, 214 + 102),
}


@pytest.fixture(scope="module")
def sass():
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
    return per_kernel


def _ops(sass, kernel):
    names = [k for k in sass if f"{len(kernel)}{kernel}E" in k]     # the mangled name of dspgn::<kernel>
    assert len(names) == 1, (kernel, sorted(sass))
    return sass[names[0]]


def _hgmma_span(ops):
    idx = [i for i, o in enumerate(ops) if o.startswith("HGMMA")]
    assert idx
    return ops[idx[0]:idx[-1] + 1], len(idx)


def _counts(ops):
    return collections.Counter(o.split(".")[0] for o in ops)


@pytest.mark.parametrize("kernel", LIMITS)
def test_hgmma_waits_are_batched(sass, kernel):
    span, n_mma = _hgmma_span(_ops(sass, kernel))
    depbar = sum(o.startswith("WARPGROUP.DEPBAR") for o in span)
    assert 4 * depbar <= n_mma, (kernel, depbar, n_mma)


@pytest.mark.parametrize("kernel", LIMITS)
def test_hgmma_span_has_no_local_memory_traffic(sass, kernel):
    span, _ = _hgmma_span(_ops(sass, kernel))
    local = [o for o in span if o.split(".")[0] in ("LDL", "STL")]
    assert not local, (kernel, len(local))


@pytest.mark.parametrize("kernel", LIMITS)
def test_lo_image_written_with_stmatrix(sass, kernel):
    c = _counts(_ops(sass, kernel))
    assert c["STSM"] > 0, (kernel, c["STSM"])


@pytest.mark.parametrize("kernel", LIMITS)
def test_split_arithmetic_unchanged(sass, kernel):
    c = _counts(_ops(sass, kernel))
    assert c["F2FP"] == F2FP, (kernel, c["F2FP"])


@pytest.mark.parametrize("kernel", LIMITS)
def test_branch_regions_within_budget(sass, kernel):
    c = _counts(_ops(sass, kernel))
    assert c["BSSY"] <= LIMITS[kernel][0], (kernel, c["BSSY"])


@pytest.mark.parametrize("kernel", LIMITS)
def test_local_memory_within_budget(sass, kernel):
    c = _counts(_ops(sass, kernel))
    assert c["LDL"] + c["STL"] <= LIMITS[kernel][1], (kernel, c["LDL"], c["STL"])
