"""The epilogues of k_gn_persistent (SDF tiles, the flagship workload), read from the built library (cuobjdump, no GPU).

  * the lo half of every next operand is written with stmatrix (STSM), not with scalar shared-memory stores;
  * no step epilogue has a branch region per fragment element: the concat step before latent_in, the skip-gradient
    step at latent_in and the first layer's backward step each used to add about 128 BSSY / BSYNC pairs to the
    kernel, and together they came to more than 380 of its 755;
  * the fp32 -> fp16 hi / lo split is the same arithmetic as before: one F2FP pack for hi and one for lo per element
    pair, 64 pairs per operand, at each of the four places an operand is built.
"""
import collections
import os
import re
import shutil
import subprocess

import pytest

BSSY_BEFORE = 755          # k_gn_persistent with the general per-element epilogue loops
F2FP = 4 * 64 * 2


@pytest.fixture(scope="module")
def ops():
    from dsp_slam_b200 import _lib
    if shutil.which("cuobjdump") is None or not os.path.isfile(_lib.LIB_PATH):
        pytest.skip("cuobjdump or the built library is not available")
    out = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    per_kernel, kern = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            kern = m.group(1)
            per_kernel[kern] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", line)
        if m and kern:
            per_kernel[kern][m.group(1).split(".")[0]] += 1
    names = [k for k in per_kernel if "k_gn_persistentENS" in k]
    assert len(names) == 1, sorted(per_kernel)
    return per_kernel[names[0]]


def test_lo_image_written_with_stmatrix(ops):
    assert ops["STSM"] > 0, ops["STSM"]


def test_no_branch_region_per_fragment_element(ops):
    assert ops["BSSY"] <= BSSY_BEFORE - 380, ops["BSSY"]


def test_split_arithmetic_unchanged(ops):
    assert ops["F2FP"] == F2FP, ops["F2FP"]
