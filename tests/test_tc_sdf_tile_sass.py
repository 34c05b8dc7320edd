"""The once-per-tile parts of k_gn_persistent's SDF tile, read from the built library (cuobjdump, no GPU).

  * the concat before latent_in and the skip gradient at latent_in are specialised for the fitted decoders (cat_off
    189, a 64-wide code): the whole-code blocks add no branch region, so the kernel keeps the branch-region count of
    the per-element-branch-free epilogues;
  * ptxas keeps the consumer tile loop in registers: the local-memory accesses of the kernel are the ones it had
    before these changes (arguments of the out-of-line solve step, outside the tile loop).
"""
import collections
import os
import re
import shutil
import subprocess

import pytest

BSSY_MAX = 373     # 372 before the specialised concat / skip / layer-0 passes; the general epilogue loops had 755
LOCAL_MAX = 33 + 36   # LDL + STL before these changes


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


def test_branch_regions_within_budget(ops):
    assert ops["BSSY"] <= BSSY_MAX, ops["BSSY"]


def test_no_new_local_memory_traffic(ops):
    assert ops["LDL"] + ops["STL"] <= LOCAL_MAX, (ops["LDL"], ops["STL"])
