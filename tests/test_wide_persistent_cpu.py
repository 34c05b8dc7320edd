"""The persistent wide kernel k_wide_persistent without a GPU: its machine code in the built library (cuobjdump).
Its tile loop keeps everything in registers and shared memory.  Local memory is touched only inside the out-of-line
functions it calls (the solve step mega_solve_and_advance and what that calls: their ABI frame and saved registers),
which k_gn_persistent calls as well.
"""
import os
import re
import shutil
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_wide_tc_cpu import _sass  # noqa: E402


def _cuobjdump(*args):
    from dsp_slam_b200 import _lib
    if shutil.which("cuobjdump") is None or not os.path.isfile(_lib.LIB_PATH):
        pytest.skip("cuobjdump or the built library is not available")
    return subprocess.run(["cuobjdump", *args, _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout


def _listing(kernel):
    """[(address, instruction)] of the one kernel whose name contains `kernel`, called functions included"""
    per, cur = {}, None
    for line in _cuobjdump("-sass").splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            per[cur] = []
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m and cur:
            per[cur].append((int(m.group(1), 16), m.group(2).strip()))
    names = [k for k in per if kernel in k]
    assert len(names) == 1, sorted(per)
    return per[names[0]]


def test_persistent_wide_kernel_is_wgmma_with_bulk_copies():
    ops = _sass("k_wide_persistent")
    assert any(o.startswith("HGMMA") for o in ops)
    assert any(o.startswith("UBLKCP") for o in ops)
    assert not any(o.startswith("HMMA") for o in ops)


def test_persistent_wide_tile_loop_has_no_local_memory_traffic():
    """Every LDL / STL of the kernel lies inside a function it calls ([CALL target, its RET]), none in the kernel body:
    no spill of the tile loop (ptxas: 0 bytes spill; the stack frame is the calls' ABI frame)."""
    L = _listing("k_wide_persistent")
    calls = sorted({int(re.search(r"CALL\.\S+\s+(0x[0-9a-f]+)", t).group(1), 16) for _, t in L if t.startswith("CALL.")})
    rets = [a for a, t in L if re.search(r"\bRET\b", t)]
    assert calls, "the solve step is an out-of-line call"
    regions = [(c, min(r for r in rets if r >= c)) for c in calls]
    local = [a for a, t in L if re.match(r"(@!?U?P\w+\s+)?(LDL|STL)\b", t)]
    body = [hex(a) for a in local if not any(lo <= a <= hi for lo, hi in regions)]
    assert not body, body[:8]
    res = _cuobjdump("-res-usage").splitlines()
    hits = [res[i + 1] for i, ln in enumerate(res) if "Function " in ln and "k_wide_persistent" in ln]
    assert len(hits) == 1 and re.search(r"\bLOCAL:0\b", hits[0]), hits
