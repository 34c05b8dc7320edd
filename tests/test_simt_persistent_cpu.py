"""The persistent SIMT kernel k_simt_persistent without a GPU: its machine code in the built library (cuobjdump).
Both instantiations (256 and 512 wide) exist, ptxas reports no spill, and every LDL / STL lies inside the out-of-line
functions the kernel calls (the solve step mega_solve_and_advance and what that calls: their ABI frame and saved
registers), none in the tile loop.
"""
import os
import re
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_wide_persistent_cpu import _cuobjdump  # noqa: E402

WIDTHS = (256, 512)


def _listings():
    """{width: [(address, instruction)]} of k_simt_persistent<width>"""
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
    out = {}
    for w in WIDTHS:
        names = [k for k in per if "k_simt_persistent" in k and f"ILi{w}E" in k]
        assert len(names) == 1, sorted(k for k in per if "simt" in k)
        out[w] = per[names[0]]
    return out


def test_both_instantiations_exist_and_are_simt():
    for w, L in _listings().items():
        ops = [t for _, t in L]
        assert any(re.match(r"(@!?U?P\w+\s+)?FFMA\b", o) for o in ops), w
        assert not any(o.startswith(("HGMMA", "HMMA")) for o in ops), w


@pytest.mark.parametrize("width", WIDTHS)
def test_tile_loop_has_no_local_memory_traffic(width):
    L = _listings()[width]
    calls = sorted({int(re.search(r"CALL\.\S+\s+(0x[0-9a-f]+)", t).group(1), 16) for _, t in L if t.startswith("CALL.")})
    rets = [a for a, t in L if re.search(r"\bRET\b", t)]
    assert calls, "the solve step is an out-of-line call"
    regions = [(c, min(r for r in rets if r >= c)) for c in calls]
    local = [a for a, t in L if re.match(r"(@!?U?P\w+\s+)?(LDL|STL)\b", t)]
    body = [hex(a) for a in local if not any(lo <= a <= hi for lo, hi in regions)]
    assert not body, body[:8]


def test_ptxas_reports_no_spill():
    res = _cuobjdump("-res-usage").splitlines()
    for w in WIDTHS:
        hits = [res[i + 1] for i, ln in enumerate(res) if "Function " in ln and "k_simt_persistent" in ln and f"ILi{w}E" in ln]
        assert len(hits) == 1 and re.search(r"\bLOCAL:0\b", hits[0]), (w, hits)
