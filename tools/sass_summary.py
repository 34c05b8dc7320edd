"""Per-kernel SASS opcode histogram of dsp_slam_b200/libdspgn.so -> profiles/sass_summary.txt
(evidence that the wgmma / bulk-copy / mbarrier path is what the library ships).   python tools/sass_summary.py"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(ROOT, "dsp_slam_b200", "libdspgn.so")
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
KEY = ["UTCHMMA", "UTCQMMA", "LDTM", "STTM", "UTCBAR", "UTCCP", "UBLKCP", "UTMALDG", "UTMASTG", "SYNCS", "WARPGROUP", "HMMA", "HGMMA",
       "FFMA", "DFMA", "LDS", "STS", "LDG", "STG", "LDGSTS", "ATOMG", "RED", "BAR", "SHFL", "MUFU", "LDL", "STL", "NANOSLEEP", "ELECT"]
kern, hist, arch = None, collections.OrderedDict(), set()
for line in out.splitlines():
    m = re.search(r"arch = (sm_\w+)", line)
    if m:
        arch.add(m.group(1))
    m = re.search(r"Function : (\S+)", line)
    if m:
        kern = m.group(1)
        hist[kern] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
    if m and kern:
        hist[kern]["_total"] += 1
        op = m.group(1)
        for k in KEY:
            if op.startswith(k):
                hist[kern][k] += 1
                break
demangle = subprocess.run(["c++filt"], input="\n".join(hist), capture_output=True, text=True).stdout.splitlines()
lines = [f"libdspgn.so SASS summary (cuobjdump -sass; arch: {', '.join(sorted(arch))})",
         "wgmma.mma_async -> HGMMA, wgmma.fence/commit/wait -> WARPGROUP, cp.async.bulk -> UBLKCP, mbarrier -> SYNCS, cp.async -> LDGSTS", ""]
for (k, h), d in zip(hist.items(), demangle):
    name = re.sub(r"\(.*", "", d)
    lines.append(f"{name}: {h['_total']} instructions")
    lines.append("    " + "  ".join(f"{op} {h[op]}" for op in KEY if h[op]))
txt = "\n".join(lines) + "\n"
os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
open(os.path.join(ROOT, "profiles", "sass_summary.txt"), "w").write(txt)
print(txt)
