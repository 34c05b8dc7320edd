"""Event timeline of the persistent kernel (env DSPGN_CLK): where one GN iteration of one object spends its time.
   python tools/mega_timeline.py [slam1|cfg3|cfg2_sdf|cfg2_full|keyframe]   (on an H100)"""
import os, sys, ctypes as C
os.environ["DSPGN_CLK"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import bench
from dsp_slam_b200 import _lib
from dsp_slam_b200.optimizer import Optimizer

wl = sys.argv[1] if len(sys.argv) > 1 else "slam1"
if wl == "keyframe":                # tracked objects pose-only + new objects joint, one run (tools/keyframe_bench.py)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import keyframe_bench
    cfg, ins, modes = keyframe_bench.keyframe_inputs()
    cls, sdf_only = "cars", False
else:
    B, M, nfg, nbg, cls, cfgname, sdf_only, desc = bench.WORKLOADS[wl]
    cfg, ins, clss, sdf_only = bench.make_inputs(wl, 1)
    modes = [0] * len(ins)
opt = Optimizer(os.path.join(ROOT, "tests", "golden", f"decoder_{cls}.npz"), cfg, sdf_only=sdf_only, engine="tc")
opt.solver.upload(ins)
for _ in range(3):
    opt.solver.run_modes(modes); opt.solver.results_raw()
cap = 1 << 18
buf = (C.c_longlong * (2 * cap))()
n = _lib.load().dspgn_debug_events(opt.solver.handle, buf, cap)
ev = np.array(buf[:2 * n], dtype=np.int64).reshape(n, 2)
t = ev[:, 0] - ev[:, 0].min()
d = ev[:, 1]
kind, mode, sm, o, tile = d >> 56, (d >> 52) & 15, (d >> 40) & 4095, (d >> 24) & 65535, d & 0xFFFFFF
K = ["tile_begin", "tile_end", "scan_begin", "scan_end", "solve_begin", "solve_end", "popped", "first_mma"]
MODE = {0: "SDF", 1: "BAND", 2: "RAY", 3: "SCAN"}
print(f"{wl}: {n} events, kernel span {t.max() / 1e3:.1f} us")
for m_, name in ((1, "pose-only"), (0, "joint")):
    objs_m = [i for i, x in enumerate(modes) if x == m_]
    if objs_m:
        fin = t[(kind == 5) & np.isin(o, objs_m)]
        print(f"{name} objects ({len(objs_m)}): last solve ends at {fin.max() / 1e3:.1f} us")
obj = 0
sel = o == obj
sb, se = np.sort(t[sel & (kind == 4)]), np.sort(t[sel & (kind == 5)])
prev_end = 0
print("object 0, per iteration (us): ray first-begin..last-end | scan | band begin..end | sdf begin..end | solve | iteration span")
for it in range(len(sb)):
    lo, hi = prev_end, se[it]
    w = sel & (t >= lo) & (t <= hi)
    def span(md, k0=0, k1=1):
        a = t[w & (mode == md) & (kind == k0)]; b = t[w & (mode == md) & (kind == k1)]
        return (a.min() / 1e3 if len(a) else -1, b.max() / 1e3 if len(b) else -1, len(a))
    ray, band, sdf = span(2), span(1), span(0)
    fm = t[w & (mode == 2) & (kind == 7)]
    scb, sce = t[w & (mode == 3) & (kind == 0)], t[w & (mode == 3) & (kind == 1)]
    print(f" it{it}: t0={lo/1e3:8.1f} ray[{ray[2]:4d}] {ray[0]-lo/1e3:6.1f}..{ray[1]-lo/1e3:6.1f} (first mma +{(fm.min()-lo)/1e3 if len(fm) else -1:5.1f}) | scan "
          f"{(scb.min()-lo)/1e3 if len(scb) else -1:6.1f}..{(sce.max()-lo)/1e3 if len(sce) else -1:6.1f} | band[{band[2]}] {band[0]-lo/1e3:6.1f}..{band[1]-lo/1e3:6.1f} | "
          f"sdf[{sdf[2]}] {sdf[0]-lo/1e3:6.1f}..{sdf[1]-lo/1e3:6.1f} | solve {(sb[it]-lo)/1e3:6.1f}..{(se[it]-lo)/1e3:6.1f} | span {(hi-lo)/1e3:6.1f}")
    prev_end = hi
# tile durations by kind
for md in (0, 1, 2, 3):
    dur = []
    for s_ in np.unique(sm):
        m_ = (sm == s_) & (mode == md)
        b_ = np.sort(t[m_ & (kind == 0)]); e_ = np.sort(t[m_ & (kind == 1)])
        k = min(len(b_), len(e_))
        dur += list((e_[:k] - b_[:k]) / 1e3)
    if dur:
        print(f"{MODE[md]} tiles: n={len(dur)} median {np.median(dur):.1f} us  p10 {np.percentile(dur,10):.1f} p90 {np.percentile(dur,90):.1f}")

# solve phases (kind 8: phase index in the tile field): 0 start, 1 loss reductions, 2 rotation prior, 3 tile partials, 4 system in smem,
# 5 elimination done, 6 update / record done
ph = kind == 8
if ph.any():
    names = ["loss-reductions", "rot-prior", "tile-partials", "assemble", "gauss-jordan", "update+record"]
    acc = {n: [] for n in names}
    for s_ in np.unique(sm[ph]):
        m_ = ph & (sm == s_)
        tt, pp = t[m_], tile[m_]
        order = np.argsort(tt)
        tt, pp = tt[order], pp[order]
        for i in range(len(tt) - 1):
            if pp[i + 1] == pp[i] + 1 and pp[i] < 6:
                acc[names[pp[i]]].append((tt[i + 1] - tt[i]) / 1e3)
    print("solve phases (us, median over all solves): " + "  ".join(f"{n} {np.median(v):.1f}" for n, v in acc.items() if v))
