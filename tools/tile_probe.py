"""Where a tensor-core tile's cycles go, from a probe build of the library (on an H100).

  python tools/tile_probe.py [--workload cfg2_sdf] [--runs 5] [--sm-budget N] [--out DIR]

Compiles the library with -DDSPGN_STALL_PROBE into DIR (the shipped library is not touched): lane 0 of consumer warp 0
of each warpgroup and the producer lane add the clock64 cycles of each part of the persistent tile loop to per-CTA
counters (dspgn_tc.cuh, ProbeSlot).  Runs the workload `runs` times after a warm-up, then prints the share of the
consumer loop spent in each part, the producer's wait for free ring stages, cycles per tile and per solve, and the card
(name, power limit, max SM clock) read in the same call.  Writes DIR/tile_probe.json.  The probe's clock reads and
counter updates add a little work of their own; the shares are what matter, not the absolute time.
--sm-budget N runs the persistent kernel on N SMs (BatchSolver.debug_sm_budget): half the SMs ask half as much of L2,
so a ring wait that is L2 contention shrinks with the budget, one that is latency does not.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# dspgn_tc.cuh: enum ProbeSlot, kProbeCtas
SLOTS = ["wfull_wait", "wgmma_wait", "gemm", "epilogue", "prologue_layer0", "jtj", "tile_end", "solve", "fifo_wait",
         "loop", "tiles", "solves", "wempty_wait", "pop", "producer_loop", "epi_entry_bar"]
# enum EpiKind; per kind: value loop, store_operand split + stores, store_operand proxy fence + warpgroup barrier
EPI_KINDS = ["fwd", "fwd_concat", "penult", "bwd", "bwd_skip", "bwd_first"]
EPI_PARTS = ["values", "split_store", "fence_bar"]
SLOTS += [f"epi_{k}_{p}" for k in EPI_KINDS for p in EPI_PARTS]
# sub-parts of prologue_layer0 and jtj (J^T r runs on lanes the probe does not read: its excess lands in tile_end)
SUB_PARTS = {"prologue_layer0": ["prologue_global", "prologue_l0"], "jtj": ["jtj_pose", "jtj_loop", "jtj_store"]}
SLOTS += [p for v in SUB_PARTS.values() for p in v]
N_SLOTS, N_CTAS = len(SLOTS), 256


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def build_probe(out):
    import __graft_entry__ as g
    lib = os.path.join(out, "libdspgn_probe.so")
    cmd = [os.environ.get("NVCC", "nvcc")] + g.NVCC_FLAGS + ["-DDSPGN_STALL_PROBE", "-o", lib,
                                                          os.path.join(g.CSRC, "dspgn_api.cu")]
    print("[probe build]", " ".join(cmd), flush=True)
    subprocess.check_call(cmd, cwd=g.CSRC)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2_sdf")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the probe build and tile_probe.json (default: temporary)")
    ap.add_argument("--sm-budget", type=int, default=0, help="SMs of the persistent kernel (default 0: every SM)")
    ap.add_argument("--lib", default=None, help="an existing probe build of this tree to run instead of compiling one")
    args = ap.parse_args()
    out = os.path.abspath(args.out) if args.out else tempfile.mkdtemp(prefix="tile_probe_")
    os.makedirs(out, exist_ok=True)
    from dsp_slam_b200 import _lib
    _lib.LIB_PATH = os.path.abspath(args.lib) if args.lib else build_probe(out)
    import bench
    from dsp_slam_b200.optimizer import Optimizer
    lib = _lib.load()
    lib.dspgn_debug_stall_probe.restype = C.c_int
    lib.dspgn_debug_stall_probe.argtypes = [C.c_int, C.POINTER(C.c_ulonglong), C.c_int]

    B, M, nfg, nbg, cls, cfgname, sdf_only, desc = bench.WORKLOADS[args.workload]
    cfg, ins, clss, sdf_only = bench.make_inputs(args.workload, 1)
    if cls == "mixed":
        raise SystemExit("one decoder class per run: pick a workload other than " + args.workload)
    opt = Optimizer(os.path.join(ROOT, "tests", "golden", f"decoder_{cls}.npz"), cfg, sdf_only=sdf_only, engine="tc")
    opt.solver.upload(ins)
    sms = opt.solver.debug_sm_budget(args.sm_budget)
    modes = [0] * len(ins)
    for _ in range(3):
        opt.solver.run_modes(modes)
        opt.solver.results_raw()
    buf = (C.c_ulonglong * (N_CTAS * 3 * N_SLOTS))()
    lib.dspgn_debug_stall_probe(0, None, 1)
    t0 = time.perf_counter()
    for _ in range(args.runs):
        opt.solver.run_modes(modes)
        opt.solver.results_raw()
    ms = (time.perf_counter() - t0) * 1e3 / args.runs
    lib.dspgn_debug_stall_probe(0, buf, 0)
    gpu = card()
    p = np.array(buf[:], dtype=np.float64).reshape(N_CTAS, 3, N_SLOTS)
    cons = p[:, 0:2, :].sum(axis=(0, 1))       # both consumer warpgroups, every CTA
    prod = p[:, 2, :].sum(axis=0)
    s = dict(zip(SLOTS, cons[:len(SLOTS)]))
    sp = dict(zip(SLOTS, prod[:len(SLOTS)]))
    ctas = int((p[:, 0, SLOTS.index("loop")] > 0).sum())
    loop = s["loop"]
    parts = ["wfull_wait", "wgmma_wait", "epilogue", "prologue_layer0", "jtj", "tile_end", "solve", "fifo_wait"]
    share = {k: s[k] / loop for k in parts}
    share["mma_issue_other"] = (s["gemm"] - s["wfull_wait"] - s["wgmma_wait"]) / loop
    share["unaccounted"] = 1.0 - sum(share.values())
    res = {
        "workload": args.workload, "gpu": gpu, "sm_budget": sms, "ctas": ctas, "runs": args.runs, "ms_per_run_probe_build": ms,
        "tiles_per_run": s["tiles"] / 2 / args.runs, "solves_per_run": s["solves"] / 2 / args.runs,
        "consumer_share": share,
        "cycles_per_tile": {k: s[k] / s["tiles"] for k in parts + ["gemm"]} | {"loop": loop / s["tiles"]},
        "cycles_per_solve": s["solve"] / max(s["solves"], 1),
        "producer_share": {k: sp[k] / max(sp["producer_loop"], 1) for k in ("wempty_wait", "pop")},
        "epilogue_cycles_per_tile": {k: s[k] / s["tiles"] for k in SLOTS if k.startswith("epi_")},
        "sub_part_cycles_per_tile": {p: s[p] / s["tiles"] for v in SUB_PARTS.values() for p in v},
    }
    print(f"{args.workload} on {gpu}: {ctas} CTAs, {res['tiles_per_run']:.0f} tiles and {res['solves_per_run']:.0f} "
          f"solves per run, {ms:.2f} ms per run (probe build)")
    print("consumer loop (warp 0 of each warpgroup), share of cycles / cycles per tile:")
    for k, v in share.items():
        per = res["cycles_per_tile"].get(k, v * loop / s["tiles"])
        print(f"  {k:18s} {100 * v:6.2f} %  {per:10.0f}")
    print(f"  {'loop':18s} {100.0:6.2f} %  {loop / s['tiles']:10.0f}")
    print("prologue and final step by part, cycles per tile:")
    for whole, subs in SUB_PARTS.items():
        print(f"  {whole:18s} " + "  ".join(f"{p} {res['sub_part_cycles_per_tile'][p]:.0f}" for p in subs))
    print("epilogue by step kind, cycles per tile (share of the epilogue):")
    ept = res["epilogue_cycles_per_tile"]
    epi = s["epilogue"] / s["tiles"]
    print(f"  {'entry barrier':18s} {ept['epi_entry_bar']:10.0f}  ({100 * ept['epi_entry_bar'] / epi:5.1f} %)")
    print(f"  {'kind':12s} " + " ".join(f"{p:>12s}" for p in EPI_PARTS) + f" {'total':>12s}")
    for k in EPI_KINDS:
        v = [ept[f"epi_{k}_{p}"] for p in EPI_PARTS]
        print(f"  {k:12s} " + " ".join(f"{x:12.0f}" for x in v) + f" {sum(v):12.0f}  ({100 * sum(v) / epi:5.1f} %)")
    print(f"producer: waiting for free ring stages {100 * res['producer_share']['wempty_wait']:.2f} %, "
          f"popping / FIFO full {100 * res['producer_share']['pop']:.2f} % of its loop")
    print(f"cycles per solve {res['cycles_per_solve']:.0f}")
    with open(os.path.join(out, "tile_probe.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
