"""What the frame-handle SM reserve costs a throughput workload: bench.py's workloads at a forced SM budget.

While a frame handle (LidarFrameBuilder / MonoFrameBuilder) is alive, the solver's grid-sized launches use
DSPGN_FRAME_RESERVE_SMS fewer SMs than the device has.  This runs bench.py's inputs for each workload (same objects, same
config, same L2 flush between steps, device events around each run) with the budget forced through
dspgn_debug_sm_budget to every SM and to k SMs fewer (k = 4, 8, 16), alternated step by step in one process.  The
records of every budget are compared bit for bit with the full budget's.  Prints one JSON line per workload with medians
and p10-p90 in ms, and the card's name, power limit and max SM clock read in the same run.

  python tools/budget_bench.py [--workload cfg2_sdf slam1] [--steps K] [--warmup W] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

RESERVES = (0, 4, 8, 16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=["cfg2_sdf", "slam1"])
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("budget_bench.py needs a CUDA device (no CPU fallback)")
    import __graft_entry__ as g
    g.build()
    from bench import WORKLOADS, make_inputs
    from dsp_slam_b200.optimizer import Optimizer
    from frame_bench import card, stats
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    stream = torch.cuda.current_stream()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    lines = []
    for wl in args.workload:
        cls = WORKLOADS[wl][4]
        cfg, ins, _, sdf_only = make_inputs(wl, 1)
        opt = Optimizer(os.path.join(ROOT, "tests", "golden", f"decoder_{cls}.npz"), cfg, sdf_only=sdf_only)
        s = opt.solver
        s.set_stream(stream.cuda_stream)
        s.upload(ins)
        t = {k: [] for k in RESERVES}
        ref, same = None, {k: True for k in RESERVES}
        for step in range(args.warmup + args.steps):
            order = RESERVES[step % len(RESERVES):] + RESERVES[:step % len(RESERVES)]
            for k in order:
                s.debug_sm_budget(n_sms - k)
                flush.fill_(1)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                s.run(0)
                b.record(stream)
                rec = np.frombuffer(s.results_raw(), np.uint32).copy()
                if k == 0 and ref is None:
                    ref = rec
                elif ref is not None:
                    same[k] &= bool(np.array_equal(rec, ref))
                if step >= args.warmup:
                    t[k].append(a.elapsed_time(b))
        s.debug_sm_budget(None)
        base = float(np.median(t[0]))
        res = {"workload": wl, "card": card(), "sms": n_sms,
               "budgets": {f"{n_sms - k}": dict(stats(t[k]), ratio_to_all_sms=float(np.median(t[k])) / base,
                                                 records_equal=same[k]) for k in RESERVES}}
        lines.append(json.dumps(res))
        print(lines[-1], flush=True)
        s.close()
    if args.out:
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
