"""How the cost of a solver call grows with num_depth_samples (D), per engine:

  reconstruct  LocalMapping's reconstruct_object call: one new car, 250 points + 250 foreground and 200 background rays,
               10 joint iterations (the shape of `bench.py --workload slam1`)
  keyframe     the gated, meshed stereo keyframe of tools/keyframe_bench.py (leg e): 6 tracked cars of which 2 fail the
               map check, 2 new cars, the new objects meshed at voxels_dim 32

for D in --depth-samples (default 50, 64, 128, 256) and engines simt, tc and tc_wide (DeepSDF's 8 x 512 decoder of
tests/wide_fixtures.py, written to a temporary directory).  One solver per (engine, D), all built first; every step runs
each call of every solver once, in turn, so slow drift of the card lands on all of them.  Each call is timed with the
host clock around the whole call (pack + H2D + run + D2H, ending in a stream sync); medians are reported.  The card's
name, power limit and SM clocks are read with nvidia-smi in the same run, before and after the timed loop.

  python tools/depth_samples_bench.py [--steps K] [--warmup W] [--depth-samples 50,64,128,256] [--engines simt,tc,tc_wide]

Prints one JSON line.
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--depth-samples", default="50,64,128,256")
    ap.add_argument("--engines", default="simt,tc,tc_wide")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    if not torch.cuda.is_available():
        raise SystemExit("depth_samples_bench.py needs a CUDA device (no CPU fallback)")
    import keyframe_bench as KB
    import wide_fixtures as WF
    from dsp_slam_b200.optimizer import Optimizer
    Ds = [int(x) for x in args.depth_samples.split(",") if x]
    engines = [e for e in args.engines.split(",") if e]
    tmp = tempfile.mkdtemp(prefix="depth_samples_bench_")
    decoders = {"simt": os.path.join(ROOT, "tests", "golden", "decoder_cars.npz")}
    decoders["tc"] = decoders["simt"]
    if "tc_wide" in engines:
        decoders["tc_wide"] = WF.write("wide", tmp)

    base_cfg, objs, modes = KB.keyframe_inputs()
    tracked, new = objs[:KB.N_TRACKED], objs[KB.N_TRACKED:]
    maps = []
    for i, o in enumerate(tracked):
        M = np.array(o["t_cam_obj"], dtype=np.float32)
        if i < 2:
            M[0, 3] += np.float32(3.0)
        maps.append(M)
    gates = [dict(t_cam_obj_map=M, t_cam_obj_sim3=o["t_cam_obj_sim3"]) for M, o in zip(maps, tracked)] + [None] * KB.N_NEW
    one = new[:1]

    solvers = {}
    for e in engines:
        for D in Ds:
            cfg = copy.deepcopy(base_cfg)
            cfg["optimizer"]["num_depth_samples"] = D
            solvers[(e, D)] = Optimizer(decoders[e], cfg, engine=e).solver
    calls = {"reconstruct": lambda s: s.reconstruct(one),
             "keyframe": lambda s: s.keyframe(objs, modes, gates, voxels_dim=32)}
    times = {(k, e, D): [] for k in calls for (e, D) in solvers}
    card_before = card()
    for step in range(args.warmup + args.steps):
        for (e, D), s in solvers.items():
            for k, fn in calls.items():
                t0 = time.perf_counter()
                fn(s)
                t1 = time.perf_counter()
                if step >= args.warmup:
                    times[(k, e, D)].append((t1 - t0) * 1e3)
    card_after = card()
    rows = {}
    for (k, e, D), t in times.items():
        rows.setdefault(k, {}).setdefault(e, {})[str(D)] = {"median_ms": round(float(np.median(t)), 3),
                                                           "min_ms": round(float(np.min(t)), 3)}
    for (e, D), s in solvers.items():                   # the render rows of the reconstruct call, for the per-D cost
        s.reconstruct(one)
        c = s.counters()
        rows["reconstruct"][e][str(D)]["rows_fwd_only"] = int(c["rows_fwd_only"])
        rows["reconstruct"][e][str(D)]["rows_fwd_bwd"] = int(c["rows_fwd_bwd"])
    print(json.dumps({"metric": "call latency by num_depth_samples (ms)", "steps": args.steps, "warmup": args.warmup,
                      "timing": "host clock around each whole call (ends in a stream sync), calls interleaved, median",
                      "card_before": card_before, "card_after": card_after, "results": rows}), flush=True)


if __name__ == "__main__":
    main()
