"""How much of a keyframe's object work a submitted call hides behind host work (dspgn_keyframe_submit / _wait).

The keyframe is tools/keyframe_bench.py's gated meshed keyframe (6 tracked cars, --rejected of them failing the map
check, and 2 new cars, meshed at each --mesh-dims voxels_dim).  Per dim, alternated in one process:

  blocking      dspgn_keyframe_batch_meshed (host clock around the call)
  submit        the host time of dspgn_keyframe_submit alone (the caller's thread is free again after it)
  overlap X     submit -> X ms of host busy-work -> wait (wall time), for X in --host-ms
  serial X      blocking call -> X ms of host busy-work (wall time): what the caller pays without the split

Ideally overlap X ~ max(X, call) and serial X = X + call.  The records and meshes of submit + wait are compared with the
blocking call's bit for bit.  Prints one JSON line with the card's name and power limit.

  python tools/async_bench.py [--steps K] [--warmup W] [--engine auto|simt|tc] [--schedule auto|launches|persistent]
                              [--rejected K] [--mesh-dims 32,64] [--host-ms 0,5,10,20]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def spin(ms):
    """Host busy-work for ms milliseconds (the mapping steps a LocalMapping thread runs meanwhile)."""
    end = time.perf_counter() + ms * 1e-3
    while time.perf_counter() < end:
        pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--engine", default="auto", choices=["auto", "simt", "tc"])
    ap.add_argument("--schedule", default="auto", choices=["auto", "launches", "persistent"])
    ap.add_argument("--rejected", type=int, default=2)
    ap.add_argument("--mesh-dims", default="32,64")
    ap.add_argument("--host-ms", default="0,5,10,20")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    from dsp_slam_b200 import _lib
    from dsp_slam_b200.optimizer import Optimizer
    from keyframe_bench import N_NEW, N_TRACKED, gpu_card, keyframe_inputs
    if not torch.cuda.is_available():
        raise SystemExit("async_bench.py needs a CUDA device (no CPU fallback)")
    cfg, objs, modes = keyframe_inputs()
    tracked = objs[:N_TRACKED]
    maps = []
    for i, o in enumerate(tracked):
        M = np.array(o["t_cam_obj"], dtype=np.float32)
        if i < args.rejected:
            M[0, 3] += np.float32(3.0)
        maps.append(M)
    gates = [dict(t_cam_obj_map=M, t_cam_obj_sim3=o["t_cam_obj_sim3"]) for M, o in zip(maps, tracked)] + [None] * N_NEW
    opt = Optimizer(os.path.join(ROOT, "tests", "golden", "decoder_cars.npz"), cfg,
                    engine=None if args.engine == "auto" else args.engine,
                    schedule=None if args.schedule == "auto" else args.schedule)
    s = opt.solver
    n = len(objs)
    dims = [int(x) for x in args.mesh_dims.split(",") if x]
    xs = [float(x) for x in args.host_ms.split(",") if x]

    def rec(out):
        return np.frombuffer(out, dtype=np.uint32, count=n * _lib.RESULT_FLOATS).copy()

    def same(a, b):
        return bool(np.array_equal(rec(a[0]), rec(b[0]))) and all(
            (x is None) == (y is None) and (x is None or (np.array_equal(x[0].view(np.uint32), y[0].view(np.uint32))
                                                          and np.array_equal(x[1], y[1]))) for x, y in zip(a[1], b[1]))

    legs, identical = {}, True
    for dim in dims:
        t_block, t_submit = [], []
        t_over, t_serial = {x: [] for x in xs}, {x: [] for x in xs}
        for step in range(args.warmup + args.steps):
            t0 = time.perf_counter(); want = s.keyframe(objs, modes, gates, voxels_dim=dim); t1 = time.perf_counter()
            s.keyframe_submit(objs, modes, gates, voxels_dim=dim); t2 = time.perf_counter()
            got = s.keyframe_wait()
            identical = identical and same(got, want)
            timed = step >= args.warmup
            if timed:
                t_block.append((t1 - t0) * 1e3); t_submit.append((t2 - t1) * 1e3)
            for x in xs:
                t0 = time.perf_counter()
                s.keyframe_submit(objs, modes, gates, voxels_dim=dim)
                spin(x)
                s.keyframe_wait()
                t1 = time.perf_counter()
                s.keyframe(objs, modes, gates, voxels_dim=dim)
                spin(x)
                t2 = time.perf_counter()
                if timed:
                    t_over[x].append((t1 - t0) * 1e3); t_serial[x].append((t2 - t1) * 1e3)
        med = lambda t: float(np.median(t))
        legs[f"dim{dim}"] = {
            "blocking_ms": med(t_block), "submit_host_ms": med(t_submit),
            "overlap": {f"X={x:g}ms": {"submit_X_wait_ms": med(t_over[x]), "blocking_plus_X_ms": med(t_serial[x]),
                                      "saved_ms": med(t_serial[x]) - med(t_over[x])} for x in xs},
            "meshes": sum(m is not None for m in want[1])}
    print(json.dumps({
        "metric": "keyframe call hidden behind host work", "unit": "ms",
        "steps": args.steps, "warmup": args.warmup, "engine": {1: "simt-fp32", 2: "wgmma-3xf16"}[s.engine],
        "schedule": args.schedule,
        "workload": f"{N_TRACKED} tracked cars ({args.rejected} rejected by the map check) + {N_NEW} new cars, meshed",
        "timing": "host clock, medians; legs alternated in one process",
        "card": gpu_card(), "legs": legs, "records_and_meshes_identical": identical,
    }), flush=True)


if __name__ == "__main__":
    main()
