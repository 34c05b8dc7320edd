"""How long a stopped keyframe call keeps its caller waiting (dspgn_keyframe_stop, LocalMapping's mbAbortBA).

The keyframe is tools/keyframe_bench.py's gated keyframe (6 tracked cars, --rejected of them failing the map check, 2 new
cars, 10 joint iterations) meshed at --dim.  Per schedule, alternated in one process:

  unstopped   submit -> wait (host clock): what LocalMapping waits for today
  stop X      submit -> X ms of host spin -> dspgn_keyframe_stop -> wait; reported: the time from the stop request to
              wait returning, the objects that ended STOPPED, and what the unstopped call still had left at X
  flag X      a registered flag byte (dspgn_solver_set_stop_flag) raised by a second thread X ms after the submit while
              wait polls it: the time from raising the flag to wait returning (steps in which something stopped)
Also what a timed 20 us sleep between polls would cost on the same host (one event query plus the sleep, from Python).

Every stopped call's records are checked against the unstopped call's: an object that did not stop is bit-identical.
Prints one JSON line with the card's name, power limit and SM clocks.

  python tools/stop_bench.py [--steps K] [--warmup W] [--legs tc:persistent,simt:launches,simt:persistent] [--dim 32]
                             [--delays-ms 0.5,2,5] [--rejected 2]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def spin(ms):
    end = time.perf_counter() + ms * 1e-3
    while time.perf_counter() < end:
        pass


def clocks():
    """Current and maximum SM clock of the card (MHz), read in the same process as the measurement."""
    try:
        import torch
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        cur, mx = (float(x) for x in q.stdout.strip().splitlines()[0].split(","))
        return {"sm_clock_mhz": cur, "sm_clock_max_mhz": mx}
    except Exception:
        return {"sm_clock_mhz": None, "sm_clock_max_mhz": None}


def sleep_20us(n=2000):
    """What a timed 20 us sleep between polls would cost on this host: one CUDA event query plus time.sleep(20e-6) (the
    same clock_nanosleep and timer slack, plus Python's overhead).  p50 / p99 / max in microseconds.  The library's wait
    yields instead of sleeping for this reason."""
    import torch
    ev = torch.cuda.Event()
    ev.record()
    torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        t0 = time.perf_counter()
        ev.query()
        time.sleep(20e-6)
        ts.append((time.perf_counter() - t0) * 1e6)
    return {"p50": float(np.percentile(ts, 50)), "p99": float(np.percentile(ts, 99)), "max": float(np.max(ts))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--legs", default="tc:persistent,simt:launches,simt:persistent")
    ap.add_argument("--dim", type=int, default=32)
    ap.add_argument("--delays-ms", default="0.5,2,5")
    ap.add_argument("--rejected", type=int, default=2)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    from dsp_slam_b200 import _lib
    from dsp_slam_b200.optimizer import Optimizer
    from keyframe_bench import N_NEW, N_TRACKED, gpu_card, keyframe_inputs
    if not torch.cuda.is_available():
        raise SystemExit("stop_bench.py needs a CUDA device (no CPU fallback)")
    cfg, objs, modes = keyframe_inputs()
    tracked = objs[:N_TRACKED]
    maps = []
    for i, o in enumerate(tracked):
        M = np.array(o["t_cam_obj"], dtype=np.float32)
        if i < args.rejected:
            M[0, 3] += np.float32(3.0)
        maps.append(M)
    gates = [dict(t_cam_obj_map=M, t_cam_obj_sim3=o["t_cam_obj_sim3"]) for M, o in zip(maps, tracked)] + [None] * N_NEW
    n = len(objs)
    delays = [float(x) for x in args.delays_ms.split(",") if x]

    def rec(out):
        return np.frombuffer(out, dtype=np.uint32, count=n * _lib.RESULT_FLOATS).reshape(n, -1).copy()

    legs, consistent = {}, True
    for leg in args.legs.split(","):
        engine, schedule = leg.split(":")
        opt = Optimizer(os.path.join(ROOT, "tests", "golden", "decoder_cars.npz"), cfg, engine=engine, schedule=schedule)
        s = opt.solver
        t_full = []
        lat = {x: [] for x in delays}
        left = {x: [] for x in delays}
        n_stopped = {x: [] for x in delays}
        flag_lat = {x: [] for x in delays}
        want = None
        for step in range(args.warmup + args.steps):
            timed = step >= args.warmup
            t0 = time.perf_counter()
            s.keyframe_submit(objs, modes, gates, voxels_dim=args.dim)
            out, _ = s.keyframe_wait()
            t1 = time.perf_counter()
            want = rec(out)
            full = (t1 - t0) * 1e3
            if timed:
                t_full.append(full)
            for x in delays:
                t0 = time.perf_counter()
                s.keyframe_submit(objs, modes, gates, voxels_dim=args.dim)
                spin(x)
                t1 = time.perf_counter()
                s.request_stop()
                out, _ = s.keyframe_wait()
                t2 = time.perf_counter()
                got = rec(out)
                st = got.view(np.int32)[:, 81]
                stopped = st == _lib.ST_STOPPED
                consistent = consistent and bool(np.array_equal(got[~stopped], want[~stopped]))
                if timed:
                    lat[x].append((t2 - t1) * 1e3)
                    left[x].append(max(full - (t1 - t0) * 1e3, 0.0))
                    n_stopped[x].append(int(stopped.sum()))
                # the same stop through a registered flag raised by another thread while the wait polls it
                flag = C.c_uint8(0)
                s.set_stop_flag(C.addressof(flag))
                t_set = []
                th = threading.Thread(target=lambda: (time.sleep(x * 1e-3), t_set.append(time.perf_counter()),
                                                      setattr(flag, "value", 1)))
                s.keyframe_submit(objs, modes, gates, voxels_dim=args.dim)
                th.start()
                out, _ = s.keyframe_wait()
                t2 = time.perf_counter()
                th.join()
                s.set_stop_flag(None)
                got = rec(out)
                stopped = got.view(np.int32)[:, 81] == _lib.ST_STOPPED
                consistent = consistent and bool(np.array_equal(got[~stopped], want[~stopped]))
                if timed and t_set and t2 > t_set[0] and stopped.any():
                    flag_lat[x].append((t2 - t_set[0]) * 1e3)
        med = lambda t: float(np.median(t))
        legs[f"{engine}:{schedule}"] = {
            "engine": {1: "simt-fp32", 2: "wgmma-3xf16"}[s.engine],
            "unstopped_submit_to_wait_ms": med(t_full),
            "stop": {f"X={x:g}ms": {"stop_to_wait_ms": med(lat[x]), "unstopped_left_ms": med(left[x]),
                                   "objects_stopped_median": med(n_stopped[x]),
                                   "flag_to_wait_ms": med(flag_lat[x]) if flag_lat[x] else None,
                                   "flag_samples": len(flag_lat[x])} for x in delays}}
        opt.solver.close()
    print(json.dumps({
        "metric": "time from a stop request to dspgn_keyframe_wait returning", "unit": "ms",
        "steps": args.steps, "warmup": args.warmup, "voxels_dim": args.dim,
        "workload": f"{N_TRACKED} tracked cars ({args.rejected} rejected by the map check) + {N_NEW} new cars, "
                    f"10 joint iterations, meshed at {args.dim}",
        "timing": "host clock, medians; legs alternated per step",
        "card": dict(gpu_card(), **clocks()), "legs": legs, "unstopped_records_identical": consistent,
        "query_plus_sleep_20us_us": sleep_20us(),
    }), flush=True)


if __name__ == "__main__":
    main()
