"""Time a KITTI LiDAR keyframe's detection construction: numpy on the host against the device (DspgnLidarFrame).

Seeded KITTI-sized frames (synth.make_lidar_frame: --points scan points, 20 boxes, 10 masks of 375 x 1242), the
config's num_lidar_max 250, min_mask_area 1000, downsample_ratio 4.  Legs, alternated step by step in one process:

  a  numpy      the numpy geometry of FrameWithLiDAR.get_detections on this host (oracle/lidar_frame.py)
  b  device     LidarFrameBuilder.detections end to end (host clock: staging, H2D, kernels, D2H, unpacking); the
                device time of its stream work (CUDA events around the call: H2D, kernels, D2H; separate pass); and
                the four kernels' time from torch.profiler (separate pass)
  c  busy       leg b issued right after keyframe_batch_async submitted tools/keyframe_bench.py's gated keyframe
                (meshed at 32), which is still running; the keyframe is collected after the timed call.  The solver's
                SM budget is forced to every SM (dspgn_debug_sm_budget): the launches as they are without a frame handle
  d<k>          leg c with the budget forced to k SMs fewer (k = 4, 8, 16): what a live frame handle does with
                DSPGN_FRAME_RESERVE_SMS = k

Legs c and d<k> alternate step by step.  Each reports the frame call's time, the fraction of steps in which the keyframe
was still running when the call returned, and the keyframe's submit->collect time beside the frame call against the
same keyframe alone at the same budget (submitted and collected just before).

Every leg's instances are compared bit for bit with leg a's.  Prints one JSON line with medians and spreads (p10-p90)
in ms, and the card's name, power limit and max SM clock read in the same run.

  python tools/frame_bench.py [--steps K] [--warmup W] [--points N] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def card():
    import torch
    out = {"name": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        pl, clk = q.stdout.strip().splitlines()[0].split(",")
        out.update(power_limit_w=float(pl), max_sm_clock_mhz=float(clk))
    except Exception:                      # noqa: BLE001 -- reported as missing
        out.update(power_limit_w=None, max_sm_clock_mhz=None)
    return out


def same(got, want):
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert np.array_equal(a["surface_points"], b["surface_points"]) and np.array_equal(a["T_cam_obj"], b["T_cam_obj"])
        assert (a["rays"] is None) == (b["rays"] is None)
        if b["rays"] is not None:
            assert np.array_equal(a["rays"], b["rays"]) and np.array_equal(a["depth"], b["depth"])


RESERVES = (4, 8, 16)


def busy_budgets(n_sms):
    """leg -> forced SM budget: c every SM, d<k> k SMs left free"""
    return dict([("c", n_sms)] + [(f"d{k}", n_sms - k) for k in RESERVES])


def busy_step(opt, new, tracked, call, leg, budget, t, keep):
    """One step of a busy leg: the keyframe alone, then again with `call` issued right after its submit.  Returns what
    `call` returned."""
    opt.solver.debug_sm_budget(budget)
    k0 = time.perf_counter()
    opt.keyframe_batch_async(new, tracked, voxels_dim=32).result()
    k1 = time.perf_counter()
    fut = opt.keyframe_batch_async(new, tracked, voxels_dim=32)
    t0 = time.perf_counter(); got = call(); t1 = time.perf_counter()
    pending = not fut.done()
    fut.result()
    k2 = time.perf_counter()
    opt.solver.debug_sm_budget(None)
    if keep:
        t.setdefault(f"{leg}_device_busy_ms", []).append(1e3 * (t1 - t0))
        t.setdefault(f"{leg}_keyframe_busy_ms", []).append(1e3 * (k2 - k1))
        t.setdefault(f"{leg}_keyframe_alone_ms", []).append(1e3 * (k1 - k0))
        t.setdefault(f"{leg}_still_running", []).append(int(pending))
    return got


def busy_report(t):
    """legs' stats, with the still-running flags as fractions"""
    legs = {k: stats(v) for k, v in t.items() if not k.endswith("_still_running")}
    frac = {k[:-len("_still_running")]: float(np.mean(v)) for k, v in t.items() if k.endswith("_still_running")}
    return legs, frac


def stats(v):
    v = np.asarray(v)
    return {"median": float(np.median(v)), "p10": float(np.percentile(v, 10)), "p90": float(np.percentile(v, 90)),
            "n": int(v.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--points", type=int, default=127000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("frame_bench.py needs a CUDA device (no CPU fallback)")
    import __graft_entry__ as g
    g.build()
    from dsp_slam_b200 import synth
    from dsp_slam_b200.lidar_frame import LidarFrameBuilder
    from dsp_slam_b200.optimizer import Optimizer
    from keyframe_bench import N_TRACKED, keyframe_inputs
    from oracle import lidar_frame as O

    cfg = dict(num_lidar_max=250, min_mask_area=1000, downsample_ratio=4.0)
    frames = [synth.make_lidar_frame(100 + i, args.points) for i in range(4)]
    K, Tcv, hw = frames[0]["K"], frames[0]["T_cam_velo"], frames[0]["img_hw"]
    invK = np.linalg.inv(K).astype(np.float32)
    b = LidarFrameBuilder(K, Tcv, cfg, hw)
    kcfg, objs, _ = keyframe_inputs()
    opt = Optimizer(os.path.join(ROOT, "tests", "golden", "decoder_cars.npz"), kcfg)
    tracked, new = objs[:N_TRACKED], objs[N_TRACKED:]

    def host(f):
        return O.detections(f["scan"], f["dets"], f["masks"], f["bboxes"], K, invK, Tcv, 250, 1000, 4.0, *hw)

    def dev(f):
        return b.detections(f["scan"], f["dets"], f["masks"], f["bboxes"])

    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    budgets = list(busy_budgets(n_sms).items())
    t = {"a_numpy_ms": [], "b_device_ms": [], "b_stream_ms": []}
    for step in range(args.warmup + args.steps):
        f = frames[step % len(frames)]
        t0 = time.perf_counter(); want = host(f); t1 = time.perf_counter()
        got = dev(f); t2 = time.perf_counter()
        same(got, want)
        for leg, budget in budgets[step % len(budgets):] + budgets[:step % len(budgets)]:
            same(busy_step(opt, new, tracked, lambda: dev(f), leg, budget, t, step >= args.warmup), want)
        if step >= args.warmup:
            t["a_numpy_ms"].append(1e3 * (t1 - t0))
            t["b_device_ms"].append(1e3 * (t2 - t1))
    # device time of the call's stream work (events around the call on the handle's stream)
    s = torch.cuda.Stream()
    b.set_stream(s.cuda_stream)
    for step in range(args.warmup + args.steps):
        f = frames[step % len(frames)]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        dev(f)
        e1.record(s)
        e1.synchronize()
        if step >= args.warmup:
            t["b_stream_ms"].append(e0.elapsed_time(e1))
    # kernel-only time from the profiler (the four k_frame_* kernels of one call)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for f in frames:
            dev(f)
    kern = [e for e in prof.key_averages() if "k_frame" in e.key]
    legs, frac = busy_report(t)
    res = {"card": card(), "points": args.points, "steps": args.steps, "sms": n_sms, "budgets": dict(budgets),
           "legs": legs, "keyframe_still_running_frac": frac,
           "kernels_us_per_call": {e.key: getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / len(frames) for e in kern},
           "outputs": "bit-identical in every leg"}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
