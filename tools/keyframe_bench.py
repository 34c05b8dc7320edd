"""Per-keyframe latency of DSP-SLAM's stereo keyframe (src/LocalMapping.cc:88-95) through the library, two ways:

  (a) one dspgn_keyframe_batch: tracked objects pose-only + new objects joint, one mode per object
  (b) dspgn_estimate_pose_batch for the tracked objects, then dspgn_reconstruct_batch for the new ones

The two legs alternate in one process; each is timed with the host clock around the whole call (pack + H2D + run + D2H,
ending in a stream sync).  Prints one JSON line with both legs, the card's name and power limit.

  python tools/keyframe_bench.py [--steps K] [--warmup W] [--engine auto|simt|tc] [--dump-outputs DIR]   (on an H100)

The keyframe has the shape of `bench.py --workload slam1`: 6 tracked cars (250 points, pose-only, pose_only_iterations)
and 2 new cars (250 points + 250 foreground and 200 background rays, 10 joint iterations), seeded.  --dump-outputs
writes the result records of both legs (DIR/a_keyframe_batch, DIR/b_estimate_pose_then_reconstruct).
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

N_TRACKED, N_NEW = 6, 2


def keyframe_inputs():
    """Tracked detections (SE(3) pose, scale, shape code) first, then the new detections (pose, points, rays, depths)."""
    from dsp_slam_b200 import synth, load_config
    cfg = load_config("config_kitti.json")
    cfg["optimizer"]["joint_optim"]["num_iterations"] = 10
    objs = []
    for i, o in enumerate(synth.make_batch(N_TRACKED + N_NEW, 250, 250, 200, cls="cars", seed0=0)):
        if i < N_TRACKED:
            T = np.array(o["t_cam_obj_init"], dtype=np.float32)
            s = float(np.cbrt(np.linalg.det(T[:3, :3].astype(np.float64))))
            T[:3, :3] /= np.float32(s)
            code = (0.1 * np.random.default_rng(500 + i).standard_normal(64)).astype(np.float32)
            objs.append(dict(t_cam_obj=T, pts=o["pts"], scale=s, code=code))
        else:
            objs.append(dict(t_cam_obj=o["t_cam_obj_init"], pts=o["pts"], rays=o["rays"], depth=o["depth"]))
    modes = [1] * N_TRACKED + [0] * N_NEW
    return cfg, objs, modes


def gpu_card():
    """Name and power limit of the card the numbers were measured on."""
    import torch
    name, limit = torch.cuda.get_device_name(), None
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        limit = float(q.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return {"name": name, "power_limit_w": limit}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--engine", default="auto", choices=["auto", "simt", "tc"])
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    from bench import dump_outputs
    from dsp_slam_b200 import _lib
    from dsp_slam_b200.optimizer import Optimizer
    if not torch.cuda.is_available():
        raise SystemExit("keyframe_bench.py needs a CUDA device (no CPU fallback)")
    cfg, objs, modes = keyframe_inputs()
    tracked, new = objs[:N_TRACKED], objs[N_TRACKED:]
    opt = Optimizer(os.path.join(ROOT, "tests", "golden", "decoder_cars.npz"), cfg,
                    engine=None if args.engine == "auto" else args.engine)
    s = opt.solver

    def leg_a():
        return s.keyframe(objs, modes)

    def leg_b():
        return s.estimate_pose(tracked), s.reconstruct(new)

    for _ in range(max(args.warmup, 3)):
        leg_a(); leg_b()
    ta, tb = [], []
    for _ in range(args.steps):
        t0 = time.perf_counter(); out_a = leg_a(); t1 = time.perf_counter(); out_b = leg_b(); t2 = time.perf_counter()
        ta.append((t1 - t0) * 1e3); tb.append((t2 - t1) * 1e3)
    leg_a(); launches_a = s.counters()["kernel_launches"]
    s.estimate_pose(tracked); launches_b = s.counters()["kernel_launches"]
    s.reconstruct(new); launches_b += s.counters()["kernel_launches"]

    def rec(out, n):
        return np.frombuffer(out, dtype=np.float32, count=n * _lib.RESULT_FLOATS).reshape(n, _lib.RESULT_FLOATS).copy()
    ra = rec(out_a, len(objs))
    rb = np.concatenate([rec(out_b[0], N_TRACKED), rec(out_b[1], N_NEW)])
    if args.dump_outputs:
        dump_outputs(os.path.join(args.dump_outputs, "a_keyframe_batch"), ra)
        dump_outputs(os.path.join(args.dump_outputs, "b_estimate_pose_then_reconstruct"), rb)
    ma, mb = float(np.median(ta)), float(np.median(tb))
    leg = lambda t, n: {"median_ms": float(np.median(t)), "mean_ms": float(np.mean(t)), "min_ms": float(np.min(t)),
                        "kernel_launches": n}
    print(json.dumps({
        "metric": "per-keyframe latency (ms)", "value": ma, "unit": "ms", "higher_is_better": False,
        "steps": args.steps, "warmup": max(args.warmup, 3),
        "workload": f"{N_TRACKED} tracked cars x 250 pts pose-only + {N_NEW} new cars x 250 pts + 450 rays x 50 samples joint",
        "engine": {1: "simt-fp32", 2: "wgmma-3xf16"}[s.engine],
        "timing": "host clock around each whole call (ends in a stream sync), legs alternated, median",
        "card": gpu_card(),
        "legs": {"a_keyframe_batch": leg(ta, launches_a), "b_estimate_pose_then_reconstruct": leg(tb, launches_b),
                 "b_over_a": mb / ma},
        "records_identical": bool(np.array_equal(ra.view(np.uint32), rb.view(np.uint32))),
        "good_objects": f"{int((ra.view(np.int32)[:, 81] == 0).sum())}/{len(objs)}",
    }), flush=True)


if __name__ == "__main__":
    main()
