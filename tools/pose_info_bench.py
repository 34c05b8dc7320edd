"""Time dspgn_pose_information after a reconstruction call of n objects (cfg2_sdf-shaped synthetic objects).

  python tools/pose_info_bench.py [--n 1 32] [--repeats 50]

The solver runs on the legacy default stream, so CUDA events recorded there before and after the call bracket its copies
and its kernel (device time); the host time of the whole call, which ends in a stream synchronisation, is printed beside
it.  The card's name, power limit and maximum SM clock are read with nvidia-smi in the same call.  Prints one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 32])
    ap.add_argument("--repeats", type=int, default=50)
    args = ap.parse_args()
    import torch
    from dsp_slam_b200 import synth
    from dsp_slam_b200.optimizer import Optimizer
    cfg = json.load(open(os.path.join(ROOT, "dsp_slam_b200", "configs", "config_kitti.json")))
    opt = Optimizer(os.path.join(ROOT, "tests", "golden", "decoder_cars.npz"), cfg, sdf_only=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    out = {"gpu": q.stdout.strip(), "pose_information": {}}
    for n in args.n:
        objs = synth.make_batch(n, 2048, 0, 0)
        opt.reconstruct_batch([dict(t_cam_obj=o["t_cam_obj_init"], pts=o["pts"]) for o in objs])
        for _ in range(5):
            opt.pose_information()
        dev, host = [], []
        for _ in range(args.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            t0 = time.perf_counter()
            opt.pose_information()
            t1 = time.perf_counter()
            e1.record()
            e1.synchronize()
            dev.append(e0.elapsed_time(e1))
            host.append(1e3 * (t1 - t0))
        out["pose_information"][n] = {"device_ms_median": statistics.median(dev), "host_ms_median": statistics.median(host)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
