"""Time a monocular keyframe's detection: numpy + OpenCV on the host against the device (DspgnMonoFrame).

Seeded frames (synth.make_mono_frame) at the Redwood (640 x 480, erosion 5) and Freiburg (960 x 540, erosion 15) sizes,
12 masks, 2000 keypoints, downsample_ratio 4.  Legs, alternated step by step in one process:

  a  host       Frame.get_detections' geometry with numpy and cv2.undistortPoints, then Tracking's cv2.erode of the
                float mask with the ellipse and the (int) read at every keypoint
  b  device     MonoFrameBuilder.detections end to end (host clock: staging, H2D, two kernels, D2H, unpacking); the
                device time of its stream work (CUDA events around the call, separate pass); and the kernels' time from
                torch.profiler (separate pass)
  c, d<k>       leg b issued right after the solver submitted tools/keyframe_bench.py's gated keyframe (meshed at 32),
                at a forced SM budget of every SM (c) or k SMs fewer (d4, d8, d16), as in tools/frame_bench.py: the
                call's time, the fraction of steps in which the keyframe still ran when it returned, and the keyframe's
                submit->collect time against its time alone at the same budget

Every step's rays and feature indices are compared bit for bit with leg a's.  Prints one JSON line with medians and
spreads (p10-p90) in ms, and the card's name, power limit and max SM clock read in the same run.

  python tools/mono_frame_bench.py [--steps K] [--warmup W] [--out FILE]
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

SIZES = {"redwood": 5, "freiburg": 15}


def host_leg(cv2, f, invK, e, alpha=4):
    """(rays, feature indices) with numpy + OpenCV as the Python loader and the Tracking thread compute them."""
    from oracle.lidar_frame import rays_of, sample_background
    masks, H, W = f["masks"], *f["img_hw"]
    m = int(np.argmax(masks.sum(axis=-1).sum(axis=-1)))
    mask_f = masks[m].astype(np.float32) * 255.
    bg = sample_background(f["bboxes"][m], mask_f.astype(bool), alpha, H, W)
    if bg.shape[0] > 200:
        bg = bg[np.linspace(0, bg.shape[0] - 1, 200).astype(np.int32)]
    und = cv2.undistortPoints(bg.reshape(1, -1, 2).astype(np.float32), f["K"], np.array([f["k1"], f["k2"], 0., 0., 0.]),
                              P=f["K"]).squeeze()
    rays = rays_of(und, invK)
    kernel = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (2 * e + 1, 2 * e + 1), (e, e))
    er = cv2.erode(mask_f, kernel)
    kp = f["keypoints"]
    inside = er[kp[:, 1].astype(np.int32), kp[:, 0].astype(np.int32)].astype(np.int32) > 0
    return rays, np.nonzero(inside)[0].astype(np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mono_frame_bench.py needs a CUDA device (no CPU fallback)")
    import cv2
    import __graft_entry__ as g
    g.build()
    from dsp_slam_b200 import synth
    from dsp_slam_b200.mono_frame import MonoFrameBuilder
    from dsp_slam_b200.optimizer import Optimizer
    from frame_bench import busy_budgets, busy_report, busy_step, card
    from keyframe_bench import N_TRACKED, keyframe_inputs
    kcfg, objs, _ = keyframe_inputs()
    opt = Optimizer(os.path.join(ROOT, "tests", "golden", "decoder_cars.npz"), kcfg)
    tracked, new = objs[:N_TRACKED], objs[N_TRACKED:]
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    budgets = list(busy_budgets(n_sms).items())
    res = {"card": card(), "steps": args.steps, "cv2": cv2.__version__, "cv2_threads": cv2.getNumThreads(), "sizes": {}}
    for cam, e in SIZES.items():
        frames = [synth.make_mono_frame(200 + i, cam, 12, 2000) for i in range(4)]
        K = frames[0]["K"]
        invK = np.linalg.inv(K)
        b = MonoFrameBuilder(K, frames[0]["k1"], frames[0]["k2"], dict(downsample_ratio=4.0), frames[0]["img_hw"], e)

        def dev(f):
            rays = b.detections(f["masks"], f["bboxes"], f["keypoints"])[0].background_rays
            return rays, b.feature_points()

        t = {"a_host_ms": [], "b_device_ms": [], "b_stream_ms": []}
        for step in range(args.warmup + args.steps):
            f = frames[step % len(frames)]
            t0 = time.perf_counter(); want = host_leg(cv2, f, invK, e); t1 = time.perf_counter()
            got = dev(f); t2 = time.perf_counter()
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
            for leg, budget in budgets[step % len(budgets):] + budgets[:step % len(budgets)]:
                busy = busy_step(opt, new, tracked, lambda: dev(f), leg, budget, t, step >= args.warmup)
                assert np.array_equal(busy[0], want[0]) and np.array_equal(busy[1], want[1])
            if step >= args.warmup:
                t["a_host_ms"].append(1e3 * (t1 - t0))
                t["b_device_ms"].append(1e3 * (t2 - t1))
        s = torch.cuda.Stream()
        b.set_stream(s.cuda_stream)
        for step in range(args.warmup + args.steps):
            f = frames[step % len(frames)]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            got = dev(f)
            e1.record(s)
            e1.synchronize()
            if step >= args.warmup:
                t["b_stream_ms"].append(e0.elapsed_time(e1))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for f in frames:
                dev(f)
        kern = [ev for ev in prof.key_averages() if "k_mono" in ev.key or "k_frame" in ev.key]
        H, W = frames[0]["img_hw"]
        legs, frac = busy_report(t)
        res["sizes"][cam] = {"img_hw": [H, W], "erosion": e, "masks": 12, "keypoints": 2000, "sms": n_sms,
                             "budgets": dict(budgets), "legs": legs, "keyframe_still_running_frac": frac,
                             "kernels_us_per_call": {ev.key: getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0)) / len(frames)
                                                     for ev in kern},
                             "outputs": "bit-identical in every step"}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
