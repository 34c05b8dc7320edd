"""Cost of a 512-wide decoder: DeepSDF's own 8 x 512 network (tests/wide_fixtures.py, written to a temporary directory)
against the 8 x 256 one (decoder_cars.npz), both on the fp32 SIMT engine and on the wide tensor-core engine
(engine="tc_wide"), and the 8 x 256 decoder on the tensor-core engine as context, for

  (a) LocalMapping's reconstruction call: 1 object, 250 points, 250 foreground + 200 background rays, 10 iterations
      (Optimizer.reconstruct_object)
  (b) the gated, meshed stereo keyframe of tools/keyframe_bench.py: 6 tracked cars of which 2 fail the map check, 2 new
      cars, meshes of every object the call creates at voxels_dim --mesh-dim (dspgn_keyframe_batch_meshed)

The legs alternate in one process; each is timed with the host clock around the whole call (it ends in a stream
sync).  Prints one JSON line: per leg and decoder the median / min / p90 in ms, the ratio of the decoder's
multiply-adds per row (forward) to the 8 x 256 decoder's, the card's name and power limit.

--schedules instead times the 8 x 512 decoder on engine="tc_wide" under schedule="launches" (k_wide_wgmma per term and
iteration) against schedule="persistent" (k_wide_persistent, one launch per call), alternated step by step, on (a),
(b) and (c) a cfg2-sized batch: 32 objects x 2048 points, SDF term only, 10 iterations (Optimizer.reconstruct_batch);
the card's SM clock is read in the same call.  --schedules --engine simt times the fp32 SIMT engine the same way
(k_decoder_simt per term and iteration against k_simt_persistent) on the 8 x 256 decoder (cars), the 8 x 512 one (wide)
and the LayerNorm / xyz_in_all / use_tanh variant (decoder_variant.npz).

  python tools/wide_bench.py [--steps K] [--warmup W] [--mesh-dim 32] [--schedules [--engine tc_wide|simt]]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

GOLDEN = os.path.join(ROOT, "tests", "golden")
DECODERS = [("256_simt", "cars", "simt"), ("512_simt", "wide", "simt"), ("256_tc", "cars", "tc"),
            ("256_tc_wide", "cars", "tc_wide"), ("512_tc_wide", "wide", "tc_wide")]


def macs_per_row(path):
    from dsp_slam_b200.decoder import DecoderWeights
    return sum(int(w.shape[0]) * int(w.shape[1]) for w in DecoderWeights.from_npz(path).W)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--mesh-dim", type=int, default=32)
    ap.add_argument("--schedules", action="store_true", help="8 x 512 tc_wide: launches against persistent")
    ap.add_argument("--engine", default="tc_wide", choices=["tc_wide", "simt"],
                    help="--schedules: the engine timed (simt: the cars, wide and variant decoders)")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    from dsp_slam_b200 import synth
    from dsp_slam_b200.optimizer import Optimizer
    from keyframe_bench import N_NEW, N_TRACKED, gpu_card, keyframe_inputs
    if not torch.cuda.is_available():
        raise SystemExit("wide_bench.py needs a CUDA device (no CPU fallback)")
    cfg, objs, modes = keyframe_inputs()
    tracked = objs[:N_TRACKED]
    gates = []
    for i, o in enumerate(tracked):
        M = np.array(o["t_cam_obj"], dtype=np.float32)
        if i < 2:
            M[0, 3] += np.float32(3.0)
        gates.append(dict(t_cam_obj_map=M, t_cam_obj_sim3=o["t_cam_obj_sim3"]))
    gates += [None] * N_NEW
    one = synth.make_object(1, 250, 250, 200)

    legs = {}
    import wide_fixtures
    tmp = tempfile.TemporaryDirectory()
    path = {"cars": os.path.join(GOLDEN, "decoder_cars.npz"), "wide": wide_fixtures.write("wide", tmp.name),
            "variant": os.path.join(GOLDEN, "decoder_variant.npz")}
    if args.schedules:
        batch = [dict(t_cam_obj=o["t_cam_obj_init"], pts=o["pts"]) for o in synth.make_batch(32, 2048, 0, 0)]
        cfg_sdf = json.load(open(os.path.join(ROOT, "dsp_slam_b200", "configs", "config_kitti.json")))
        for dec in (["wide"] if args.engine == "tc_wide" else ["cars", "wide", "variant"]):
            for sch in ("launches", "persistent"):
                tag = sch if args.engine == "tc_wide" else f"{dec}_{sch}"
                opt = Optimizer(path[dec], cfg, engine=args.engine, schedule=sch)
                legs[f"a_localmapping_{tag}"] = lambda opt=opt: opt.reconstruct_object(
                    one["t_cam_obj_init"], one["pts"], one["rays"], one["depth"])
                legs[f"b_keyframe_meshed_{tag}"] = lambda s=opt.solver: s.keyframe(objs, modes, gates, voxels_dim=args.mesh_dim)
                opt_sdf = Optimizer(path[dec], cfg_sdf, engine=args.engine, schedule=sch, sdf_only=True)
                legs[f"c_cfg2_sdf_{tag}"] = lambda opt=opt_sdf: opt.reconstruct_batch(batch)
    for label, dec, engine in ([] if args.schedules else DECODERS):
        opt = Optimizer(path[dec], cfg, engine=engine)
        legs[f"a_localmapping_{label}"] = lambda opt=opt: opt.reconstruct_object(
            one["t_cam_obj_init"], one["pts"], one["rays"], one["depth"])
        legs[f"b_keyframe_meshed_{label}"] = lambda s=opt.solver: s.keyframe(objs, modes, gates, voxels_dim=args.mesh_dim)
    for f in legs.values():
        for _ in range(args.warmup):
            f()
    times = {k: [] for k in legs}
    for _ in range(args.steps):
        for k, f in legs.items():
            t0 = time.perf_counter()
            f()
            times[k].append((time.perf_counter() - t0) * 1e3)
    base = macs_per_row(path["cars"])
    out = {"metric": "wide_schedule_ms" if args.schedules else "wide_decoder_ms", "engine": args.engine if args.schedules else None, "steps": args.steps, "mesh_dim": args.mesh_dim,
           "legs": {k: {"median": float(np.median(v)), "min": float(np.min(v)), "p90": float(np.percentile(v, 90))}
                    for k, v in times.items()},
           "gpu": gpu_card()}
    if args.schedules:
        import subprocess
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        out["gpu"]["sm_clock"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None
    else:
        out["decoder_macs_ratio"] = {label: macs_per_row(path[dec]) / base for label, dec, _ in DECODERS}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
