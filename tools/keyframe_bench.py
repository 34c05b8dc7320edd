"""Per-keyframe latency of DSP-SLAM's stereo keyframe (src/LocalMapping.cc:88-95) through the library, two ways:

  (a) one dspgn_keyframe_batch: tracked objects pose-only + new objects joint, one mode per object
  (b) dspgn_estimate_pose_batch for the tracked objects, then dspgn_reconstruct_batch for the new ones

and, with GetNewObservations' map-consistency check (src/LocalMapping_util.cc:104-147) on the tracked objects, of which
--rejected K fail it (their map pose is 3 m off) and are reconstructed from their Sim(3) detection pose (:179):

  (c) one dspgn_keyframe_batch_gated: the check on the device, the rejected detections' joint runs in the same run
  (d) dspgn_keyframe_batch, the check on the host (oracle/gate_check.py), then dspgn_reconstruct_batch of the rejected

and, for the same gated keyframe, the meshes of every object it creates (CreateNewMapObjects, :179-196), at each
--mesh-dims voxels_dim:

  (e) one dspgn_keyframe_batch_meshed: the mesh decision, the grid decode and the iso-surface after the run, same call
  (f) dspgn_keyframe_batch_gated, the good codes picked on the host, then dspgn_mesh_batch of those codes

The legs alternate in one process; each is timed with the host clock around the whole call (pack + H2D + run + D2H,
ending in a stream sync).  Prints one JSON line with both legs, the card's name and power limit.

  python tools/keyframe_bench.py [--steps K] [--warmup W] [--engine auto|simt|tc] [--rejected K] [--mesh-dims 32,64]
                                 [--dump-outputs DIR]

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
            objs.append(dict(t_cam_obj=T, pts=o["pts"], scale=s, code=code, rays=o["rays"], depth=o["depth"],
                             t_cam_obj_sim3=np.array(o["t_cam_obj_init"], dtype=np.float32)))
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
    ap.add_argument("--rejected", type=int, default=2, help="tracked objects that fail the map check in legs c/d (0..6)")
    ap.add_argument("--mesh-dims", default="32,64", help="voxels_dim of legs e/f, comma separated (empty: none)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import gate_check
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
    # legs a/b: the tracked objects without the detection's rays (the workload of the keyframe call as before)
    plain = [dict(t_cam_obj=o["t_cam_obj"], pts=o["pts"], scale=o["scale"], code=o["code"]) for o in tracked] + new
    opt = Optimizer(os.path.join(ROOT, "tests", "golden", "decoder_cars.npz"), cfg,
                    engine=None if args.engine == "auto" else args.engine)
    s = opt.solver

    def leg_a():
        return s.keyframe(plain, modes)

    def leg_b():
        return s.estimate_pose(plain[:N_TRACKED]), s.reconstruct(new)

    # map poses: the first --rejected tracked objects 3 m off in x (rejected), the others where the detection is (kept)
    maps = []
    for i, o in enumerate(tracked):
        M = np.array(o["t_cam_obj"], dtype=np.float32)
        if i < args.rejected:
            M[0, 3] += np.float32(3.0)
        maps.append(M)
    gates = [dict(t_cam_obj_map=M, t_cam_obj_sim3=o["t_cam_obj_sim3"]) for M, o in zip(maps, tracked)] + [None] * N_NEW

    def leg_c():
        return s.keyframe(objs, modes, gates)

    def leg_d():
        out = s.keyframe(objs, modes)
        rej = []
        for i, o in enumerate(tracked):
            Z = (np.frombuffer(out[i].t_cam_obj, dtype=np.float32).reshape(4, 4) if out[i].status == _lib.ST_OK
                 else o["t_cam_obj"])
            if gate_check.gate(Z, maps[i]) == gate_check.REJECTED:
                rej.append(i)
        joint = s.reconstruct([dict(t_cam_obj=tracked[i]["t_cam_obj_sim3"], pts=tracked[i]["pts"], rays=tracked[i]["rays"],
                                    depth=tracked[i]["depth"]) for i in rej]) if rej else None
        return out, rej, joint

    dims = [int(x) for x in args.mesh_dims.split(",") if x]

    def leg_e(dim):
        return s.keyframe(objs, modes, gates, voxels_dim=dim)

    def leg_f(dim):
        out = s.keyframe(objs, modes, gates)
        good = [i for i in range(len(objs)) if out[i].status == _lib.ST_OK and
                (modes[i] == _lib.MODE_JOINT or out[i].gate == _lib.GATE_REJECTED)]
        codes = np.array([out[i].code[:] for i in good], dtype=np.float32).reshape(len(good), -1)
        return out, good, (s.mesh(codes, dim) if good else [])

    for _ in range(max(args.warmup, 3)):
        leg_a(); leg_b(); leg_c(); leg_d()
        for dim in dims:
            leg_e(dim); leg_f(dim)
    ta, tb, tc, td = [], [], [], []
    te, tf = {d: [] for d in dims}, {d: [] for d in dims}
    out_e, out_f = {}, {}
    for _ in range(args.steps):
        t0 = time.perf_counter(); out_a = leg_a(); t1 = time.perf_counter(); out_b = leg_b(); t2 = time.perf_counter()
        out_c = leg_c(); t3 = time.perf_counter(); out_d = leg_d(); t4 = time.perf_counter()
        ta.append((t1 - t0) * 1e3); tb.append((t2 - t1) * 1e3); tc.append((t3 - t2) * 1e3); td.append((t4 - t3) * 1e3)
        for dim in dims:
            t0 = time.perf_counter(); out_e[dim] = leg_e(dim); t1 = time.perf_counter()
            out_f[dim] = leg_f(dim); t2 = time.perf_counter()
            te[dim].append((t1 - t0) * 1e3); tf[dim].append((t2 - t1) * 1e3)
    leg_c(); launches_c = s.counters()["kernel_launches"]
    leg_a(); launches_a = s.counters()["kernel_launches"]
    s.estimate_pose(plain[:N_TRACKED]); launches_b = s.counters()["kernel_launches"]
    s.reconstruct(new); launches_b += s.counters()["kernel_launches"]

    ma, mb = float(np.median(ta)), float(np.median(tb))
    leg = lambda t, n: {"median_ms": float(np.median(t)), "mean_ms": float(np.mean(t)), "min_ms": float(np.min(t)),
                        "kernel_launches": n}

    def rec(out, n):
        return np.frombuffer(out, dtype=np.float32, count=n * _lib.RESULT_FLOATS).reshape(n, _lib.RESULT_FLOATS).copy()
    ra = rec(out_a, len(objs))
    rb = np.concatenate([rec(out_b[0], N_TRACKED), rec(out_b[1], N_NEW)])
    rc = rec(out_c, len(objs))
    rd = rec(out_d[0], len(objs))
    for k, i in enumerate(out_d[1]):                   # the host path's result, in the gated call's form
        rd[i] = rec(out_d[2], len(out_d[1]))[k]
        rd[i].view(np.int32)[85] = 2
    for i in range(N_TRACKED):
        if i not in out_d[1]:
            rd[i].view(np.int32)[85] = 1
    mesh_legs = {}
    for dim in dims:                                   # e against f: records (but the mesh word) and meshes identical
        (oe, me), (of_, good, mf) = out_e[dim], out_f[dim]
        re_, rf = rec(oe, len(objs)), rec(of_, len(objs))
        re_.view(np.int32)[:, 86] = 0
        done = [i for i in range(len(objs)) if me[i] is not None]
        same = bool(np.array_equal(re_.view(np.uint32), rf.view(np.uint32))) and done == good and all(
            np.array_equal(me[i][0], mf[k][0]) and np.array_equal(me[i][1], mf[k][1]) for k, i in enumerate(good))
        leg_e(dim); le = s.counters()["kernel_launches"]
        mesh_legs[f"dim{dim}"] = {"e_keyframe_batch_meshed": leg(te[dim], le),
                                  "f_keyframe_gated_then_mesh_batch": leg(tf[dim], None),
                                  "f_over_e": float(np.median(tf[dim])) / float(np.median(te[dim])),
                                  "meshes": len(done), "records_and_meshes_identical": same}
    if args.dump_outputs:
        dump_outputs(os.path.join(args.dump_outputs, "a_keyframe_batch"), ra)
        dump_outputs(os.path.join(args.dump_outputs, "b_estimate_pose_then_reconstruct"), rb)
        dump_outputs(os.path.join(args.dump_outputs, "c_keyframe_batch_gated"), rc)
    print(json.dumps({
        "metric": "per-keyframe latency (ms)", "value": ma, "unit": "ms", "higher_is_better": False,
        "steps": args.steps, "warmup": max(args.warmup, 3),
        "workload": f"{N_TRACKED} tracked cars x 250 pts pose-only + {N_NEW} new cars x 250 pts + 450 rays x 50 samples joint",
        "engine": {1: "simt-fp32", 2: "wgmma-3xf16"}[s.engine],
        "timing": "host clock around each whole call (ends in a stream sync), legs alternated, median",
        "card": gpu_card(),
        "legs": {"a_keyframe_batch": leg(ta, launches_a), "b_estimate_pose_then_reconstruct": leg(tb, launches_b),
                 "b_over_a": mb / ma,
                 "c_keyframe_batch_gated": leg(tc, launches_c),
                 "d_keyframe_host_check_then_reconstruct": leg(td, None),
                 "d_over_c": float(np.median(td)) / float(np.median(tc)), "c_over_a": float(np.median(tc)) / ma,
                 **mesh_legs},
        "rejected": f"{len(out_d[1])}/{N_TRACKED} (requested {args.rejected})",
        "records_identical": bool(np.array_equal(ra.view(np.uint32), rb.view(np.uint32))),
        "gated_records_identical": bool(np.array_equal(rc.view(np.uint32), rd.view(np.uint32))),
        "good_objects": f"{int((ra.view(np.int32)[:, 81] == 0).sum())}/{len(objs)}",
    }), flush=True)


if __name__ == "__main__":
    main()
