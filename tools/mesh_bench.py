"""Mesh extraction of K object codes, two legs alternated in one process on cuda:0:

  host    per object: MeshExtractor.sdf_grid(code) (GPU decode, 1 MB grid back to the host) + the numpy marching
          tetrahedra of dsp_slam_b200.mesh -- what extract_mesh_from_code ran without scikit-image before the device
          path existed
  device  one MeshExtractor.extract_meshes(codes) call (dspgn_mesh_batch): grids and iso-surfaces on the GPU

Prints one JSON line per (dim, K): median / min / max wall time of each leg, the device leg's split between the decode
kernels and the rest of the call -- query points, iso-surface passes, scans, read-backs (CUDA events of the library,
enable_timing) -- whether both legs return the same bytes, and the card's
name, power limit and max SM clock read in the same run.

  python tools/mesh_bench.py [--dims 32 64] [--ks 1 8] [--reps 7] [--engine auto|simt|tc]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, pl, clk = [s.strip() for s in q.split(",")]
        return dict(gpu=name, power_limit=pl, max_sm_clock=clk)
    except Exception as e:            # noqa: BLE001
        return dict(gpu=f"unknown ({e!r})")


def host_leg(mx, codes):
    from dsp_slam_b200.mesh import marching_tetrahedra
    h = 2.0 / (mx.voxels_dim - 1)
    out = []
    for c in codes:
        v, f = marching_tetrahedra(mx.sdf_grid(c), 0.0, [h] * 3)
        out.append(((v + np.array([-1.0, -1.0, -1.0])).astype(np.float32), f.astype(np.int32)))
    return out


def device_leg(mx, codes):
    return [(m.vertices, m.faces) for m in mx.extract_meshes(codes)]


def stats(ts):
    ts = sorted(ts)
    return dict(median_ms=round(1e3 * ts[len(ts) // 2], 3), min_ms=round(1e3 * ts[0], 3), max_ms=round(1e3 * ts[-1], 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--engine", default="auto")
    a = ap.parse_args()
    from dsp_slam_b200.optimizer import MeshExtractor
    G = os.path.join(ROOT, "tests", "golden")
    base = np.load(os.path.join(G, "recon_kitti250.npz"))["code"].astype(np.float32)
    rng = np.random.default_rng(0)
    info = card()
    for dim in a.dims:
        mx = MeshExtractor(os.path.join(G, "decoder_cars.npz"), 64, dim, engine=a.engine)
        for K in a.ks:
            codes = (base[None] + 0.05 * rng.standard_normal((K, 64))).astype(np.float32)
            legs = {"host": host_leg, "device": device_leg}
            res = {k: f(mx, codes) for k, f in legs.items()}          # warm-up of every shape
            same = all(hv.tobytes() == dv.tobytes() and np.array_equal(hf, df)
                       for (hv, hf), (dv, df) in zip(res["host"], res["device"]))
            ts = {k: [] for k in legs}
            dec, tot = [], []
            for _ in range(a.reps):
                for k, f in legs.items():
                    mx.solver.enable_timing(k == "device")
                    t0 = time.perf_counter()
                    f(mx, codes)
                    ts[k].append(time.perf_counter() - t0)
                    if k == "device":
                        c = mx.solver.counters()
                        dec.append(c["decoder_ms"]); tot.append(c["total_ms"])
            mx.solver.enable_timing(False)
            rec = dict(dim=dim, K=K, engine=mx.solver.engine, reps=a.reps, host=stats(ts["host"]),
                       device=stats(ts["device"]), device_decode_ms=round(float(np.median(dec)), 3),
                       device_rest_ms=round(float(np.median(np.subtract(tot, dec))), 3),
                       vertices=int(sum(v.shape[0] for v, _ in res["device"])),
                       faces=int(sum(f.shape[0] for _, f in res["device"])), bit_identical=bool(same), **info)
            rec["speedup_median"] = round(rec["host"]["median_ms"] / rec["device"]["median_ms"], 2)
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
