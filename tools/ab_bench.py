"""A/B timing of this tree against a baseline tree, with an output comparison.

  python tools/ab_bench.py BASE_DIR [--workload cfg2_sdf ...] [--repeats 3] [--steps K] [--warmup W] [--out DIR]

Workload "keyframe" runs tools/keyframe_bench.py (the whole keyframe calls, legs a-d) instead of bench.py; for bench.py
workloads the end-to-end call's time is reported beside the device time per step (under "figures").
BASE_DIR is an unpacked copy of the baseline commit, e.g.  git archive <commit> | tar -x -C ab_base  (ab_base/ is
ignored).  Both trees are built first (their own __graft_entry__.build()).  Then, per workload and repeat, bench.py runs
in the baseline tree and in this tree alternately, each with --dump-outputs, so slow drift of the card (clocks, other
work on the host) lands on both sides.  The result records of every run are compared with the first run of this tree
(np.array_equal; max |delta| when they differ).  The card's name, power limit and maximum SM clock are read with
nvidia-smi in the same call.  Prints one JSON line per workload and a summary line; writes them to DIR/ab.json.
"""
import argparse
import glob
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_bench(tree, workload, steps, warmup, dump):
    if workload == "keyframe":          # tools/keyframe_bench.py: the whole keyframe calls, host clock per call
        cmd = [sys.executable, os.path.join("tools", "keyframe_bench.py"), "--steps", str(10 * steps), "--warmup",
               str(warmup), "--mesh-dims", "", "--dump-outputs", dump]
    else:
        cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
               "--workload", workload, "--dump-outputs", dump]
    p = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(f"bench.py failed in {tree} ({workload}):\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
    return json.loads(lines[-1])


def load_dump(d):
    return {os.path.relpath(f, d)[:-4]: np.load(f) for f in sorted(glob.glob(os.path.join(d, "**", "*.npy"), recursive=True))}


def step_ms(j):
    """The timed figures of one run: bench.py's device time per step and its end-to-end call (Optimizer.reconstruct_batch,
    host clock), or keyframe_bench.py's median per-call time of each leg."""
    if "legs" in j:
        return {k: v["median_ms"] for k, v in j["legs"].items() if isinstance(v, dict) and "median_ms" in v}
    return {"ms_per_step": j["ms_per_step"], "e2e_ms_per_step": (j.get("e2e") or {}).get("ms_per_step")}


def compare(a, b):
    """(all fields array_equal, max |delta| over the float fields, names of the fields that differ)"""
    diff, worst = [], 0.0
    for k in sorted(set(a) | set(b)):
        if k not in a or k not in b or a[k].shape != b[k].shape:
            diff.append(k)
            worst = float("inf")
            continue
        if not np.array_equal(a[k], b[k], equal_nan=True):
            diff.append(k)
            worst = max(worst, float(np.nanmax(np.abs(a[k].astype(np.float64) - b[k].astype(np.float64)))))
    return not diff, worst, diff


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def build(tree):
    subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=tree, check=True,
                   stdout=subprocess.DEVNULL)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("base", help="baseline tree (unpacked git archive of the commit to compare against)")
    ap.add_argument("--workload", nargs="+", default=["cfg2_sdf"])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the dumps and ab.json (default: a temporary directory)")
    args = ap.parse_args()
    base = os.path.abspath(args.base)
    out = os.path.abspath(args.out) if args.out else tempfile.mkdtemp(prefix="ab_bench_")
    os.makedirs(out, exist_ok=True)
    trees = {"base": base, "new": ROOT}
    for t in trees.values():
        build(t)
    gpu = card()
    results = []
    for wl in args.workload:
        runs = {"base": [], "new": []}
        for r in range(args.repeats):
            order = ("base", "new") if r % 2 == 0 else ("new", "base")
            for side in order:
                dump = os.path.join(out, f"{wl}_{side}_{r}")
                runs[side].append((run_bench(trees[side], wl, args.steps, args.warmup, dump), dump))
        ref = load_dump(runs["new"][0][1])
        checks = [compare(ref, load_dump(d)) for side in ("base", "new") for _, d in runs[side]]
        figs = {s: [step_ms(j) for j, _ in runs[s]] for s in runs}
        names = [k for k, v in figs["new"][0].items() if v is not None]
        ms = {k: {s: [f[k] for f in figs[s]] for s in runs} for k in names}
        med = {k: {s: statistics.median(v) for s, v in ms[k].items()} for k in names}
        first = names[0]
        res = {
            "workload": wl, "gpu": gpu,
            "ms_per_step": ms[first], "median_ms": med[first], "speedup": med[first]["base"] / med[first]["new"],
            "spread_ms": {s: max(v) - min(v) for s, v in ms[first].items()},
            "figures": {k: {"median_ms": med[k], "speedup": med[k]["base"] / med[k]["new"],
                            "spread_ms": {s: max(v) - min(v) for s, v in ms[k].items()}, "ms": ms[k]} for k in names},
            "outputs_equal": all(c[0] for c in checks), "max_abs_delta": max(c[1] for c in checks),
            "fields_differing": sorted(set(f for c in checks for f in c[2])),
            "clocks": {s: [j.get("clocks") for j, _ in runs[s]] for s in runs},
            "roofline_achieved": {s: [(j.get("roofline") or {}).get("achieved") for j, _ in runs[s]] for s in runs},
        }
        print(json.dumps(res), flush=True)
        results.append(res)
    with open(os.path.join(out, "ab.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps({"summary": [(r["workload"], round(r["median_ms"]["base"], 3), round(r["median_ms"]["new"], 3),
                                   round(r["speedup"], 3), r["outputs_equal"]) for r in results], "gpu": gpu}))


if __name__ == "__main__":
    main()
