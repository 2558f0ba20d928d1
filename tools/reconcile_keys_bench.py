"""Cost of reconcile(key) on the device (kt_reconcile_throttles) against what a caller had before it: a FRESH_STATUS |
SKIP_CHECK pass over the whole snapshot plus kt_get_reconcile_rows of the same columns.  For C2 and C5: 1, 10 and 100
namespaced Throttles (picked at random) and the ClusterThrottle that matches the most rows.  The two sides run alternately, rep
by rep; device time from CUDA events around the calls (both synchronise their stream before they return), wall time for the
whole call.  Then, on a plugin loaded with a C2-shaped world (tools/plugin_bench.py), kth_reconcile of 1 / 10 / 100 keys against
kth_reconcile_all, alternately too.

    python tools/reconcile_keys_bench.py [--configs C2,C5] [--reps 20] [--no-plugin] [--out reconcile_keys.json]

Needs an H100; prints one JSON object (card name, power limit and max SM clock included)."""
from __future__ import annotations

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

import kube_throttler_b200 as kt  # noqa: E402
from kube_throttler_b200 import abi, synth  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def alternate(fns, reps):
    """Median device and wall ms of each callable, run alternately rep by rep after one warm-up each."""
    import torch

    for f in fns.values():
        f()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev = {k: [] for k in fns}
    wall = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            start.record()
            f()
            end.record()
            end.synchronize()
            wall[k].append(time.perf_counter() - t0)
            dev[k].append(start.elapsed_time(end))
    return {k: {"device_ms_median": round(float(np.median(dev[k])), 4), "wall_ms_median": round(float(np.median(wall[k]) * 1e3), 4)} for k in fns}


def engine_side(cfg, reps):
    import torch

    snap = synth.generate(cfg)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    eng.upload_snapshot(snap)
    eng.evaluate(snap.now, abi.EVAL_FRESH_STATUS | abi.EVAL_SKIP_CHECK)
    _, off_all, _ = eng.reconcile_throttles(snap.now, np.arange(snap.m))
    counts = np.diff(off_all)
    rng = np.random.default_rng(0)
    kinds = np.asarray(snap.kind)
    named = np.flatnonzero(kinds == abi.KIND_THROTTLE)
    cluster = np.flatnonzero(kinds == abi.KIND_CLUSTERTHROTTLE)
    sets = [(f"{k}_throttles", rng.choice(named, size=k, replace=False)) for k in (1, 10, 100) if len(named) >= k]
    if len(cluster):
        sets.append(("busiest_clusterthrottle", np.array([cluster[np.argmax(counts[cluster])]])))
    out = []
    for label, idx in sets:
        idx = np.ascontiguousarray(idx, np.int32)
        cap = int(eng.reconcile_throttles(snap.now, idx)[1][-1])

        def full_pass():
            eng.evaluate(snap.now, abi.EVAL_FRESH_STATUS | abi.EVAL_SKIP_CHECK)
            eng.get_reconcile_rows(idx)

        t = alternate({"reconcile_throttles": lambda: eng.reconcile_throttles(snap.now, idx, cap=cap), "pass_plus_reconcile_rows": full_pass}, reps)
        row = {"config": cfg, "n": int(snap.running.n), "m": int(snap.m), "keys": label, "k": int(len(idx)), "matched_rows": cap, **t}
        print(json.dumps(row), flush=True)
        out.append(row)
    eng.close()
    return out


def plugin_side(reps):
    from plugin_bench import NOW, c2_world

    w, running, _ = c2_world(0)
    for m in running:
        w._L.kth_apply(w._h, m)
    w.reconcile_all(NOW)
    rng = np.random.default_rng(1)
    names = [f"ns{i % 50}/t{i}" for i in range(1000)]
    out = []
    for k in (1, 10, 100):
        keys = list(rng.choice(names, size=k, replace=False))

        def timed(f):
            ts = []
            for _ in range(reps):
                t0 = time.perf_counter()
                f()
                ts.append(time.perf_counter() - t0)
            return ts

        w.reconcile(keys, NOW)
        w.reconcile_all(NOW)
        a, b = [], []
        for _ in range(reps):  # alternately
            a += timed(lambda: w.reconcile(keys, NOW))[:1]
            b += timed(lambda: w.reconcile_all(NOW))[:1]
        row = {"plugin": "C2 world (50 namespaces, 1000 Throttles, 100k running pods)", "keys": k,
               "kth_reconcile_ms_median": round(float(np.median(a)) * 1e3, 4), "kth_reconcile_all_ms_median": round(float(np.median(b)) * 1e3, 4)}
        print(json.dumps(row), flush=True)
        out.append(row)
    w.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,C5")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--no-plugin", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    torch.cuda.init()
    res = {"card": card(), "reps": args.reps, "engine": [], "plugin": []}
    for cfg in args.configs.split(","):
        res["engine"] += engine_side(cfg, args.reps)
    if not args.no_plugin:
        res["plugin"] = plugin_side(args.reps)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
