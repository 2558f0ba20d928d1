"""What laying the pod rows out by namespace buys and costs (include/kt_b200.h "row order of the pod tables").

    python tools/row_order_bench.py [--steps 200] [--reps 20] [--out row_order.json]

  pass       device us per pass, bench.py's method: enough engine contexts rotated to exceed the 50 MB L2 twice, the passes
             launched back to back between ONE pair of CUDA events.  C2 sorted; C2, C3 and C5 in arrival order, laid out
             automatically (by namespace) and forced "as given".
  upload     wall us of kt_upload_pods_packed (both kinds) + kt_sync: C2 sorted, and C2 in arrival order laid out automatically
             and forced "as given".
  step       wall us of one kt_step_submit + kt_step_wait round trip (packed rows of both kinds), the same three ways.
Needs an H100; prints one JSON object (card name, power limit and max SM clock included)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bench  # noqa: E402  (rotation_count, algorithmic_bytes: the headline's own sizing)
import kube_throttler_b200 as kt  # noqa: E402
from kube_throttler_b200 import abi, synth  # noqa: E402

RUN, PEND = abi.PODS_RUNNING, abi.PODS_PENDING


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def engines_for(snap, count, mode, stream):
    out = []
    for _ in range(count):
        e = kt.Engine(snap.R, snap.L, snap.LN)
        e.set_stream(stream)
        for kind in (RUN, PEND):
            e.set_row_order(kind, mode)
        e.upload_snapshot(snap)
        out.append(e)
    return out


def pass_us(snap, mode, steps):
    import torch

    stream = torch.cuda.Stream()  # the engines' stream (the default stream's handle would mean "the engine's own stream")
    probe = engines_for(snap, 1, mode, stream.cuda_stream)
    E = bench.rotation_count(bench.algorithmic_bytes(snap, probe[0].words_per_row)["total"], 1)
    engines = probe + engines_for(snap, E - 1, mode, stream.cuda_stream)
    clustered = [probe[0].row_order(kind)[0] for kind in (RUN, PEND)]
    for i in range(max(3, E)):
        engines[i % E].evaluate(snap.now)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(steps * 60e3) + 2_000_000)  # every launch is queued before the first pass starts
        a.record(stream)
        for i in range(steps):
            engines[i % E].evaluate(snap.now)
        b.record(stream)
    torch.cuda.synchronize()
    for e in engines:
        e.close()
    return {"us_per_pass": a.elapsed_time(b) * 1e3 / steps, "contexts_rotated": E, "clustered_running_pending": clustered}


def wall_us(fn, reps):
    fn()
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return float(np.median(t) * 1e6)


def upload_and_step_us(snap, mode, reps):
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    for kind in (RUN, PEND):
        eng.set_row_order(kind, mode)
    eng.upload_snapshot(snap)
    eng.set_sparse_check(4 * snap.pending.n + 1024)
    packed = [abi.packed_pods(p, code_requests=True) for p in (snap.running, snap.pending)]

    def upload():
        eng.upload_pods_packed(RUN, packed[0])
        eng.upload_pods_packed(PEND, packed[1])
        eng.sync()

    def step():
        eng.step_submit(packed[0], packed[1], snap.now)
        eng.step_wait()

    res = {"upload_us": wall_us(upload, reps), "step_us": wall_us(step, reps), "clustered_running_pending": [eng.row_order(k)[0] for k in (RUN, PEND)]}
    eng.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    torch.cuda.init()
    res = {"card": card(), "steps": args.steps, "reps": args.reps, "pass": [], "upload_and_step": []}
    runs = [("C2", True, abi.ROW_ORDER_AUTO)] + [(cfg, False, mode) for cfg in ("C2", "C3", "C5") for mode in (abi.ROW_ORDER_AUTO, abi.ROW_ORDER_AS_GIVEN)]
    for cfg, sort, mode in runs:
        snap = synth.generate(cfg, sort_by_namespace=sort)
        r = {"config": cfg, "rows": "sorted" if sort else "arrival", "order": {0: "automatic", 1: "as given"}[mode]}
        r.update(pass_us(snap, mode, args.steps))
        res["pass"].append(r)
        print(json.dumps(r), flush=True)
    for sort, mode in ((True, abi.ROW_ORDER_AUTO), (False, abi.ROW_ORDER_AUTO), (False, abi.ROW_ORDER_AS_GIVEN)):
        snap = synth.generate("C2", sort_by_namespace=sort)
        r = {"config": "C2", "rows": "sorted" if sort else "arrival", "order": {0: "automatic", 1: "as given"}[mode]}
        r.update(upload_and_step_us(snap, mode, args.reps))
        res["upload_and_step"].append(r)
        print(json.dumps(r), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
