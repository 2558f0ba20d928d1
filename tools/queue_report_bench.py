"""Cost of summarising the scheduling queue per throttle (kth_queue_report) against the only way to get the same numbers before
it: kth_affected_pods for every throttle (which has no onlyBlocker).

Plugin side: tools/plugin_bench.py's C2 world (50 namespaces, 1000 Throttles, 100k running pods, 10k queued pods).  Wall time of
  - report_current   a report right after a report: the cached verdicts and the device's codes are current (one device call);
  - report_stale     a report after a Reserve / Unreserve of a queued pod voided cached verdicts (one pass, then the call);
  - affected_pods_all  kth_affected_pods for each of the 1000 throttles, after the same Reserve / Unreserve.
Engine side: kt_get_check_summary over the whole pending table of BASELINE C2 and C5 after a whole pass, device time (CUDA
events around the call on the engine's stream) and wall time.

    python tools/queue_report_bench.py [--reps 20] [--out queue_report.json]

Needs an H100; prints one JSON object (card name, power limit and max SM clock included)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import kube_throttler_b200 as kt  # noqa: E402
from kube_throttler_b200 import synth  # noqa: E402
from reconcile_keys_bench import card  # noqa: E402


def wall_ms(fn, reps, before=None):
    """Median wall ms of fn() (every call ends in a device synchronisation), `before()` run untimed ahead of each rep."""
    fn()
    out = []
    for _ in range(reps):
        if before:
            before()
        t0 = time.perf_counter()
        fn()
        out.append(time.perf_counter() - t0)
    return round(float(np.median(out)) * 1e3, 4)


def plugin_side(reps):
    from plugin_bench import NOW, c2_world

    w, running, pending = c2_world(0)
    L, h = w._L, w._h
    for m in running:
        L.kth_apply(h, m)
    for m in pending:
        L.kth_apply(h, json.dumps(m).encode())
    w.reconcile_all(NOW)
    report = w.queue_report()
    keys = [(m["metadata"]["namespace"], m["metadata"]["name"]) for m in pending[:64]]
    flip = {"i": 0}

    def void_verdicts():  # Reserve, or Unreserve, one queued pod: the cached verdicts of the pods sharing its throttles are void
        k = keys[flip["i"] % len(keys)]
        (w.reserve_key if (flip["i"] // len(keys)) % 2 == 0 else w.unreserve_key)(*k)
        flip["i"] += 1

    names = [tuple(e["key"].split("/", 1)[::-1]) for e in report["throttles"]]

    def affected_all():
        for name, ns in names:
            w.affected_pods(name, ns)

    row = {"throttles": len(report["throttles"]), "queued": report["queued"], "running": len(running),
           "held_back_throttles": sum(1 for e in report["throttles"] if e["heldBack"]),
           "report_current_ms": wall_ms(w.queue_report, reps),
           "report_stale_ms": wall_ms(w.queue_report, reps, void_verdicts),
           "affected_pods_all_ms": wall_ms(affected_all, max(2, reps // 10), void_verdicts)}
    stats = w.queue_stats()
    row["queue_passes"], row["queue_hits"] = stats["passes"], stats["hits"]
    print(json.dumps(row), flush=True)
    w.close()
    return row


def engine_side(config, reps):
    import torch

    snap = synth.generate(config)
    stream = torch.cuda.Stream()
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.set_stream(stream.cuda_stream)
    eng.upload_snapshot(snap)
    eng.evaluate(snap.now)
    codes = np.zeros((snap.pending.n, 2 * eng.words_per_row), np.uint32)
    admit = np.zeros(snap.pending.n, np.uint8)
    eng.get_check(codes, admit)
    fns = {"check_summary": lambda: eng.check_summary(0, snap.pending.n)}
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev, wall = {k: [] for k in fns}, {k: [] for k in fns}
    for f in fns.values():
        f()
    for _ in range(reps):
        for k, f in fns.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            start.record(stream)
            f()
            end.record(stream)
            end.synchronize()
            wall[k].append(time.perf_counter() - t0)
            dev[k].append(start.elapsed_time(end))
    row = {"config": config, "m": int(snap.m), "pending": int(snap.pending.n), "words_per_row": int(eng.words_per_row),
           "rejected_rows": int((admit == 0).sum())}
    for k in fns:
        row[k] = {"device_ms_median": round(float(np.median(dev[k])), 4), "wall_ms_median": round(float(np.median(wall[k]) * 1e3), 4)}
    print(json.dumps(row), flush=True)
    eng.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--configs", default="C2,C5")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    torch.cuda.init()
    res = {"card": card(), "engine": [engine_side(c, args.reps) for c in args.configs.split(",")], "plugin": plugin_side(args.reps)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
