"""Cost of applying informer events in batches (kth_apply_events) against event by event (kth_apply / kth_delete).

Worlds: tools/plugin_bench.py's C2 world (50 namespaces, 1000 Throttles) with 10k or 100k running pods and 10k or 100k queued
pods.  The stream: 1000 deletes of bound pods and 1000 relabels of counted (bound) pods, interleaved.  Event by event, each such
event runs a pass over the whole pending table; in a batch, the pod events between two table events take one kt_match_pods
call.  Three ways to apply the stream run on disjoint pods of the same world: one call per event, one kth_apply_events call for
the whole stream, and kth_apply_events in batches of 64.  Wall time per event, with a device synchronisation inside the timed
region.  Then kt_match_pods' own device time (CUDA events) for k = 1 ... 10^4 pods on BASELINE C2's tables.

    python tools/apply_events_bench.py [--worlds 10000:10000,100000:10000,100000:100000] [--events 1000] [--out apply_events.json]

Needs an H100; prints one JSON object (card name, power limit and max SM clock included)."""
from __future__ import annotations

import argparse
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import kube_throttler_b200 as kt  # noqa: E402
from kube_throttler_b200 import synth  # noqa: E402
from reconcile_keys_bench import alternate, card  # noqa: E402


def stream(running, lo, n, rng):
    """n deletes of bound pods and n relabels of counted pods, interleaved, on running[lo : lo + 2n]."""
    dels = [json.loads(m) for m in running[lo:lo + n]]
    rel = [json.loads(m) for m in running[lo + n:lo + 2 * n]]
    out = []
    for d, r in zip(dels, rel):
        r["metadata"]["labels"] = {"app": f"a{rng.randrange(64)}", "tier": f"x{rng.randrange(8)}", "rel": f"r{rng.randrange(16)}"}
        out.append({"type": "DELETED", "object": d})
        out.append({"type": "MODIFIED", "object": r})
    return out


def world_side(n_run, n_pend, n_events):
    import torch
    from plugin_bench import NOW, c2_world

    w, running, pending = c2_world(0, n_run=n_run, n_pend=n_pend)
    L, h = w._L, w._h
    for m in running:
        L.kth_apply(h, m)
    for m in pending:
        L.kth_apply(h, json.dumps(m).encode())
    w.reconcile_all(NOW)
    rng = random.Random(1)
    row = {"running": n_run, "queued": n_pend, "events": 2 * n_events}

    def one_by_one(evs):
        for e in evs:
            o = e["object"]
            if e["type"] == "DELETED":
                L.kth_delete(h, b"Pod", o["metadata"]["namespace"].encode(), o["metadata"]["name"].encode())
            else:
                L.kth_apply(h, json.dumps(o).encode())

    def batched(size):
        def go(evs):
            for i in range(0, len(evs), size):
                L.kth_apply_events(h, json.dumps(evs[i:i + size]).encode())
        return go

    modes = [("event_by_event", one_by_one), ("one_batch", batched(1 << 30)), ("batches_of_64", batched(64))]
    for i, (name, fn) in enumerate(modes):
        evs = stream(running, 2 * n_events * i, n_events, rng)
        fn(evs[:8])  # warm-up on the first events
        evs = evs[8:]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(evs)
        torch.cuda.synchronize()
        row[name + "_us_per_event"] = round((time.perf_counter() - t0) / len(evs) * 1e6, 2)
    print(json.dumps(row), flush=True)
    w.close()
    return row


def kernel_side(reps):
    import torch

    snap = synth.generate("C2")
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    eng.upload_snapshot(snap)
    rng = np.random.default_rng(0)
    out = []
    for k in (1, 16, 256, 4096, 10_000):
        rows = rng.integers(0, snap.pending.n, size=k)
        labels, ns = np.ascontiguousarray(snap.pending.labels[:, rows]), np.ascontiguousarray(snap.pending.ns_id[rows])
        t = alternate({"match_pods": lambda: eng.match_pods(labels, ns)}, reps)["match_pods"]
        row = {"config": "C2", "m": int(snap.m), "words_per_row": int(eng.words_per_row), "k": k, **t}
        print(json.dumps(row), flush=True)
        out.append(row)
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="10000:10000,100000:10000,100000:100000")
    ap.add_argument("--events", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    torch.cuda.init()
    res = {"card": card(), "kernel": kernel_side(args.reps), "plugin": []}
    for wspec in args.worlds.split(","):
        n_run, n_pend = (int(x) for x in wspec.split(":"))
        res["plugin"].append(world_side(n_run, n_pend, args.events))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
