"""Cost of kt_get_match_columns (affectedPods from the throttles' side) against downloading the bitmap and transposing it on
the host.  For each shape and kind: one throttle, and all M.  Device time from CUDA events around the call (the call
synchronises its stream, so the end event follows its copies); wall time for the whole call.

    python tools/match_columns_bench.py [--configs C2,C5] [--reps 20] [--out match_columns.json]

Needs an H100; prints one JSON object (card name and power limit included)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import kube_throttler_b200 as kt  # noqa: E402
from kube_throttler_b200 import abi, synth  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def host_transpose(bitmap, idx, codes=None):
    """The same lists from the downloaded bitmap, word by word (only the words of the listed throttles are unpacked)."""
    idx = np.asarray(idx, np.int64)
    lists = {}
    shifts = np.arange(32, dtype=np.uint32)
    for w in np.unique(idx >> 5):
        col = bitmap[:, w]
        nzr = np.flatnonzero(col)
        bits = (col[nzr][:, None] >> shifts) & 1
        for b in range(32):
            lists[int(w) * 32 + b] = nzr[bits[:, b] != 0]
    rows = [lists[int(t)] for t in idx]
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])])
    if codes is not None:
        [((codes[r, t >> 4] >> np.uint32(2 * (t & 15))) & 3).astype(np.uint8) for r, t in zip(rows, idx)]
    return off


def timed(fn, reps):
    import torch

    fn()  # warm-up: scratch buffers grow once
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev, wall = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        start.record()
        fn()
        end.record()
        end.synchronize()
        wall.append(time.perf_counter() - t0)
        dev.append(start.elapsed_time(end) / 1e3)
    return {"device_ms_median": float(np.median(dev) * 1e3), "wall_ms_median": float(np.median(wall) * 1e3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,C5")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    torch.cuda.init()
    res = {"card": card(), "reps": args.reps, "results": []}
    for cfg in args.configs.split(","):
        snap = synth.generate(cfg)
        eng = kt.Engine(snap.R, snap.L, snap.LN)
        eng.set_stream(torch.cuda.current_stream().cuda_stream)
        eng.upload_snapshot(snap)
        eng.evaluate(snap.now)
        W = eng.words_per_row
        for kind, name in ((abi.PODS_RUNNING, "running"), (abi.PODS_PENDING, "pending")):
            n = eng.n[kind]
            # a throttle with many affected pods, so that one-throttle numbers are not of an empty column
            off_all, _, _ = eng.match_columns(kind, np.arange(snap.m))
            busiest = int(np.argmax(np.diff(off_all)))
            bitmap = np.zeros((n, W), np.uint32)
            codes = np.zeros((snap.pending.n, 2 * W), np.uint32) if kind == abi.PODS_PENDING else None
            for label, idx in (("one", np.array([busiest])), ("all", np.arange(snap.m))):
                cap = int(eng.match_columns(kind, idx)[0][-1])
                cols = timed(lambda: eng.match_columns(kind, idx, cap=cap), args.reps)

                def download_and_transpose():
                    eng._ck(eng._L.kt_get_match_bitmap(eng._h, kind, abi.ptr(bitmap)))
                    if codes is not None:
                        eng.get_check(codes, None)
                    host_transpose(bitmap, idx, codes)

                base = timed(download_and_transpose, max(3, args.reps // 4))
                res["results"].append({"config": cfg, "kind": name, "throttles": label, "k": int(len(idx)), "entries": cap,
                                       "match_columns": cols, "bitmap_plus_host_transpose": base})
                print(json.dumps(res["results"][-1]), flush=True)
        eng.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
