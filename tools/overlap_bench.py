"""Fused passes queued back to back against passes one at a time, and the in-kernel trace of two consecutive passes.

A fused pass queued right behind another one runs its first phase (match, pre-record and reconcile tiles) while the pass
ahead of it still decides.  This measures, on one GPU at the given shape (default C2):
  - `queued`:   K passes of ONE context queued back to back behind a spin kernel, CUDA events around the K (bench.py rotates
                over several contexts; this shows the gain does not depend on that);
  - `isolated`: K single passes, each between CUDA events and followed by a device synchronise (the latency of one pass);
  - `trace`:    two contexts on one stream, pass A then pass B queued back to back with the in-kernel trace on: when B's first
                tile starts and B's last CTA exits, against when A's first tile starts and A's CTAs exit (µs since A's start).
Prints one JSON line with the card's name and power limit.
python tools/overlap_bench.py [--config C2] [--steps 50]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import kube_throttler_b200 as kt
from kube_throttler_b200 import synth


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0)


def engine(snap, stream):
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.set_stream(stream.cuda_stream)
    eng.upload_snapshot(snap)
    return eng


def queued_us(eng, stream, now, steps):
    with torch.cuda.stream(stream):
        for _ in range(5):
            eng.evaluate(now)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(steps * 60e3) + 2_000_000)  # every launch is queued before the first one runs
        a.record(stream)
        for _ in range(steps):
            eng.evaluate(now)
        b.record(stream)
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / steps


def isolated_us(eng, stream, now, steps):
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            a.record(stream)
            eng.evaluate(now)
            b.record(stream)
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e3)
    return float(np.median(times)), float(np.min(times)), float(np.max(times))


def trace_pair(a, b, stream, now):
    for e in (a, b):
        e.enable_trace(True)
    with torch.cuda.stream(stream):
        a.evaluate(now)
        b.evaluate(now)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(2_000_000)
        a.evaluate(now)
        b.evaluate(now)
    torch.cuda.synchronize()
    (ra, _), (rb, _) = a.trace(), b.trace()
    for e in (a, b):
        e.enable_trace(False)
    ra, rb = ra.astype(np.float64), rb.astype(np.float64)
    t0 = ra[:, 2][ra[:, 2] > 0].min()
    us = lambda x: round((float(x) - t0) / 1e3, 2)
    ea, eb = ra[ra[:, 29] > 0, 29], rb[rb[:, 29] > 0, 29]
    return {"A_first_tile_start": us(t0), "A_first_cta_exit": us(ea.min()), "A_last_cta_exit": us(ea.max()),
            "B_first_tile_start": us(rb[:, 2][rb[:, 2] > 0].min()), "B_last_tile_start": us(rb[:, 2].max()), "B_last_cta_exit": us(eb.max()),
            "B_tiles_started_before_A_exited": int((rb[:, 2][rb[:, 2] > 0] < ea.max()).sum()), "B_tiles": int((rb[:, 2] > 0).sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    snap = synth.generate(args.config)
    stream = torch.cuda.Stream()
    a, b = engine(snap, stream), engine(snap, stream)
    out = {"card": card(), "config": args.config, "steps": args.steps}
    out["queued_one_context_us_per_pass"] = round(queued_us(a, stream, snap.now, args.steps), 2)
    med, lo, hi = isolated_us(a, stream, snap.now, args.steps)
    out["isolated_us_per_pass"] = {"median": round(med, 2), "min": round(lo, 2), "max": round(hi, 2)}
    out["trace_two_passes"] = trace_pair(a, b, stream, snap.now)
    print(json.dumps(out))
    for e in (a, b):
        e.close()


if __name__ == "__main__":
    main()
