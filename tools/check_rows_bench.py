"""Cost of PreFilter for listed pending rows on the device (kt_check_pending_rows) against what a caller had before it: a
GIVEN_STATUS | SKIP_RECONCILE pass over the whole pending table plus kt_get_check_rows of the same rows.  For C2 (P = 10k) and
C5 (P = 100k): k = 1, 16, 256 and 4096 random rows.  The two sides run alternately, rep by rep; device time from CUDA events
around the calls (both synchronise their stream before they return), wall time for the whole call.  Then, on a plugin loaded
with tools/plugin_bench.py's C2 world (10k queued pods) and with the same world and a 100k-pod queue, the scheduler's cycle by
key -- PreFilter, then Reserve on Success -- with kth_pre_filter_key against kth_pre_filter_keys([key]), in alternating chunks of
pods.

    python tools/check_rows_bench.py [--configs C2,C5] [--reps 20] [--no-plugin] [--out check_rows.json]

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
from kube_throttler_b200 import abi, synth  # noqa: E402
from reconcile_keys_bench import alternate, card  # noqa: E402

GIVEN = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE


def engine_side(cfg, reps):
    import torch

    snap = synth.generate(cfg)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    eng.upload_snapshot(snap)
    eng.evaluate(snap.now)
    st = eng.download()
    snap.status = dict(calculated=np.ones(snap.m, np.uint8), calc_thr=st.calc_thr, calc_present=st.calc_present, calc_cnt=st.calc_cnt,
                       used=st.used, used_present=st.used_present, used_cnt=st.used_cnt, throttled=st.throttled)
    snap.normalize()
    eng.upload_status(snap)
    rng = np.random.default_rng(0)
    out = []
    for k in (1, 16, 256, 4096):
        rows = np.ascontiguousarray(rng.integers(0, snap.pending.n, size=k), np.int64)

        def full_pass():
            eng.evaluate(0, GIVEN)
            eng.get_check_rows(rows)

        t = alternate({"check_pending_rows": lambda: eng.check_pending_rows(rows), "pass_plus_check_rows": full_pass}, reps)
        row = {"config": cfg, "p": int(snap.pending.n), "m": int(snap.m), "k": k, **t}
        print(json.dumps(row), flush=True)
        out.append(row)
    eng.close()
    return out


def plugin_side(n_pend, chunk=100, chunks=6):
    from plugin_bench import NOW, c2_world

    w, running, pending = c2_world(0, n_pend=n_pend)
    L, h = w._L, w._h
    for m in running:
        L.kth_apply(h, m)
    w.reconcile_all(NOW)
    for m in pending:
        L.kth_apply(h, json.dumps(m).encode())
    keys = [(m["metadata"]["namespace"], m["metadata"]["name"]) for m in pending]
    by_key = lambda ns, name: L.kth_pre_filter_key(h, ns.encode(), name.encode())
    by_keys = lambda ns, name: L.kth_pre_filter_keys(h, json.dumps([ns + "/" + name]).encode())

    def cycle(pre, part):  # the scheduler's cycle by key: PreFilter -> Reserve on Success
        admitted = 0
        t0 = time.perf_counter()
        for ns, name in part:
            r = pre(ns, name)
            if b'"code":"Success"' in r[:24]:
                L.kth_reserve_key(h, ns.encode(), name.encode())
                admitted += 1
        return (time.perf_counter() - t0) / len(part) * 1e6, admitted

    w.queue_stats()
    cycle(by_key, keys[-20:]), cycle(by_keys, keys[-40:-20])  # warm-up
    res = {"pre_filter_key": [], "pre_filter_keys": []}
    adm = {"pre_filter_key": 0, "pre_filter_keys": 0}
    passes = {"pre_filter_key": 0, "pre_filter_keys": 0}
    for c in range(2 * chunks):  # alternately, chunk by chunk
        name, pre = ("pre_filter_key", by_key) if c % 2 == 0 else ("pre_filter_keys", by_keys)
        s0 = w.queue_stats()["passes"]
        us, a = cycle(pre, keys[c * chunk:(c + 1) * chunk])
        passes[name] += w.queue_stats()["passes"] - s0
        res[name].append(us)
        adm[name] += a
    row = {"plugin": f"C2 world (50 namespaces, 1000 Throttles, 100k running pods), {n_pend} queued pods", "pods_per_side": chunk * chunks}
    for name in res:
        row[name] = {"us_per_pod_median": round(float(np.median(res[name])), 1), "admitted": adm[name], "device_queue_passes": passes[name]}
    print(json.dumps(row), flush=True)
    w.close()
    return row


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
        res["plugin"] = [plugin_side(10_000), plugin_side(100_000)]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
