"""Cost of PreFilter for pods given by value on the device (kt_check_pods) against what the host layer did before it for a
manifest: the pods written into scratch rows behind the queue (kt_update_pod_rows), a GIVEN_STATUS | SKIP_RECONCILE pass over the
whole pending table, and kt_get_check_rows + kt_get_match_rows of the scratch rows.  C2's tables and running pods with pending
queues of 10^3 up to C2's 10^4 rows; k = 1, 16 and 256 pods.  The two sides run alternately, rep by rep (tools/reconcile_keys_bench.py
`alternate`: device time from CUDA events around the calls, wall time for the whole call).  Then kth_pre_filter(manifest) end to end
on a plugin loaded with tools/plugin_bench.py's C2 world, against the length of its resident queue.

    python tools/check_pods_bench.py [--queues 1000,3000,10000] [--reps 20] [--no-plugin] [--out check_pods.json]

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


def engine_side(p, reps):
    import torch

    snap = synth.generate("C2", p=p + 256)  # the last 256 rows are the scratch rows of the old path
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
    for k in (1, 16, 256):
        pods = snap.pending.rows(rng.integers(0, p, size=k))
        scratch = np.arange(p, p + k, dtype=np.int64)

        def scratch_pass():
            eng.update_pod_rows(abi.PODS_PENDING, scratch, pods)
            eng.evaluate(0, GIVEN)
            eng.get_check_rows(scratch)
            eng.match_rows(abi.PODS_PENDING, scratch)

        t = alternate({"check_pods": lambda: eng.check_pods(pods.labels, pods.req, pods.present, pods.ns_id), "scratch_rows_pass": scratch_pass}, reps)
        row = {"config": "C2", "queue": p, "m": int(snap.m), "k": k, **t}
        print(json.dumps(row), flush=True)
        out.append(row)
    eng.close()
    return out


def plugin_side(n_pend, calls=200):
    from plugin_bench import NOW, c2_world

    w, running, pending = c2_world(0, n_pend=n_pend)
    L, h = w._L, w._h
    for m in running:
        L.kth_apply(h, m)
    w.reconcile_all(NOW)
    for m in pending:
        L.kth_apply(h, json.dumps(m).encode())
    w.prefilter_queue()
    # manifests the informer does not hold: queued pods under other names
    manifests = [json.dumps(dict(m, metadata=dict(m["metadata"], name="manifest-" + m["metadata"]["name"]))).encode() for m in pending[:calls]]
    for m in manifests[:20]:  # warm-up
        L.kth_pre_filter(h, m)
    times = []
    for m in manifests:
        t0 = time.perf_counter()
        L.kth_pre_filter(h, m)
        times.append((time.perf_counter() - t0) * 1e6)
    row = {"plugin": f"C2 world (50 namespaces, 1000 Throttles, 100k running pods), {n_pend} queued pods", "calls": calls,
           "pre_filter_us_median": round(float(np.median(times)), 1), "pre_filter_us_p10": round(float(np.percentile(times, 10)), 1),
           "pre_filter_us_p90": round(float(np.percentile(times, 90)), 1), "device_queue_passes": w.queue_stats()["passes"]}
    print(json.dumps(row), flush=True)
    w.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queues", default="1000,3000,10000")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--no-plugin", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    torch.cuda.init()
    queues = [int(x) for x in args.queues.split(",")]
    res = {"card": card(), "reps": args.reps, "engine": [], "plugin": []}
    for p in queues:
        res["engine"] += engine_side(p, args.reps)
    if not args.no_plugin:
        res["plugin"] = [plugin_side(p) for p in queues]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
