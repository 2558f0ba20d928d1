"""Namespace row deltas on a GPU: what kt_update_namespace_rows costs beside a whole kt_upload_namespaces (which recompiles every
selector table on the host and uploads them again), and what the plugin's scheduling cycle gains when namespaces come and go.

    python tools/namespace_rows_bench.py [--baseline-library PATH] [--out FILE]

Engine: each call is timed with a host clock around the whole call (both end in a stream synchronisation), median of 50 after
5 warm-up calls, the two calls alternating, for k = 1, 16 and 256 relabelled namespaces against the full upload of the same rows,
at C2's throttle count (1000 throttles) and C5's (10k), 40% of them ClusterThrottles (the synthetic C2 and C5 have none), 500
namespaces and a 100k-row pod slice (which neither call reads).
Plugin: a C2-shaped world (50 namespaces, 1000 throttles of which 300 ClusterThrottles, 100k running pods, 10k queued pods).
The scheduler cycle by key (PreFilter, Reserve on Success) runs over 1000 queued pods; a new namespace is created every 10 pods.
Reported: us per pod and the queue passes (kth_queue_stats).  With --baseline-library (a libkt_b200.so without the row path,
e.g. the parent commit's) the same cycle runs on it too, the two alternating round by round.  The card's name, power limit and
clocks are printed with the numbers."""
import argparse
import ctypes as C
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from plugin_bench import SCHED, THROTTLER, namespace, pod, throttle  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def alternate_us(fa, fb, n=50, warm=5):
    """Medians (us) of two calls timed alternately."""
    for _ in range(warm):
        fa()
        fb()
    ta, tb = [], []
    for _ in range(n):
        for f, ts in ((fa, ta), (fb, tb)):
            t0 = time.perf_counter()
            f()
            ts.append(time.perf_counter() - t0)
    return round(statistics.median(ta) * 1e6, 1), round(statistics.median(tb) * 1e6, 1)


def engine_calls():
    import kube_throttler_b200 as kt
    from kube_throttler_b200 import synth

    out = {}
    for name, kw in (("C2_1k", dict(config="C2", n=100_000, p=10_000)), ("C5_10k", dict(config="C5", n=100_000, p=10_000))):
        cfg = kw.pop("config")
        snap = synth.generate(cfg, cluster_frac=0.4, n_ns=500, **kw).normalize()
        rng = np.random.default_rng(0)
        e = kt.Engine(snap.R, snap.L, snap.LN)
        e.upload_snapshot(snap)
        e.evaluate(snap.now)
        rows = snap.ns_labels.copy()
        n = rows.shape[1]
        tb = e.ns_tables()
        row = {"m": snap.m, "n_ns": n, "max_ns_words": tb["max_ns_words"], "words": int(tb["nsw_off"][-1])}
        for k in (1, 16, 256):
            idx = np.sort(rng.choice(n, size=k, replace=False)).astype(np.int32)
            variants = [rows[:, rng.permutation(n)[:k]] for _ in range(4)]  # other namespaces' labels: selectors flip both ways
            state = {"i": 0}

            def delta():
                state["i"] += 1
                v = variants[state["i"] % 4]
                rows[:, idx] = v
                e.update_namespace_rows(n, idx, v)

            def full():
                e.upload_namespaces(rows)

            row[f"update_namespace_rows_k{k}_us"], row[f"upload_namespaces_k{k}_us"] = alternate_us(delta, full)
        e.close()
        out[name] = row
    return out


def world(library, n_ns, n_thr, n_cluster, n_run, n_pend, seed=2):
    from kube_throttler_b200 import host

    rng = random.Random(seed)
    w = host.Plugin(THROTTLER, SCHED, library=library)
    nss = [f"ns{i}" for i in range(n_ns)]
    w.apply(*[namespace(n, {"team": f"t{i % 7}"}) for i, n in enumerate(nss)])
    for i in range(n_thr):
        t = {"resourceRequests": {"cpu": str(rng.randrange(50, 400)), "memory": f"{rng.randrange(64, 2048)}Gi"}}
        if rng.random() < 0.5:
            t["resourceCounts"] = {"pod": rng.randrange(20, 400)}
        if i < n_cluster:
            m = {"kind": "ClusterThrottle", "metadata": {"name": f"c{i}"},
                 "spec": {"throttlerName": THROTTLER, "threshold": t,
                          "selector": {"selectorTerms": [{"podSelector": {"matchLabels": {"app": f"a{rng.randrange(64)}"}},
                                                          "namespaceSelector": {"matchLabels": {"team": f"t{rng.randrange(7)}"}}}]}}}
        else:
            m = throttle(nss[i % n_ns], f"t{i}", {"app": f"a{rng.randrange(64)}"}, t)
        w.apply(m)

    def mk(i, pending):
        reqs = {"cpu": f"{rng.randrange(1, 80) * 50}m", "memory": f"{1 << rng.randrange(6, 14)}Mi"}
        labels = {"app": f"a{rng.randrange(64)}", "tier": f"x{rng.randrange(8)}"}
        return pod(rng.choice(nss), f"{'q' if pending else 'p'}{i}", labels, reqs, node="" if pending else "n", phase="Pending" if pending else "Running")

    for lo in range(0, n_run, 10_000):
        w.apply(*[mk(i, False) for i in range(lo, min(n_run, lo + 10_000))])
    pending = [mk(i, True) for i in range(n_pend)]
    w.apply(*pending)
    w.prefilter_queue()
    return w, pending


def cycle(w, pods, tag, every):
    """PreFilter by key and Reserve on Success for `pods`, a new namespace every `every` pods.  Returns (seconds, queue passes)."""
    passes0 = w.queue_stats()["passes"]
    t0 = time.perf_counter()
    for i, p in enumerate(pods):
        if i % every == 0:
            w.apply(namespace(f"job-{tag}-{i}", {"team": f"t{i % 7}"}))
        ns, name = p["metadata"]["namespace"], p["metadata"]["name"]
        if w.prefilter_key(ns, name)["code"] == "Success":
            w.reserve_key(ns, name)
    return time.perf_counter() - t0, w.queue_stats()["passes"] - passes0


def plugin_cycles(baseline, every=10):
    import kube_throttler_b200 as kt

    libs = {"row_path": kt.lib()}
    if baseline:
        libs["baseline"] = C.CDLL(baseline)
    out = {}
    for name, shape in (("C2", (50, 1000, 300, 100_000, 10_000)),):
        worlds = {k: world(L, *shape) for k, L in libs.items()}
        res = {k: {"seconds": 0.0, "passes": 0, "pods": 0} for k in libs}
        for r in range(10):  # 1000 pods, 100 per round; the builds alternate round by round
            for k, (w, pending) in worlds.items():
                s, n = cycle(w, pending[r * 100:(r + 1) * 100], f"r{r}", every)
                res[k]["seconds"] += s
                res[k]["passes"] += n
                res[k]["pods"] += 100
        out[name] = {k: {"us_per_pod": round(v["seconds"] / v["pods"] * 1e6, 1), "queue_passes": v["passes"], "pods": v["pods"],
                         "namespace_every": every} for k, v in res.items()}
        for w, _ in worlds.values():
            w.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-library", default=None, help="a libkt_b200.so without the namespace row path, run alternately with this build")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card(), "engine": engine_calls(), "plugin": plugin_cycles(args.baseline_library), "card_after": card()}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
