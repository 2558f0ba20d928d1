"""Throttle-side column deltas on a GPU: what kt_update_status_rows / kt_update_reserved_rows cost beside the whole-table
kt_upload_status / kt_set_reserved, and what the plugin's scheduling cycle gains from them.

    python tools/throttle_rows_bench.py [--baseline-library PATH] [--out FILE]

Engine: every call is timed with a host clock around the whole call (each one ends in a stream synchronisation), median of 200
after 20 warm-up calls, for k = 1, 16 and 256 listed columns against the full call, at BASELINE C2 (1000 throttles) and C5's
throttle count (10k throttles; a 100k-row pod slice, which the calls do not read).
Plugin: a C2-shaped world (50 namespaces, 1000 Throttles, 100k running pods) and a C5-sized one (500 namespaces, 10k Throttles,
100k running pods), each with 10k queued pods.  The scheduler cycle by key (PreFilter, Reserve on Success) runs over 1000 queued
pods; every 100 pods the reserved ones are bound, the Throttles of the namespaces those pods live in are reconciled by key, and
every status the reconcile wrote comes back through the informer (the echo).  Reported: us per pod and the queue passes (kth_queue_stats).  With
--baseline-library (a build of libkt_b200.so without the column deltas, e.g. the parent commit's) the same cycle runs on it too,
the two alternating round by round.  The card's name and power limit are printed with the numbers."""
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

from plugin_bench import NOW, SCHED, THROTTLER, namespace, pod, throttle  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def median_us(f, n=200, warm=20):
    for _ in range(warm):
        f()
    ts = []
    for _ in range(n):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return round(statistics.median(ts) * 1e6, 1)


def engine_calls():
    import kube_throttler_b200 as kt
    from kube_throttler_b200 import abi, synth

    out = {}
    for name, kw in (("C2", dict(config="C2")), ("C5_throttles", dict(config="C5", n=100_000, p=10_000))):
        cfg = kw.pop("config")
        snap = synth.generate(cfg, **kw).normalize()
        m, R = snap.m, snap.R
        rng = np.random.default_rng(0)
        snap.status = dict(calculated=np.ones(m, np.uint8), calc_thr=rng.integers(0, 1 << 30, (R, m)), calc_present=np.full(m, 0xF, np.uint32),
                           calc_cnt=rng.integers(0, 100, m), used=rng.integers(0, 1 << 30, (R, m)), used_present=np.full(m, 0xF, np.uint32),
                           used_cnt=rng.integers(0, 100, m), throttled=np.zeros(m, np.uint32))
        snap.reserved, snap.reserved_present, snap.reserved_cnt = rng.integers(0, 1 << 20, (R, m)), np.full(m, abi.COUNT_BIT | 0xF, np.uint32), rng.integers(0, 9, m)
        snap.normalize()
        e = kt.Engine(snap.R, snap.L, snap.LN)
        e.upload_snapshot(snap)
        row = {"m": m, "upload_status_us": median_us(lambda: e.upload_status(snap)), "set_reserved_us": median_us(lambda: e.set_reserved(snap))}
        for k in (1, 16, 256):
            idx = np.sort(rng.choice(m, size=k, replace=False)).astype(np.int32)
            st = {f: (v[:, idx] if v.ndim == 2 else v[idx]) for f, v in snap.status.items()}
            res = (snap.reserved[:, idx].copy(), snap.reserved_present[idx].copy(), snap.reserved_cnt[idx].copy())
            row[f"update_status_rows_k{k}_us"] = median_us(lambda: e.update_status_rows(idx, st))
            row[f"update_reserved_rows_k{k}_us"] = median_us(lambda: e.update_reserved_rows(idx, *res))
        e.close()
        out[name] = row
    return out


def world(library, n_ns, n_thr, n_run, n_pend, seed=2):
    from kube_throttler_b200 import host

    rng = random.Random(seed)
    w = host.Plugin(THROTTLER, SCHED, library=library)
    nss = [f"ns{i}" for i in range(n_ns)]
    w.apply(*[namespace(n, {"team": f"t{i % 7}"}) for i, n in enumerate(nss)])
    thr = {}
    for i in range(n_thr):
        t = {"resourceRequests": {"cpu": str(rng.randrange(50, 400)), "memory": f"{rng.randrange(64, 2048)}Gi"}}
        if rng.random() < 0.5:
            t["resourceCounts"] = {"pod": rng.randrange(20, 400)}
        m = throttle(nss[i % n_ns], f"t{i}", {"app": f"a{rng.randrange(64)}"}, t)
        thr[f"{nss[i % n_ns]}/t{i}"] = m
        w.apply(m)

    def mk(i, pending):
        reqs = {"cpu": f"{rng.randrange(1, 80) * 50}m", "memory": f"{1 << rng.randrange(6, 14)}Mi"}
        labels = {"app": f"a{rng.randrange(64)}", "tier": f"x{rng.randrange(8)}"}
        return pod(rng.choice(nss), f"{'q' if pending else 'p'}{i}", labels, reqs, node="" if pending else "n", phase="Pending" if pending else "Running")

    for lo in range(0, n_run, 10_000):
        w.apply(*[mk(i, False) for i in range(lo, min(n_run, lo + 10_000))])
    pending = [mk(i, True) for i in range(n_pend)]
    w.apply(*pending)
    by_ns = {}
    for key in thr:
        by_ns.setdefault(key.split("/")[0], []).append(key)
    w.reconcile_all(NOW)
    return w, thr, by_ns, pending


def cycle(w, thr, by_ns, pods, now):
    """PreFilter by key and Reserve on Success for `pods`; afterwards reconcile(key) of the Throttles of their namespaces and the
    echo of every status it wrote.  Returns (seconds, queue passes)."""
    passes0 = w.queue_stats()["passes"]
    t0 = time.perf_counter()
    nss, bound = set(), []
    for p in pods:
        ns, name = p["metadata"]["namespace"], p["metadata"]["name"]
        nss.add(ns)
        if w.prefilter_key(ns, name)["code"] == "Success":
            w.reserve_key(ns, name)
            bound.append(dict(p, spec=dict(p["spec"], nodeName="n"), status={"phase": "Running"}))
    w.apply(*bound)  # the reserved pods are bound: the reconcile below counts them
    keys = [k for ns in sorted(nss) for k in by_ns.get(ns, [])]
    got = w.reconcile(keys, now)
    for key in got["changed"]:
        ns, _, name = key.partition("/")
        w.apply(dict(thr[key], status=json.loads(w.status_manifest(name, ns))))
    return time.perf_counter() - t0, w.queue_stats()["passes"] - passes0


def plugin_cycles(baseline):
    import kube_throttler_b200 as kt

    libs = {"deltas": kt.lib()}
    if baseline:
        libs["baseline"] = C.CDLL(baseline)
    out = {}
    for name, shape in (("C2", (50, 1000, 100_000, 10_000)), ("C5_sized", (500, 10_000, 100_000, 10_000))):
        worlds = {k: world(L, *shape) for k, L in libs.items()}
        res = {k: {"seconds": 0.0, "passes": 0, "pods": 0} for k in libs}
        times = ["2026-01-01T00:00:%02dZ" % s for s in range(60)]
        for r in range(10):  # 1000 pods, 100 per round; the builds alternate round by round
            for k, (w, thr, by_ns, pending) in worlds.items():
                s, n = cycle(w, thr, by_ns, pending[r * 100:(r + 1) * 100], times[r + 1])
                res[k]["seconds"] += s
                res[k]["passes"] += n
                res[k]["pods"] += 100
        out[name] = {k: {"us_per_pod": round(v["seconds"] / v["pods"] * 1e6, 1), "queue_passes": v["passes"], "pods": v["pods"]} for k, v in res.items()}
        for w, *_ in worlds.values():
            w.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-library", default=None, help="a libkt_b200.so without the column deltas, run alternately with this build")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card(), "engine": engine_calls(), "plugin": plugin_cycles(args.baseline_library)}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
