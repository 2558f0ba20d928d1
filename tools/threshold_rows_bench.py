"""Threshold column deltas on a GPU: what kt_update_threshold_rows costs beside a whole kt_upload_throttles (which recompiles every
selector table on the host and uploads every spec column again), and what the plugin's scheduling cycle gains when operators edit
temporaryThresholdOverrides.

    python tools/threshold_rows_bench.py [--baseline-library PATH] [--out FILE]

Engine: each call is timed with a host clock around the whole call (both end in a stream synchronisation), median of 50 after
5 warm-up calls, the two calls alternating, for k = 1, 16 and 256 edited throttles against the whole upload, at C2's throttle
count (1000 throttles) and C5's (10k), 20% of them with overrides as in C4, and a 100k-row pod slice (which neither call reads).
Each size runs twice: with the override counts kept (the in-place scatter) and with one override added to every listed throttle
(the override columns are rebuilt).  The whole upload is timed alone; the host layer's full path also re-sends the status and the reservations after it.
Plugin: a C2-shaped world (50 namespaces, 1000 throttles, 100k running pods, 10k queued pods).  The scheduler cycle by key
(PreFilter, Reserve on Success) runs over 1000 queued pods; every `every` pods one throttle gains or loses a temporary override.
Reported: us per pod and the queue passes (kth_queue_stats).  With --baseline-library (a libkt_b200.so without the delta path,
e.g. the parent commit's) the same cycle runs on it too, the two alternating round by round.  The card's name, power limit and
clocks are printed with the numbers."""
import argparse
import copy
import ctypes as C
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from namespace_rows_bench import alternate_us, card  # noqa: E402
from plugin_bench import SCHED, THROTTLER, namespace, pod, throttle  # noqa: E402


def listed_columns(snap, idx, bump, extra):
    """The threshold columns of the listed throttles as kt_update_threshold_rows takes them: thresholds raised by `bump`, and with
    `extra` one open override more per throttle."""
    from kube_throttler_b200 import abi

    R, off = snap.R, snap.ovr_off
    ent = np.concatenate([np.arange(off[t], off[t + 1]) for t in idx]).astype(np.int64) if len(idx) else np.zeros(0, np.int64)
    cnt = (off[idx + 1] - off[idx]).astype(np.int64)
    cols = dict(thr=snap.thr[:, idx] + bump, thr_present=snap.thr_present[idx], thr_cnt=snap.thr_cnt[idx], ovr_begin=snap.ovr_begin[ent],
                ovr_end=snap.ovr_end[ent], ovr_flags=snap.ovr_flags[ent], ovr_thr=snap.ovr_thr[:, ent], ovr_present=snap.ovr_present[ent],
                ovr_cnt=snap.ovr_cnt[ent])
    if extra:  # one more entry at the end of every listed throttle's overrides
        ends = np.cumsum(cnt)
        ins = lambda a, v: np.insert(a, ends, v, axis=a.ndim - 1)  # noqa: E731
        cols.update(ovr_begin=ins(cols["ovr_begin"], abi.TIME_OPEN_BEGIN), ovr_end=ins(cols["ovr_end"], abi.TIME_OPEN_END),
                    ovr_flags=ins(cols["ovr_flags"], 0), ovr_thr=ins(cols["ovr_thr"], 7), ovr_present=ins(cols["ovr_present"], 1),
                    ovr_cnt=ins(cols["ovr_cnt"], 0))
        cnt = cnt + 1
    cols["ovr_off"] = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
    return cols


def engine_calls():
    import kube_throttler_b200 as kt
    from kube_throttler_b200 import synth

    out = {}
    for name, kw in (("C2_1k", dict(config="C2", n=100_000, p=10_000)), ("C5_10k", dict(config="C5", n=100_000, p=10_000))):
        cfg = kw.pop("config")
        snap = synth.generate(cfg, override_frac=0.2, **kw).normalize()
        rng = np.random.default_rng(0)
        e = kt.Engine(snap.R, snap.L, snap.LN)
        e.upload_snapshot(snap)
        e.evaluate(snap.now)
        row = {"m": snap.m, "n_ovr": int(snap.ovr_off[-1])}
        for k in (1, 16, 256):
            idx = np.sort(rng.choice(snap.m, size=k, replace=False)).astype(np.int32)
            for extra in (False, True):
                # the whole upload restores the snapshot's columns, so every delta changes the listed columns again
                variants = [listed_columns(snap, idx, b, extra) for b in (1, 2)]
                state = {"i": 0}

                def delta():
                    state["i"] += 1
                    e.update_threshold_rows(idx, variants[state["i"] % 2])

                def full():
                    e.upload_throttles(snap)

                tag = "counts_changed" if extra else "counts_kept"
                row[f"update_threshold_rows_k{k}_{tag}_us"], row[f"upload_throttles_k{k}_{tag}_us"] = alternate_us(delta, full)
        e.close()
        out[name] = row
    return out


def world(library, n_ns, n_thr, n_run, n_pend, seed=2):
    from kube_throttler_b200 import host

    rng = random.Random(seed)
    w = host.Plugin(THROTTLER, SCHED, library=library)
    nss = [f"ns{i}" for i in range(n_ns)]
    w.apply(*[namespace(n) for n in nss])
    manifests = []
    for i in range(n_thr):
        t = {"resourceRequests": {"cpu": str(rng.randrange(50, 400)), "memory": f"{rng.randrange(64, 2048)}Gi"}}
        if rng.random() < 0.5:
            t["resourceCounts"] = {"pod": rng.randrange(20, 400)}
        manifests.append(throttle(nss[i % n_ns], f"t{i}", {"app": f"a{rng.randrange(64)}"}, t))
    w.apply(*manifests)

    def mk(i, pending):
        reqs = {"cpu": f"{rng.randrange(1, 80) * 50}m", "memory": f"{1 << rng.randrange(6, 14)}Mi"}
        labels = {"app": f"a{rng.randrange(64)}", "tier": f"x{rng.randrange(8)}"}
        return pod(rng.choice(nss), f"{'q' if pending else 'p'}{i}", labels, reqs, node="" if pending else "n", phase="Pending" if pending else "Running")

    for lo in range(0, n_run, 10_000):
        w.apply(*[mk(i, False) for i in range(lo, min(n_run, lo + 10_000))])
    pending = [mk(i, True) for i in range(n_pend)]
    w.apply(*pending)
    w.prefilter_queue()
    return w, pending, manifests


def cycle(w, pods, manifests, r, every):
    """PreFilter by key and Reserve on Success for `pods`; every `every` pods one throttle gains or loses a temporary override.
    Returns (seconds, queue passes)."""
    passes0 = w.queue_stats()["passes"]
    t0 = time.perf_counter()
    for i, p in enumerate(pods):
        if i % every == 0:
            j = (r * len(pods) + i) // every
            m = copy.deepcopy(manifests[(j * 37) % len(manifests)])
            if j % 2 == 0:
                m["spec"]["temporaryThresholdOverrides"] = [{"begin": "2025-01-01T00:00:00Z", "end": "",
                                                             "threshold": {"resourceRequests": {"cpu": str(100 + j % 50)}}}]
            w.apply(m)
        ns, name = p["metadata"]["namespace"], p["metadata"]["name"]
        if w.prefilter_key(ns, name)["code"] == "Success":
            w.reserve_key(ns, name)
    return time.perf_counter() - t0, w.queue_stats()["passes"] - passes0


def plugin_cycles(baseline, every=10):
    import kube_throttler_b200 as kt

    libs = {"delta_path": kt.lib()}
    if baseline:
        libs["baseline"] = C.CDLL(baseline)
    out = {}
    for name, shape in (("C2", (50, 1000, 100_000, 10_000)),):
        worlds = {k: world(L, *shape) for k, L in libs.items()}
        res = {k: {"seconds": 0.0, "passes": 0, "pods": 0} for k in libs}
        for r in range(10):  # 1000 pods, 100 per round; the builds alternate round by round
            for k, (w, pending, manifests) in worlds.items():
                s, n = cycle(w, pending[r * 100:(r + 1) * 100], manifests, r, every)
                res[k]["seconds"] += s
                res[k]["passes"] += n
                res[k]["pods"] += 100
        out[name] = {k: {"us_per_pod": round(v["seconds"] / v["pods"] * 1e6, 1), "queue_passes": v["passes"], "pods": v["pods"],
                         "override_edit_every": every} for k, v in res.items()}
        for w, _, _ in worlds.values():
            w.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-library", default=None, help="a libkt_b200.so without the threshold delta path, run alternately with this build")
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
