"""Selector column deltas on a GPU: what kt_update_selector_rows costs beside a whole kt_upload_throttles (which recompiles every
selector table on the host and uploads every spec column again), and what the plugin's scheduling cycle gains when Throttles are
deleted or their selectors edited.

    python tools/selector_rows_bench.py [--baseline-library PATH] [--out FILE]

Engine: each call is timed with a host clock around the whole call (both end in a stream synchronisation), median of 50 after
5 warm-up calls, the two calls alternating, for k = 1, 16 and 256 listed throttles against the whole upload, at C2's throttle
count (1000 throttles) and C5's (10k), 40% of them ClusterThrottles, 500 namespaces and a 100k-row pod slice.  Two kinds of
delta: deletions (no terms, flags 0) and selector edits (each listed column takes another column's terms); every other call puts
the original columns back, so every call changes its columns and every call fits the resident tables.
Plugin: tools/plugin_bench.py's C2-shaped world (50 namespaces, 1000 throttles, 100k running pods, 10k queued pods).  The
scheduler cycle by key (PreFilter, Reserve on Success) runs over 1000 queued pods; every `every` pods one throttle is deleted or
its podSelector moved to another label value the dictionaries hold, in turn.  Reported: us per pod and the queue passes
(kth_queue_stats).  With --baseline-library (a libkt_b200.so without the delta path, e.g. the parent commit's) the same cycle runs
on it too, the two alternating round by round.  The card's name, power limit and clocks are printed with the numbers."""
import argparse
import copy
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from namespace_rows_bench import alternate_us, card  # noqa: E402
from threshold_rows_bench import world  # noqa: E402


def listed_columns(snap, idx, terms_of):
    """kind / thr_ns / thr_flags and the selector CSR of the listed columns, column idx[i] taking the terms of column terms_of[i]
    (-1: none, flags 0 -- a deletion)."""
    term_flags, pod_off, ns_off, key, op, val_off, vals, tcount = [], [0], [], [], [], [0], [], []
    terms = [j for s in terms_of for j in (range(snap.term_off[s], snap.term_off[s + 1]) if s >= 0 else ())]

    def push(q0, q1):
        for q in range(q0, q1):
            key.append(snap.req_key[q])
            op.append(snap.req_op[q])
            vals.extend(snap.req_vals[snap.req_val_off[q]:snap.req_val_off[q + 1]])
            val_off.append(len(vals))

    for s in terms_of:
        tcount.append(0 if s < 0 else int(snap.term_off[s + 1] - snap.term_off[s]))
    for j in terms:
        term_flags.append(snap.term_flags[j])
        push(snap.pod_req_off[j], snap.pod_req_off[j + 1])
        pod_off.append(len(key))
    ns_off.append(len(key))
    for j in terms:
        push(snap.ns_req_off[j], snap.ns_req_off[j + 1])
        ns_off.append(len(key))
    flags = np.where(np.asarray(terms_of) >= 0, snap.thr_flags[idx], 0).astype(np.uint8)
    return dict(kind=snap.kind[idx], thr_ns=snap.thr_ns[idx], thr_flags=flags, term_off=np.cumsum([0] + tcount).astype(np.int32),
                term_flags=np.array(term_flags, np.uint8), pod_req_off=np.array(pod_off, np.int32), ns_req_off=np.array(ns_off, np.int32),
                req_key=np.array(key, np.uint32), req_op=np.array(op, np.uint8), req_val_off=np.array(val_off, np.int32),
                req_vals=np.array(vals, np.uint32))


def engine_calls():
    import kube_throttler_b200 as kt
    from kube_throttler_b200 import synth

    out = {}
    for name, cfg in (("C2_1k", "C2"), ("C5_10k", "C5")):
        snap = synth.generate(cfg, n=100_000, p=10_000, n_ns=500, cluster_frac=0.4).normalize()
        rng = np.random.default_rng(0)
        e = kt.Engine(snap.R, snap.L, snap.LN)
        e.upload_snapshot(snap)
        e.evaluate(snap.now)
        row = {"m": snap.m, "n_ns": snap.n_ns}
        for k in (1, 16, 256):
            idx = np.sort(rng.choice(snap.m, size=k, replace=False)).astype(np.int32)
            same_kind = {kd: np.nonzero(snap.kind == kd)[0] for kd in np.unique(snap.kind)}
            for what in ("delete", "edit"):
                other = np.full(k, -1) if what == "delete" else np.array([rng.choice(same_kind[snap.kind[t]]) for t in idx])
                variants = [listed_columns(snap, idx, other), listed_columns(snap, idx, idx)]  # changed, then back
                state = {"i": 0, "recompiled": 0}

                def delta():
                    state["i"] += 1
                    state["recompiled"] += e.update_selector_rows(idx, variants[state["i"] % 2])

                def full():
                    e.upload_throttles(snap)

                row[f"update_selector_rows_k{k}_{what}_us"], row[f"upload_throttles_k{k}_{what}_us"] = alternate_us(delta, full)
                row[f"k{k}_{what}_recompiled_calls"] = state["recompiled"]
        e.close()
        out[name] = row
    return out


def cycle(w, pods, manifests, r, every, state):
    """PreFilter by key and Reserve on Success for `pods`; every `every` pods one throttle is deleted or its podSelector moved to
    another label value, in turn.  Returns (seconds, queue passes)."""
    passes0 = w.queue_stats()["passes"]
    t0 = time.perf_counter()
    for i, p in enumerate(pods):
        if i % every == 0:
            j = (r * len(pods) + i) // every
            t = manifests[(j * 37) % len(manifests)]
            key = (t["metadata"]["namespace"], t["metadata"]["name"])
            if j % 2 == 0 and key not in state["deleted"]:
                w.delete("Throttle", key[1], key[0])
                state["deleted"].add(key)
            elif key not in state["deleted"]:
                m = copy.deepcopy(t)
                m["spec"]["selector"]["selectorTerms"] = [{"podSelector": {"matchLabels": {"app": f"a{(j * 11) % 64}"}}}]
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
        state = {k: {"deleted": set()} for k in libs}
        res = {k: {"seconds": 0.0, "passes": 0, "pods": 0} for k in libs}
        for r in range(10):  # 1000 pods, 100 per round; the builds alternate round by round
            for k, (w, pending, manifests) in worlds.items():
                s, n = cycle(w, pending[r * 100:(r + 1) * 100], manifests, r, every, state[k])
                res[k]["seconds"] += s
                res[k]["passes"] += n
                res[k]["pods"] += 100
        out[name] = {k: {"us_per_pod": round(v["seconds"] / v["pods"] * 1e6, 1), "queue_passes": v["passes"], "pods": v["pods"],
                         "delete_or_edit_every": every} for k, v in res.items()}
        for w, _, _ in worlds.values():
            w.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-library", default=None, help="a libkt_b200.so without the selector delta path, run alternately with this build")
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
