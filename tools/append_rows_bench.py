"""Column appends on a GPU: what kt_append_throttle_rows costs beside the whole path it replaces for a Throttle or ClusterThrottle
creation (kt_upload_throttles of the grown spec, which recompiles every selector table on the host, then the status and the
reservations uploaded again), and what a hole fill through the existing column deltas costs beside the same whole path.

    python tools/append_rows_bench.py [--baseline-library PATH] [--out FILE]

Each call is timed with a host clock around the whole call (every call ends in a stream synchronisation), median of 50 after 5
warm-up calls, delta and whole path alternating, at C2's throttle count (1000 throttles) and C5's (10k), 40% of them
ClusterThrottles, 500 namespaces and a 100k-row pod slice.  The engine cannot drop columns, so before every timed append (and
every timed whole path) the base spec is uploaded again, untimed.  Cases: k = 1 inside the last 32-throttle word, k = 4 across a
word boundary, k = 4 across a 128-column boundary (the bitmap row width grows), k = 256; and a hole fill: one column's
selector, thresholds, status and reservations replaced through kt_update_selector_rows, kt_update_threshold_rows,
kt_update_status_rows and kt_update_reserved_rows.
Plugin: tools/plugin_bench.py's C2-shaped world (50 namespaces, 1000 throttles, 100k running pods, 10k queued pods).  The
scheduler cycle by key (PreFilter, Reserve on Success) runs over 1000 queued pods; every `every` pods one Throttle is deleted and
another created in a namespace that has throttles, with a known podSelector.  Reported: us per pod and the queue passes
(kth_queue_stats).  With --baseline-library (a libkt_b200.so without the creation delta, e.g. the parent commit's) the same
cycle runs on it too, the two alternating round by round.  The card's name, power limit and clocks are printed with the
numbers."""
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
from selector_rows_bench import listed_columns  # noqa: E402
from threshold_rows_bench import world  # noqa: E402

STATUS = ("calculated", "calc_thr", "calc_present", "calc_cnt", "used", "used_present", "used_cnt", "throttled")


def columns_of(snap, idx):
    """The listed columns shaped for kt_append_throttle_rows / kt_upload_throttles: spec, thresholds and override CSR."""
    idx = np.asarray(idx)
    spans = [(int(snap.ovr_off[t]), int(snap.ovr_off[t + 1])) for t in idx]
    e = np.array([j for a, b in spans for j in range(a, b)], np.int64)
    d = listed_columns(snap, idx, idx)
    d.update(thr=snap.thr[:, idx], thr_present=snap.thr_present[idx], thr_cnt=snap.thr_cnt[idx],
             ovr_off=np.cumsum([0] + [b - a for a, b in spans]).astype(np.int32), ovr_begin=snap.ovr_begin[e], ovr_end=snap.ovr_end[e],
             ovr_flags=snap.ovr_flags[e], ovr_thr=snap.ovr_thr[:, e], ovr_present=snap.ovr_present[e], ovr_cnt=snap.ovr_cnt[e])
    return d


def prefix(snap, m):
    """The snapshot with its first m throttle columns, an observed status and reservations."""
    s = copy.copy(snap)
    for f, v in columns_of(snap, np.arange(m)).items():
        setattr(s, f, np.ascontiguousarray(v))
    rng = np.random.default_rng(m)
    s.status = {f: rng.integers(0, 3, size=(snap.R, m) if f in ("calc_thr", "used") else m) for f in STATUS}
    s.reserved = np.zeros((snap.R, m), np.int64)
    s.reserved_present, s.reserved_cnt = np.zeros(m, np.uint32), np.zeros(m, np.int64)
    return s.normalize()


def engine_calls():
    import kube_throttler_b200 as kt
    from kube_throttler_b200 import synth

    out = {}
    for name, cfg in (("C2_1k", "C2"), ("C5_10k", "C5")):
        snap = synth.generate(cfg, n=100_000, p=10_000, n_ns=500, cluster_frac=0.4).normalize()
        m = snap.m
        q = (m - 300) // 128
        cases = {"in_word_k1": (32 * 4 * q + 5, 1), "cross_word_k4": (32 * 4 * q + 30, 4), "cross_wp_k4": (128 * (q + 1) - 2, 4),
                 "k256": (m - 256, 256)}
        e = kt.Engine(snap.R, snap.L, snap.LN)
        e.upload_snapshot(snap)
        row = {"m": m, "n_ns": snap.n_ns}
        for case, (m0, k) in cases.items():
            base, grown = prefix(snap, m0), prefix(snap, m0 + k)
            grown.status = {f: np.concatenate([base.status[f], np.zeros(base.status[f].shape[:-1] + (k,), base.status[f].dtype)], axis=-1)
                            for f in STATUS}
            new = {f: np.ascontiguousarray(v) for f, v in columns_of(snap, np.arange(m0, m0 + k)).items()}
            state = {"recompiled": 0}

            def reset():
                e.upload_throttles(base)
                e.upload_status(base)
                e.set_reserved(base)
                e.evaluate(snap.now)

            def delta():
                state["recompiled"] += e.append_throttle_rows(new)

            def full():
                e.upload_throttles(grown)
                e.upload_status(grown)
                e.set_reserved(grown)

            ta, tb = [], []
            for i in range(55):  # 5 warm-up rounds, then 50 timed
                for f, ts in ((delta, ta), (full, tb)):
                    reset()
                    t0 = time.perf_counter()
                    f()
                    dt = time.perf_counter() - t0
                    if i >= 5:
                        ts.append(dt)
            row[f"append_{case}_us"] = round(float(np.median(ta)) * 1e6, 1)
            row[f"whole_{case}_us"] = round(float(np.median(tb)) * 1e6, 1)
            row[f"{case}_recompiled_calls"] = state["recompiled"]
        # a hole fill through the existing deltas against the whole path
        full_snap = prefix(snap, m)
        e.upload_throttles(full_snap)
        e.upload_status(full_snap)
        e.set_reserved(full_snap)
        t = np.array([m // 2], np.int32)
        cols = columns_of(full_snap, t)
        st = {f: (v[:, t] if v.ndim == 2 else v[t]) for f, v in full_snap.status.items()}

        def hole():
            e.update_selector_rows(t, cols)
            e.update_threshold_rows(t, cols)
            e.update_status_rows(t, st)
            e.update_reserved_rows(t, full_snap.reserved[:, t], full_snap.reserved_present[t], full_snap.reserved_cnt[t])

        def whole():
            e.upload_throttles(full_snap)
            e.upload_status(full_snap)
            e.set_reserved(full_snap)

        row["hole_fill_us"], row["whole_hole_fill_us"] = alternate_us(hole, whole)
        e.close()
        out[name] = row
    return out


def churn_cycle(w, pods, manifests, r, every, state):
    """PreFilter by key and Reserve on Success for `pods`; every `every` pods one Throttle is deleted and another created (a new
    name in the same namespace, with the podSelector of a throttle that exists).  Returns (seconds, queue passes)."""
    passes0 = w.queue_stats()["passes"]
    t0 = time.perf_counter()
    for i, p in enumerate(pods):
        if i % every == 0:
            j = (r * len(pods) + i) // every
            old = manifests[(j * 37) % len(manifests)]
            key = (old["metadata"]["namespace"], old["metadata"]["name"])
            if key not in state["deleted"]:
                w.delete("Throttle", key[1], key[0])
                state["deleted"].add(key)
            m = copy.deepcopy(manifests[(j * 53 + 1) % len(manifests)])
            m["metadata"] = dict(m["metadata"], name=f"churn-{j}")
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
    worlds = {k: world(L, 50, 1000, 100_000, 10_000) for k, L in libs.items()}
    state = {k: {"deleted": set()} for k in libs}
    res = {k: {"seconds": 0.0, "passes": 0, "pods": 0} for k in libs}
    for r in range(10):  # 1000 pods, 100 per round; the builds alternate round by round
        for k, (w, pending, manifests) in worlds.items():
            s, n = churn_cycle(w, pending[r * 100:(r + 1) * 100], manifests, r, every, state[k])
            res[k]["seconds"] += s
            res[k]["passes"] += n
            res[k]["pods"] += 100
    for w, _, _ in worlds.values():
        w.close()
    return {"C2": {k: {"us_per_pod": round(v["seconds"] / v["pods"] * 1e6, 1), "queue_passes": v["passes"], "pods": v["pods"],
                       "delete_and_create_every": every} for k, v in res.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-library", default=None, help="a libkt_b200.so without the creation delta path, run alternately with this build")
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
