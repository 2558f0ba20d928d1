"""Column moves on a GPU: what kt_move_throttle_columns costs beside the whole path it replaces (kt_upload_throttles of the new
layout, which recompiles every selector table on the host, then the status and the reservations uploaded again).

    python tools/move_columns_bench.py [--out FILE]

Each call is timed with a host clock around the whole call (every call ends in a stream synchronisation), median of 50 after 5
warm-up calls, move and whole path alternating, at C2's throttle count (1000 throttles) and C5's (10k), 40% of them
ClusterThrottles, 500 namespaces and a 100k-row pod slice.  Before every timed call the starting layout is uploaded again,
untimed.  Cases:
  - creation into a full group: an empty column opened in the middle (every later column moves one place), then filled through
    kt_update_selector_rows, kt_update_threshold_rows, kt_update_status_rows and kt_update_reserved_rows;
  - compaction of 10% and of 50% holes (deleted columns: no terms, flags 0) spread over the layout.
The card's name, power limit and clocks are printed with the numbers."""
import argparse
import copy
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from append_rows_bench import STATUS, columns_of  # noqa: E402
from namespace_rows_bench import card  # noqa: E402
from selector_rows_bench import listed_columns  # noqa: E402


def layout(snap, idx, dead=()):
    """The snapshot whose column j is column idx[j] of snap (the `dead` positions deleted: no terms, flags 0), with an observed
    status and reservations gathered the same way from a status of the whole snap."""
    s = copy.copy(snap)
    idx = np.asarray(idx)
    for f, v in columns_of(snap, idx).items():
        setattr(s, f, np.ascontiguousarray(v))
    if len(dead):
        terms_of = idx.copy()
        terms_of[np.asarray(dead)] = -1
        for f, v in listed_columns(snap, idx, terms_of).items():
            setattr(s, f, np.ascontiguousarray(v))
        s.thr_flags = s.thr_flags.copy()
        s.thr_flags[np.asarray(dead)] = 0
    rng = np.random.default_rng(0)
    status = {f: rng.integers(0, 3, size=(snap.R, snap.m) if f in ("calc_thr", "used") else snap.m) for f in STATUS}
    s.status = {f: np.ascontiguousarray(v[..., idx]) for f, v in status.items()}
    res = rng.integers(0, 1000, size=(snap.R, snap.m))
    s.reserved = np.ascontiguousarray(res[:, idx])
    s.reserved_present = np.ones(len(idx), np.uint32)
    s.reserved_cnt = np.ones(len(idx), np.int64)
    return s.normalize()


def timed(reset, fa, fb, n=50, warm=5):
    """Medians (us) of two calls timed alternately, each after an untimed reset."""
    ta, tb = [], []
    for i in range(warm + n):
        for f, ts in ((fa, ta), (fb, tb)):
            reset()
            t0 = time.perf_counter()
            f()
            dt = time.perf_counter() - t0
            if i >= warm:
                ts.append(dt)
    return round(float(np.median(ta)) * 1e6, 1), round(float(np.median(tb)) * 1e6, 1)


def engine_calls():
    import kube_throttler_b200 as kt
    from kube_throttler_b200 import synth

    out = {}
    for name, cfg in (("C2_1k", "C2"), ("C5_10k", "C5")):
        snap = synth.generate(cfg, n=100_000, p=10_000, n_ns=500, cluster_frac=0.4).normalize()
        m = snap.m
        e = kt.Engine(snap.R, snap.L, snap.LN)
        e.upload_snapshot(snap)
        row = {"m": m, "n_ns": snap.n_ns}
        rng = np.random.default_rng(1)
        # creation into a full group: columns [0, m-1) resident, column m-1 created at position p
        p = m // 2
        base = layout(snap, np.arange(m - 1))
        order = np.concatenate([np.arange(p), [m - 1], np.arange(p, m - 1)])
        grown = layout(snap, order)
        src = np.concatenate([np.arange(p), [-1], np.arange(p, m - 1)]).astype(np.int32)
        t = np.array([p], np.int32)
        cols = columns_of(grown, t)
        st = {f: np.ascontiguousarray(v[..., t]) for f, v in grown.status.items()}
        cases = {}

        def create():
            e.move_throttle_columns(src)
            e.update_selector_rows(t, cols)
            e.update_threshold_rows(t, cols)
            e.update_status_rows(t, st)
            e.update_reserved_rows(t, grown.reserved[:, t], grown.reserved_present[t], grown.reserved_cnt[t])

        cases["create_full_group"] = (base, grown, create)
        for frac in (0.1, 0.5):
            holes = np.sort(rng.choice(m, size=int(m * frac), replace=False))
            keep = np.setdiff1d(np.arange(m), holes).astype(np.int32)
            cases[f"compact_{int(frac * 100)}pct"] = (layout(snap, np.arange(m), holes), layout(snap, keep),
                                                       lambda keep=keep: e.move_throttle_columns(keep))
        for case, (start, end, move) in cases.items():
            def reset(start=start):
                e.upload_throttles(start)
                e.upload_status(start)
                e.set_reserved(start)
                e.evaluate(snap.now)

            def whole(end=end):
                e.upload_throttles(end)
                e.upload_status(end)
                e.set_reserved(end)

            row[f"move_{case}_us"], row[f"whole_{case}_us"] = timed(reset, move, whole)
        e.close()
        out[name] = row
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card(), "engine": engine_calls(), "card_after": card()}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
