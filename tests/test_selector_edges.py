"""The selector match at its edges, against the columnar oracle (oracle/ko_columnar.h, requirement by requirement).

synth.generate draws a narrow family of selectors: distinct keys per term, no empty selectors, no flagged terms, tidy label
rows with their gaps last, small ids, L <= 16 and at most six required keys.  `edge_world` here builds snapshots outside that
family: a key twice in a term (every pairing of operators), Everything podSelectors and zero-term throttles, only-negative
terms, In / NotIn sets of up to 300 values at both sides of the direct value table's span rule, terms needing exactly L keys,
L + 1 keys and 63 / 64 / 65 keys, ids at their edges (key 0, key 65535, keys past the direct key table, values next to 2^32),
term and throttle flags, namespaces out of range, and label rows with their labels in random slots.

Without a GPU the compiled tables (kt_debug_compile_tables, walked in numpy by test_tables_cpu.match_bitmap) must give the
oracle's relation; on the GPU every fused and chained kernel variant, every upload format, row deltas, table re-uploads, the
column lists and the queue admission must give the oracle's bits."""
import copy
import dataclasses
import functools
import zlib

import numpy as np
import pytest

from kube_throttler_b200 import abi, synth
from test_tables_cpu import compile_tables, match_bitmap

IN, NOTIN, EXISTS, DNE = abi.OP_IN, abi.OP_NOTIN, abi.OP_EXISTS, abi.OP_DOESNOTEXIST
THROTTLE, CLUSTER = abi.KIND_THROTTLE, abi.KIND_CLUSTERTHROTTLE
NS_KEYS = (200, 201, 202)
NS_KEY_NOBODY = 203  # a namespace label key no namespace carries
U32 = 0xFFFFFFFF

# The pairings of two requirements on one key inside one term (matchLabels k=v is In{v}).
DUP_CASES = ("in_in_overlap", "in_in_disjoint", "in_notin", "exists_in", "notin_notin", "notin_dne", "exists_dne", "match_labels_expr")


# ---- the edge-world generator ---------------------------------------------------------------------------------------------
def _key_ids(rng, ids, K):
    """(mentioned key ids [K], unmentioned key ids) for an id regime."""
    if ids == "small":      # everything fits the compact upload's 12 + 20 bit split
        ment = np.concatenate([[0], np.sort(rng.choice(np.arange(1, 3000), K - 1, replace=False))])
        top = int(ment[-1])
        unm = [top + 1, top + 7, 4095]
    elif ids in ("direct", "key65535"):
        ment = np.concatenate([[0], np.sort(rng.choice(np.arange(1, 60000), K - 1, replace=False))])
        if ids == "key65535":
            ment[-1] = 65535  # a 65536-entry direct key table
        top = int(ment[-1])
        unm = [top + 1, top + 1000, 1 << 20, 0xFFFFFFFE]  # unmentioned keys past the direct key table
    else:                   # "hashed": a key >= 65536, so every label goes through the hash
        spread = np.unique(rng.integers(70000, U32 - 1, size=2 * K, dtype=np.int64))
        ment = np.concatenate([[0, 65536], np.sort(rng.choice(spread, K - 2, replace=False))])
        unm = [65535, 65537, 0xFFFFFFFE]
    ment = [int(k) for k in ment]
    between = [k + 1 for k in ment[:8] if k + 1 not in ment]  # unmentioned keys among the mentioned ones
    return ment, sorted(set(unm + between) - set(ment))


def _value_set(rng, regime, c, small):
    """The mentioned value ids of one key: dense, at the top of the 32-bit range, spread out, or c values whose span is just
    inside (4c + 64) or just outside (4c + 65) the span the direct value table accepts."""
    vmax = (1 << 20) - 1 if small else 0xFFFFFFFE
    if regime == "dense":
        lo = 0 if rng.random() < 0.5 else int(rng.integers(0, 1000))
        return list(range(lo, lo + c))
    if regime == "top" and not small:
        return list(range(0xFFFFFFFE - c + 1, 0xFFFFFFFF))
    if regime in ("span_in", "span_out"):
        span = 4 * c + (64 if regime == "span_in" else 65)
        lo = int(rng.integers(0, vmax - span))
        mid = rng.choice(np.arange(1, span - 1), c - 2, replace=False)
        return sorted([lo, lo + span - 1] + [lo + int(x) for x in mid])
    return sorted(set(int(v) for v in rng.integers(0, vmax, size=c, dtype=np.int64)))


def _holds(op, vals, v):
    """A requirement on a key, for a pod whose value for it is v (None: the key is absent)."""
    if op == IN:
        return v is not None and v in vals
    if op == NOTIN:
        return v is None or v not in vals
    if op == EXISTS:
        return v is not None
    return v is None


def _label(k, v):
    x = (int(k) << 32) | int(v)
    return x - (1 << 64) if x >= 1 << 63 else x


def edge_world(seed, *, m, n, p, L, R=2, LN=3, n_ns=6, terms=1, q_max=3, ids="direct", cluster=0.3, dup=True, everything=True,
               negative=True, big_sets=True, need_limit=False, huge_need=True, flags=True, ns_edges=True, wide_ns=False, specials=True):
    """A seeded Snapshot outside synth.generate's family.  Knobs switch the edge cases on; meta["cases"] names the ones the
    snapshot holds, meta["terms"] the selectors per throttle as [(pod reqs, ns reqs, term flag)], meta["ids"] the key ids."""
    rng = np.random.default_rng(seed)
    small = ids == "small"
    cases = set()
    K = max(14, L + 2 if need_limit else 0, 66 if huge_need else 0)
    ment, unment = _key_ids(rng, ids, K)
    if 0 in ment:
        cases.add("key0")
    cases.add({"small": "direct_keys", "direct": "direct_keys", "key65535": "key65535", "hashed": "hashed_keys"}[ids])
    regimes = ("dense", "span_in", "span_out", "top", "sparse")
    vsets = {}
    for i, k in enumerate(ment):
        reg = regimes[i % len(regimes)]
        big = big_sets and i % 7 == 1
        c = int(rng.integers(150, 301)) if big else int(rng.integers(2, 9))
        vsets[k] = _value_set(rng, "dense" if big and reg in ("top", "sparse") else reg, c, small)
    if ment[0] == 0 and vsets[0][0] != 0:
        vsets[0] = [0] + vsets[0][1:]
    cases.add("value0")
    hot = ment[:9] + ment[-1:]  # the keys ordinary terms draw from (the largest one included): few, so keys repeat within a term
    vmax = (1 << 20) - 1 if small else U32

    def other_values(k):
        vs = vsets[k]
        out = [(vs[0] - 1) & U32, (vs[-1] + 1) & U32, 0, 0xFFFFFFFE, U32, int(rng.integers(0, vmax))]
        gap = sorted(set(range(vs[0], min(vs[-1], vs[0] + 400))) - set(vs))
        if gap:
            out.append(gap[int(rng.integers(len(gap)))])
        return [v for v in out if v <= vmax and v not in vs]

    def values(k, lo, hi):
        vs = vsets[k]
        return sorted(set(int(v) for v in rng.choice(vs, min(len(vs), int(rng.integers(lo, hi + 1))), replace=False)))

    def req(k, op, big=False):
        if op in (EXISTS, DNE):
            return (k, op, [])
        if big and len(vsets[k]) > 3:
            return (k, op, list(vsets[k]) if rng.random() < 0.5 else values(k, 1, 300))
        return (k, op, values(k, 1, 3))

    def ordinary_term():
        q = int(rng.integers(0 if everything and rng.random() < 0.1 else 1, q_max + 1))
        keys = [int(k) for k in rng.choice(hot, q, replace=dup)]
        return [req(k, int(rng.choice([IN, NOTIN, EXISTS, DNE], p=[0.5, 0.2, 0.15, 0.15])), big_sets and rng.random() < 0.1) for k in keys]

    def ns_reqs(kind):
        if kind != CLUSTER or (wide_ns and rng.random() < 0.85):
            return []
        out = []
        for _ in range(int(rng.integers(0, 3))):
            k = int(rng.choice(NS_KEYS + (NS_KEY_NOBODY,)))
            op = int(rng.integers(0, 4))
            out.append((k, op, [] if op in (EXISTS, DNE) else sorted(set(int(v) for v in rng.integers(0, 3, size=int(rng.integers(1, 3)))))))
            cases.add(f"ns_op{op}")
        return out

    # ---- dedicated throttles for the cases that must be there: (case, kind or None, [pod reqs per term], pod-invalid term) ----
    spec = []
    if specials:
        a, b = int(ment[1]), int(ment[2])
        if dup:
            va = vsets[a]
            spec += [("in_in_overlap", None, [[(a, IN, va[:2]), (a, IN, va[1:3])]]),
                     ("in_in_disjoint", None, [[(a, IN, va[:1]), (a, IN, va[1:2])]]),
                     ("in_notin", None, [[(a, IN, va[:3]), (a, NOTIN, va[1:2])]]),
                     ("exists_in", None, [[(a, EXISTS, []), (a, IN, va[:2]), (b, EXISTS, [])]]),
                     ("notin_notin", None, [[(a, NOTIN, va[:1]), (a, NOTIN, va[1:2])]]),
                     ("notin_dne", None, [[(a, NOTIN, va[:1]), (a, DNE, [])]]),
                     ("exists_dne", None, [[(a, EXISTS, []), (a, DNE, [])]]),
                     ("match_labels_expr", None, [[(a, IN, va[:1]), (a, NOTIN, va[2:3]), (b, IN, vsets[b][:1])]])]
        if everything:
            spec += [("everything_throttle", THROTTLE, [[]]), ("everything_cluster", CLUSTER, [[]]), ("zero_terms", None, [])]
        if negative:
            spec += [("negative_only", THROTTLE, [[(a, NOTIN, vsets[a][:2]), (b, DNE, [])]])]
        if big_sets:
            span_keys = [k for i, k in enumerate(ment) if len(vsets[k]) > 100]
            for k in span_keys[:2]:
                spec += [("big_set", None, [[(k, IN, list(vsets[k]))]]), ("big_set", None, [[(k, NOTIN, list(vsets[k]))]])]
        if need_limit:
            pos = lambda c: [(k, IN, vsets[k][:2]) if i % 2 else (k, EXISTS, []) for i, k in enumerate(ment[:c])]
            spec += [("need_L", THROTTLE, [pos(L)]), ("need_L_plus_1", THROTTLE, [pos(L + 1)])]
        if huge_need:
            spec += [(f"need_{c}", None, [[(k, EXISTS, []) for k in ment[:c]]]) for c in (63, 64, 65)]
        if flags:
            where = {1: ["only"], 2: ["first", "last"]}.get(terms, ["first", "middle", "last"])
            for w in where:
                T = max(1, min(terms, 3))
                spec.append((f"pod_invalid_{w}", None, [ordinary_term() for _ in range(T)], {"only": 0, "first": 0, "middle": 1, "last": T - 1}[w]))
    if len(spec) + 1 > m:
        spec = []

    # ---- throttles ----
    n_cluster = int(round(m * cluster))
    kind = np.array([THROTTLE] * (m - n_cluster) + [CLUSTER] * n_cluster, np.uint8)
    rng.shuffle(kind)
    for i, s in enumerate(spec):
        if s[1] is not None:
            kind[i] = s[1]
    hi_ns = n_ns + 2 if ns_edges else n_ns
    thr_ns = np.where(kind == THROTTLE, rng.integers(0, hi_ns, size=m), -1).astype(np.int32)
    for i, s in enumerate(spec):
        if kind[i] == THROTTLE:
            thr_ns[i] = i % n_ns  # the dedicated throttles sit in real namespaces
    if ns_edges and (thr_ns >= n_ns).any():
        cases.add("throttle_ns_out_of_range")
    thr_flags = np.full(m, abi.THR_RESPONSIBLE, np.uint8)
    per_thr, at = [], {}
    for t in range(m):
        if t < len(spec):
            s = spec[t]
            cases.add(s[0])
            at.setdefault(s[0], t)
            tl = [(pr, ns_reqs(kind[t]), 0) for pr in s[2]]
            if len(s) > 3:
                tl[s[3]] = (tl[s[3]][0], tl[s[3]][1], abi.TERM_POD_INVALID)
        else:
            T = terms if t == m - 1 else int(rng.integers(0 if everything and rng.random() < 0.05 else 1, terms + 1))
            tl = [(ordinary_term(), ns_reqs(kind[t]), 0) for _ in range(T)]
            if flags:
                for j in range(T):
                    if kind[t] == CLUSTER and rng.random() < 0.08:
                        tl[j] = (tl[j][0], tl[j][1], abi.TERM_NS_INVALID)
                        cases.add("ns_invalid")
                if T and rng.random() < 0.08:
                    j = int(rng.integers(T))
                    tl[j] = (tl[j][0], tl[j][1], tl[j][2] | abi.TERM_POD_INVALID)
                u = rng.random()
                if u < 0.04:
                    thr_flags[t] |= abi.THR_SELECTOR_ERROR
                    cases.add("selector_error")
                elif u < 0.08:
                    thr_flags[t] = 0
                    cases.add("not_responsible")
        per_thr.append(tl)
    term_off = np.concatenate([[0], np.cumsum([len(tl) for tl in per_thr])]).astype(np.int32)
    flat = [x for tl in per_thr for x in tl]
    sel = synth.build_selector_csr(term_off, [x[0] for x in flat], [x[1] for x in flat], [x[2] for x in flat])

    # ---- namespaces: some lack keys, the last one has no labels at all ----
    ns_labels = np.full((LN, n_ns), abi.LABEL_EMPTY, np.int64)
    for ns in range(n_ns - 1):
        keys = [k for k in NS_KEYS if ns == 0 or rng.random() < 0.7][:LN]
        slots = rng.permutation(LN)[: len(keys)]
        for s, k in zip(slots, keys):
            ns_labels[s, ns] = _label(k, int(rng.integers(0, 3)))
    cases.add("namespace_without_labels")

    # ---- pods ----
    def pod_rows(count, running):
        lab = np.full((L, count), abi.LABEL_EMPTY, np.int64)
        ns = rng.integers(0, n_ns + 3 if ns_edges else n_ns, size=count).astype(np.int32)
        for i in range(count):
            labels = {}
            t = int(rng.integers(len(spec) if spec and rng.random() < 0.4 else m))  # the dedicated throttles more often
            if rng.random() < 0.45 and per_thr[t]:  # planted: a pod meant to satisfy one term of throttle t
                pr = per_thr[t][int(rng.integers(len(per_thr[t])))][0]
                by_key = {}
                for k, op, vals in pr:
                    by_key.setdefault(k, []).append((op, vals))
                for k, rq in by_key.items():
                    named = [int(v) for _, vals in rq for v in vals]
                    choices = ([None] if rng.random() < 0.5 else []) + [int(v) for v in rng.permutation(named)[:6]] + \
                              [int(v) for v in rng.permutation(vsets[k])[:6]] + other_values(k) + [None]
                    v = next((v for v in choices if all(_holds(op, vals, v) for op, vals in rq)), "no")
                    if v not in (None, "no"):
                        labels[k] = v
                if len(labels) > L:
                    labels = dict(list(labels.items())[:L])
                if labels and rng.random() < 0.3:  # a near miss
                    k = list(labels)[int(rng.integers(len(labels)))]
                    if rng.random() < 0.5:
                        del labels[k]
                    else:
                        labels[k] = other_values(k)[int(rng.integers(len(other_values(k))))]
                if kind[t] == THROTTLE:
                    ns[i] = thr_ns[t]
                elif rng.random() < 0.9:
                    ns[i] = int(rng.integers(0, n_ns))
            elif rng.random() > 0.1:
                for _ in range(int(rng.integers(0, L + 1))):
                    u = rng.random()
                    if u < 0.75:
                        k = int(rng.choice(hot if rng.random() < 0.7 else ment))
                        labels[k] = int(rng.choice(vsets[k])) if rng.random() < 0.6 else other_values(k)[int(rng.integers(len(other_values(k))))]
                    else:
                        labels[int(rng.choice(unment))] = int(rng.integers(0, vmax + 1))
                labels = dict(list(labels.items())[:L])
            # free slots around the labels: random positions, or (L > 8) the last chunk of eight only
            room = L - 8 * ((L - 1) // 8)
            if L > 8 and len(labels) <= room and rng.random() < 0.2:
                slots = (L - room) + rng.permutation(room)[: len(labels)]
                if labels:
                    cases.add("labels_in_last_chunk_only")
            else:
                slots = rng.permutation(L)[: len(labels)]
            for s, (k, v) in zip(slots, labels.items()):
                lab[s, i] = _label(k, v)
        empty = lab == abi.LABEL_EMPTY
        if (empty.all(axis=0)).any():
            cases.add("label_less_row")
        if (empty[0] & ~empty.all(axis=0)).any():
            cases.add("leading_empty_slot")
        if ns_edges and (ns >= n_ns).any():
            cases.add("pod_ns_out_of_range")
        req = rng.integers(1, 5, size=(R, count)).astype(np.int64)
        present = np.ones(count, np.uint32)
        for r in range(1, R):
            present |= np.where(rng.random(count) < 0.8, 1 << r, 0).astype(np.uint32)
        req *= ((present[None, :] >> np.arange(R, dtype=np.uint32)[:, None]) & 1).astype(np.int64)
        if running:
            u = rng.random(count)
            fl = np.full(count, 7, np.uint32)
            fl = np.where(u < 0.05, 3, np.where(u < 0.08, 6, np.where(u < 0.10, 5, fl))).astype(np.uint32)
        else:
            fl = np.full(count, abi.POD_SCHEDULER_MATCH | abi.POD_NOT_FINISHED, np.uint32)
        return abi.PodCols(lab, req, present, fl, ns)

    running, pending = pod_rows(n, True), pod_rows(p, False)
    for pods in (running, pending):
        v = pods.labels & U32
        mentioned = np.isin((pods.labels >> 32) & U32, ment) & (pods.labels != abi.LABEL_EMPTY)
        if (mentioned & (v == U32)).any():
            cases.add("pod_value_ffffffff")
        if (mentioned & (v == 0xFFFFFFFE)).any():
            cases.add("pod_value_fffffffe")
        if (~mentioned & (pods.labels != abi.LABEL_EMPTY) & (((pods.labels >> 32) & U32) > max(ment))).any():
            cases.add("unmentioned_key_past_keydir")

    z = np.zeros
    snap = abi.Snapshot(R=R, L=L, LN=LN, running=running, pending=pending, ns_labels=ns_labels, kind=kind, thr_ns=thr_ns, thr_flags=thr_flags,
                        thr=z((R, m), np.int64), thr_present=z(m, np.uint32), thr_cnt=z(m, np.int64), ovr_off=z(m + 1, np.int32),
                        ovr_begin=z(0, np.int64), ovr_end=z(0, np.int64), ovr_flags=z(0, np.uint8), ovr_thr=z((R, 0), np.int64),
                        ovr_present=z(0, np.uint32), ovr_cnt=z(0, np.int64), now=synth.NOW_2026, **sel,
                        meta=dict(cases=cases, terms=per_thr, ids=ment, special_at=at, seed=seed))
    snap.normalize()

    # ---- thresholds from the matched sums: below them, about one pod above, far above, or below any one pod's request ----
    used, _, ucnt = synth.true_used_numpy(snap)
    regime = rng.integers(0, 4, size=m)
    thr = np.select([regime == 0, regime == 1, regime == 2], [used // 2, used + 2, used + 1000], 1)
    present = np.ones(m, np.uint32)
    for r in range(1, R):
        present |= np.where(rng.random(m) < 0.5, 1 << r, 0).astype(np.uint32)
    has_cnt = rng.random(m) < 0.3
    snap.thr = (thr * ((present[None, :] >> np.arange(R, dtype=np.uint32)[:, None]) & 1)).astype(np.int64)
    snap.thr_present = np.where(has_cnt, present | abi.COUNT_BIT, present).astype(np.uint32)
    snap.thr_cnt = np.where(has_cnt, np.select([regime == 0, regime == 1, regime == 2], [ucnt // 2, ucnt + 1, ucnt + 100], 0), 0).astype(np.int64)
    return snap.normalize()


def with_throttles(snap, per_thr, kind, thr_ns, thr_flags):
    """The snapshot with another throttle table (selectors per throttle as in meta["terms"]); thresholds of 1 on resource 0."""
    s = copy.copy(snap)
    m = len(per_thr)
    term_off = np.concatenate([[0], np.cumsum([len(tl) for tl in per_thr])]).astype(np.int32)
    flat = [x for tl in per_thr for x in tl]
    for f, v in synth.build_selector_csr(term_off, [x[0] for x in flat], [x[1] for x in flat], [x[2] for x in flat]).items():
        setattr(s, f, v)
    s.kind, s.thr_ns, s.thr_flags = np.asarray(kind, np.uint8), np.asarray(thr_ns, np.int32), np.asarray(thr_flags, np.uint8)
    s.thr = np.zeros((s.R, m), np.int64)
    s.thr[0] = 1
    s.thr_present, s.thr_cnt, s.ovr_off = np.ones(m, np.uint32), np.zeros(m, np.int64), np.zeros(m + 1, np.int32)
    s.status = s.reserved = s.reserved_present = s.reserved_cnt = None
    s.meta = dict(snap.meta, terms=per_thr)
    return s.normalize()


# ---- the worlds -----------------------------------------------------------------------------------------------------------
# One world per dispatch_pass variant, with the (tile, tpc, b, rt) it must reach (rt 0: the general family) and its term planes
# per table entry.  256-row tiles need a namespace whose word list is long (ClusterThrottles whose namespaceSelectors admit most
# namespaces: wide_ns); B = 2 needs every term to need at most 3 keys, so the need-at-L worlds are the L = 3 one and the B = 6 ones.
VARIANTS = [
    ("fast128_t1_r4", dict(seed=1, m=97, n=2000, p=600, L=8, R=2, terms=1, ids="small"), (128, 1, 2, 4), 1),
    ("fast128_t1_r8", dict(seed=2, m=65, n=2000, p=600, L=8, R=6, terms=1, ids="key65535"), (128, 1, 2, 8), 1),
    ("fast128_t2_r4", dict(seed=3, m=64, n=2000, p=600, L=3, R=4, terms=2, need_limit=True), (128, 2, 2, 4), 2),
    ("fast128_t2_r8", dict(seed=4, m=63, n=2000, p=600, L=8, R=8, terms=2, ids="hashed"), (128, 2, 2, 8), 2),
    ("fast256_t1_r4", dict(seed=5, m=260, n=3000, p=700, L=8, R=3, terms=1, cluster=0.85, wide_ns=True), (256, 1, 2, 4), 1),
    ("fast256_t1_r8", dict(seed=6, m=257, n=3000, p=700, L=5, R=5, terms=1, cluster=0.85, wide_ns=True, ids="key65535"), (256, 1, 2, 8), 1),
    ("fast256_t2_r4", dict(seed=7, m=288, n=3000, p=700, L=8, R=4, terms=4, cluster=0.85, wide_ns=True, ids="hashed"), (256, 2, 2, 4), 4),
    ("fast256_t2_r8", dict(seed=8, m=270, n=3000, p=700, L=8, R=7, terms=2, cluster=0.85, wide_ns=True, ids="small"), (256, 2, 2, 8), 2),
    ("general_t1_b2", dict(seed=9, m=33, n=2000, p=600, L=12, R=2, terms=1, ids="small"), (128, 1, 2, 0), 1),
    ("general_t1_b6", dict(seed=10, m=97, n=2000, p=600, L=8, R=3, terms=1, q_max=6, need_limit=True), (128, 1, 6, 0), 1),
    ("general_t2_b2", dict(seed=11, m=96, n=2000, p=600, L=20, R=2, terms=4, ids="key65535"), (128, 2, 2, 0), 4),
    ("general_t2_b6", dict(seed=12, m=120, n=2000, p=600, L=32, R=4, terms=3, q_max=6, need_limit=True, ids="hashed"), (128, 2, 6, 0), 4),
]
# beyond one world per variant: L = 32 with direct keys, and the ABI's limits on both R and L
EXTRA = [
    ("limits_l32_direct", dict(seed=13, m=100, n=2000, p=600, L=32, R=8, terms=2, q_max=6, need_limit=True, ids="key65535"), (128, 2, 6, 0), 2),
    ("limits_r31_l32", dict(seed=14, m=70, n=1500, p=500, L=32, R=31, terms=1, need_limit=True, ids="direct"), (128, 1, 6, 0), 1),
]
WORLDS = {name: (kw, v, tppad) for name, kw, v, tppad in VARIANTS + EXTRA}
SHAPE_M = (1, 31, 32, 33, 63, 64, 65, 97)


@functools.lru_cache(maxsize=None)
def _world(name, small=False):
    kw = dict(WORLDS[name][0])
    if small:
        kw.update(n=300, p=250)
    return edge_world(**kw)


def world(name, small=False):
    return copy.deepcopy(_world(name, small))


@functools.lru_cache(maxsize=None)
def _shape_world(m):
    return edge_world(100 + m, m=m, n=300, p=200, L=9, R=3, terms=min(4, 1 + m % 4), q_max=4)


def n_need(pod_reqs):
    return len({k for k, op, _ in pod_reqs if op in (IN, EXISTS)})


# ---- CPU half -------------------------------------------------------------------------------------------------------------
CPU_WORLDS = [(name, True) for name in WORLDS] + [(f"m{m}", False) for m in SHAPE_M]
_cpu_cases = set()
_cpu_ran = set()


def cpu_world(name, small):
    return copy.deepcopy(_world(name, True) if small else _shape_world(int(name[1:])))


@pytest.mark.parametrize("name,small", CPU_WORLDS, ids=[c[0] for c in CPU_WORLDS])
def test_compiled_tables_on_edge_worlds(kt, oracle, name, small):
    """The relation the compiled tables give equals the oracle's for both pod kinds, and the tables hold what the kernels
    rely on: unsatisfiable terms switched off, the direct tables only where the ids allow them, B = 6 exactly when some
    satisfiable term needs more than three keys, nothing of a zero-term throttle in any plane."""
    snap = cpu_world(name, small)
    t = compile_tables(kt, snap)
    want = oracle.columnar_evaluate(snap, words_per_row=t["Wp"])
    np.testing.assert_array_equal(match_bitmap(t, snap.running, True), want.run_bitmap)
    np.testing.assert_array_equal(match_bitmap(t, snap.pending, False), want.pend_bitmap)
    if small:
        assert t["TPpad"] == WORLDS[name][2]

    L, per_thr, ment = snap.L, snap.meta["terms"], snap.meta["ids"]
    needs = [n_need(pr) for tl in per_thr for pr, _, _ in tl]
    assert t["B"] == (6 if any(3 < d <= L for d in needs) else 2)
    for th, tl in enumerate(per_thr):
        w, bit = th >> 5, np.uint32(1 << (th & 31))
        if not tl:  # a zero-term throttle
            assert not (t["nsmask"][:, w, :] & bit).any() and not (t["need"][w] & bit).any()
        for s, (pr, _, _) in enumerate(tl):
            if n_need(pr) > L:  # can never match: switched off, needs nothing (so no counter can wrap onto it)
                assert not (t["nsmask"][:, w, s] & bit).any(), (th, s)
                assert not (t["need"][w, s] & bit).any(), (th, s)
    mentioned = sorted(set(int(k) for k in snap.req_key[: snap.ns_req_off[0]]))
    if not mentioned:
        assert t["n_keydir"] == 0
    elif mentioned[-1] >= 1 << 16:
        assert t["n_keydir"] == 0  # a key past the direct table: every label is hashed
    else:
        assert t["n_keydir"] == mentioned[-1] + 1
        if "key65535" in snap.meta["cases"]:
            assert t["n_keydir"] == 1 << 16
        for k in mentioned:  # the direct value table takes a key's values when their span is at most 4 per value + 64
            vals = set()
            for q in np.nonzero(snap.req_key[: snap.ns_req_off[0]] == k)[0]:
                vals |= set(int(v) for v in snap.req_vals[snap.req_val_off[q]:snap.req_val_off[q + 1]])
            if vals:
                span = max(vals) - min(vals) + 1
                assert (t["keydir"][k, 3] == U32) == (span > 4 * len(vals) + 64), (k, span, len(vals))
                _cpu_cases.add("span_hashed" if span > 4 * len(vals) + 64 else "span_direct")
                if span > 4 * len(vals) + 64 and span <= 4 * len(vals) + 65:
                    _cpu_cases.add("span_just_outside")
                if span == 4 * len(vals) + 64:
                    _cpu_cases.add("span_just_inside")
    # the dedicated throttles do what their case is about, on the oracle's side too
    at = snap.meta["special_at"]
    run = want.match_matrix("running", snap.m)
    if "need_L" in at and run[:, at["need_L"]].any():
        _cpu_cases.add("need_L_matched")
    if "need_L_plus_1" in at:
        assert not run[:, at["need_L_plus_1"]].any()
    if "negative_only" in at:
        th = at["negative_only"]
        bare = (snap.running.labels == abi.LABEL_EMPTY).all(axis=0) & (snap.running.ns_id == snap.thr_ns[th]) & ((snap.running.flags & 3) == 3)
        assert (run[bare, th] == 1).all(), "an only-negative term must match the label-less pods of its namespace"
        if bare.any():
            _cpu_cases.add("negative_only_matched_label_less")
    _cpu_cases.update(snap.meta["cases"])
    _cpu_ran.add(name)


ALL_CASES = set(DUP_CASES) | {
    "everything_throttle", "everything_cluster", "zero_terms", "negative_only", "negative_only_matched_label_less", "big_set",
    "need_L", "need_L_plus_1", "need_L_matched", "need_63", "need_64", "need_65", "key0", "value0", "key65535", "hashed_keys",
    "direct_keys", "pod_value_ffffffff", "pod_value_fffffffe", "unmentioned_key_past_keydir", "span_direct", "span_hashed",
    "span_just_inside", "span_just_outside", "pod_invalid_only", "pod_invalid_first", "pod_invalid_middle", "pod_invalid_last",
    "ns_invalid", "selector_error", "not_responsible", "ns_op0", "ns_op1", "ns_op2", "ns_op3", "namespace_without_labels",
    "throttle_ns_out_of_range", "pod_ns_out_of_range", "label_less_row", "leading_empty_slot", "labels_in_last_chunk_only"}


def test_cpu_worlds_cover_every_case():
    """Runs after the worlds above: together they hold every edge case the generator knows."""
    if _cpu_ran != {c[0] for c in CPU_WORLDS}:
        pytest.skip("the CPU worlds did not run in full")
    assert ALL_CASES <= _cpu_cases, sorted(ALL_CASES - _cpu_cases)


def test_generator_is_deterministic():
    a, b = edge_world(5, m=40, n=50, p=30, L=12), edge_world(5, m=40, n=50, p=30, L=12)
    for f in ("req_key", "req_vals", "term_flags", "thr", "thr_cnt"):
        np.testing.assert_array_equal(getattr(a, f), getattr(b, f))
    np.testing.assert_array_equal(a.running.labels, b.running.labels)


# ---- GPU half -------------------------------------------------------------------------------------------------------------
FRESH, GIVEN = abi.EVAL_FRESH_STATUS, abi.EVAL_GIVEN_STATUS
REC_ONLY = abi.EVAL_FRESH_STATUS | abi.EVAL_SKIP_CHECK
CHK_ONLY = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE
RUN, PEND = abi.PODS_RUNNING, abi.PODS_PENDING
_fused = set()     # (tile, tpc, b, rt) the fused plans ran
_chained = set()   # ("reconcile", (tpc, b, rt)) / ("check", (tpc, b, register rows))
_worlds_ran = set()  # (name, L, hashed) of the worlds whose fused plans ran


def _engine(kt, snap):
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    return eng


def _oracle(oracle, snap, flags=FRESH, W=None):
    return oracle.columnar_evaluate(snap, flags, words_per_row=W)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WORLDS))
def test_fused_plans(kt, oracle, name):
    """The world reaches its dispatch_pass variant; the automatic fused pass and forced plans (both residencies x both decide
    modes, on the device's grid and on one CTA) give the oracle's bits."""
    from test_pass_plans import DECIDES, THREADS, automatic, forced, variant
    from test_gpu_parity import assert_same

    _, want_variant, tppad = WORLDS[name]
    snap = world(name)
    t = compile_tables(kt, snap)
    assert t["TPpad"] == tppad
    eng = _engine(kt, snap)
    got, plan = automatic(eng, snap)
    want = _oracle(oracle, snap, W=got.words_per_row)
    assert_same(snap, got, want)
    assert variant(plan) == want_variant, (variant(plan), want_variant)
    codes = set(np.unique(want.code_matrix(snap.m)[want.match_matrix("pending", snap.m) == 1]).tolist())
    assert codes == {0, 1, 2, 3}, codes
    for threads in THREADS:
        for decide in DECIDES:
            for cap in (0, 1):
                got, plan = forced(eng, snap, threads, decide, cap)
                assert variant(plan) == want_variant
                assert_same(snap, got, want)
    eng.close()
    _fused.add(want_variant)
    _worlds_ran.add((name, snap.L, t["n_keydir"] == 0))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WORLDS))
def test_chained_passes(kt, oracle, name):
    """The chained kernels on the same worlds: a whole pass with timing on (k_reconcile, k_finalize, k_check), reconcile-only,
    and check-only against an observed status."""
    from test_gpu_parity import assert_same
    from test_partial_passes import check_variant, observed_status, reconcile_variant, run_pass, with_pending_of

    snap = world(name)
    eng = _engine(kt, snap)
    prev = run_pass(eng, snap, FRESH, 1)
    plan = eng.pass_plan()
    W = prev.words_per_row
    assert_same(snap, prev, _oracle(oracle, snap, W=W))
    got = run_pass(eng, snap, FRESH, 3, timing=True)
    fresh = _oracle(oracle, snap, W=W)
    assert_same(snap, got, fresh)
    got = run_pass(eng, snap, REC_ONLY, 2)
    assert_same(snap, got, with_pending_of(_oracle(oracle, snap, REC_ONLY, W), prev))
    _chained.add(("reconcile", reconcile_variant(plan)))
    snap.status = observed_status(fresh, snap, np.random.default_rng(zlib.crc32(name.encode())))
    snap.normalize()
    eng.upload_status(snap)
    got = run_pass(eng, snap, CHK_ONLY, 2)
    assert_same(snap, got, _oracle(oracle, snap, CHK_ONLY, W), check_reconcile=False)
    _chained.add(("check", check_variant(plan, snap.L)))
    eng.close()


def extreme_packed(pods):
    """The packed rows with their pair dictionary padded to its 65535 entries and the used pairs moved to its end: the
    indices k_unpack_packed reads are the largest the format allows (65534 included), next to the 0xFFFF empty slot."""
    pk = abi.packed_pods(pods)
    used = pk.pairs.shape[0]
    top = 65535 - used
    pairs = np.empty(65535, np.int64)
    pairs[:top] = _label(0x7FFFFFF0, 0) + np.arange(top)  # never referenced
    pairs[top:] = pk.pairs
    idx = pk.labels16.astype(np.int64)
    lab16 = np.where(idx == 0xFFFF, 0xFFFF, idx + top).astype(np.uint16)
    out = dataclasses.replace(pk, pairs=pairs, labels16=np.ascontiguousarray(lab16))
    np.testing.assert_array_equal(out.unpack().labels, pods.labels)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WORLDS))
def test_upload_formats(kt, oracle, name):
    """The same rows through the packed upload (extreme pair indices, 0xFFFF gaps inside rows) and, where the ids fit its
    12 + 20 bit split, the compact one; where they do not, abi.compact_pods refuses them."""
    from test_gpu_parity import assert_same
    from test_pass_plans import automatic

    snap = world(name)
    eng = _engine(kt, snap)
    got, _ = automatic(eng, snap)
    want = _oracle(oracle, snap, W=got.words_per_row)
    assert_same(snap, got, want)
    if snap.R > 28:  # presence (R bits), flags and a namespace id do not fit the packed meta word
        with pytest.raises(ValueError):
            abi.packed_pods(snap.running)
    else:
        for kind, pods in ((RUN, snap.running), (PEND, snap.pending)):
            empty = pods.labels == abi.LABEL_EMPTY
            assert (empty[:-1] & ~empty[1:]).any(), "no row has a gap before a label"
            eng.upload_pods_packed(kind, extreme_packed(pods))
        got, _ = automatic(eng, snap)
        assert_same(snap, got, want)
        if "key65535" in snap.meta["cases"]:
            assert ((snap.running.labels >> 32) == 65535).any(), "no key-65535 pair went through the packed upload"
    if WORLDS[name][0].get("ids") == "small":
        for kind, pods in ((RUN, snap.running), (PEND, snap.pending)):
            eng.upload_pods_compact(kind, abi.compact_pods(pods))
        got, _ = automatic(eng, snap)
        assert_same(snap, got, want)
    else:
        with pytest.raises(ValueError):
            abi.compact_pods(snap.running)
    eng.close()


def _delta(snap, kind, rng):
    """Rows whose labels move to other slots, rows emptied of labels, rows moved to another namespace (in range or not)."""
    pods = snap.running if kind == RUN else snap.pending
    rows = np.sort(rng.choice(pods.n, size=min(pods.n, 150), replace=False)).astype(np.int64)
    d = pods.rows(rows)
    what = rng.integers(0, 3, size=rows.shape[0])
    for j in np.nonzero(what == 0)[0]:
        d.labels[:, j] = d.labels[rng.permutation(snap.L), j]
    d.labels[:, what == 1] = abi.LABEL_EMPTY
    moved = what == 2
    d.ns_id[moved] = rng.integers(0, snap.n_ns + 3, size=int(moved.sum()))
    return rows, d


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WORLDS))
def test_row_deltas(kt, oracle, name):
    """kt_update_pod_rows patches the resident row offsets of the rows it scatters (k_translate_rows on those rows only);
    a fused and a chained pass after the delta give the oracle's bits on the changed snapshot."""
    from test_gpu_parity import assert_same
    from test_partial_passes import run_pass

    snap = world(name)
    eng = _engine(kt, snap)
    run_pass(eng, snap, FRESH, 1)
    rng = np.random.default_rng(zlib.crc32(name.encode()) + 1)
    for kind in (RUN, PEND):
        rows, d = _delta(snap, kind, rng)
        eng.update_pod_rows(kind, rows, d)
        pods = snap.running if kind == RUN else snap.pending
        pods.labels[:, rows] = d.labels
        pods.ns_id[rows] = d.ns_id
    for launches, timing in ((1, False), (3, True)):
        got = run_pass(eng, snap, FRESH, launches, timing)
        assert_same(snap, got, _oracle(oracle, snap, W=got.words_per_row))
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WORLDS))
def test_columns_and_admission(kt, oracle, name):
    """kt_get_match_columns of both kinds against the oracle's bitmaps; kt_admit_queue on the whole queue and on a
    sub-range against the oracle's pod-by-pod admission."""
    from test_match_columns import numpy_columns
    from test_partial_passes import observed_status

    snap = world(name)
    eng = _engine(kt, snap)
    eng.evaluate(snap.now)
    eng.sync()
    W = eng.words_per_row
    want = _oracle(oracle, snap, W=W)
    rng = np.random.default_rng(zlib.crc32(name.encode()) + 2)
    for idx in (np.arange(snap.m), rng.integers(0, snap.m, size=max(1, snap.m // 3)), np.array([snap.m - 1])):
        for kind, bitmap, codes in ((RUN, want.run_bitmap, None), (PEND, want.pend_bitmap, want.codes)):
            off, rows, cs = eng.match_columns(kind, idx)
            w_off, w_rows, w_cs = numpy_columns(bitmap, snap.m, idx, codes)
            np.testing.assert_array_equal(off, w_off)
            np.testing.assert_array_equal(rows, w_rows)
            if codes is not None:
                np.testing.assert_array_equal(cs, w_cs)
    snap.status = observed_status(want, snap, rng)
    snap.normalize()
    eng.upload_status(snap)
    P = snap.pending.n
    for first, count in ((0, P), (P // 4, P // 2)):
        _, admitted = eng.admit_queue(first, count)
        got = eng.download()
        ref, n_adm, _ = oracle.columnar_admit_queue(snap, first, count, 0, words_per_row=W)
        np.testing.assert_array_equal(got.pend_bitmap, ref.pend_bitmap)
        np.testing.assert_array_equal(got.codes, ref.codes)
        np.testing.assert_array_equal(got.admit, ref.admit)
        assert admitted == n_adm
    eng.close()


@pytest.mark.gpu
def test_table_reupload_switches_key_tables_and_counters(kt, oracle):
    """On one engine, throttles re-uploaded from direct keys and 2-bit counters to hashed keys (a key >= 65536) and 6-bit
    counters (a term needing five keys), and back: each pass after a re-upload gives the oracle's bits."""
    from test_gpu_parity import assert_same
    from test_partial_passes import run_pass

    snap = world("general_t2_b2")
    base = compile_tables(kt, snap)
    assert base["n_keydir"] > 0 and base["B"] == 2
    ment = snap.meta["ids"]
    extra = [[([(k, EXISTS, []) for k in ment[1:6]], [], 0)], [([(1 << 20, NOTIN, [3]), (ment[0], EXISTS, [])], [], 0)]]
    other = with_throttles(snap, snap.meta["terms"] + extra, list(snap.kind) + [THROTTLE, CLUSTER], list(snap.thr_ns) + [0, -1],
                           list(snap.thr_flags) + [1, 1])
    t = compile_tables(kt, other)
    assert t["n_keydir"] == 0 and t["B"] == 6
    eng = _engine(kt, snap)
    for s in (snap, other, snap, other):
        eng.upload_throttles(s)
        for launches, timing in ((1, False), (3, True)):
            got = run_pass(eng, s, FRESH, launches, timing)
            assert_same(s, got, _oracle(oracle, s, W=got.words_per_row))
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("m", SHAPE_M)
def test_throttle_counts(kt, oracle, m):
    """Throttle counts around the 32-throttle words (partial last words, one throttle), fused and chained."""
    from test_gpu_parity import assert_same
    from test_partial_passes import run_pass

    snap = copy.deepcopy(_shape_world(m))
    eng = _engine(kt, snap)
    for launches, timing in ((1, False), (3, True)):
        got = run_pass(eng, snap, FRESH, launches, timing)
        assert_same(snap, got, _oracle(oracle, snap, W=got.words_per_row))
    eng.close()


@pytest.mark.gpu
def test_every_variant_reached():
    """Runs after the worlds above: all 12 fused variants, all 8 k_reconcile and all 6 k_check variants ran on edge worlds,
    among them one at L = 32 and one with hashed keys."""
    from test_partial_passes import CHECK_VARIANTS, RECONCILE_VARIANTS

    if {w[0] for w in _worlds_ran} != set(WORLDS):
        pytest.skip("the fused plans did not run on every world")
    assert _fused == {v for _, _, v, _ in VARIANTS} and len(_fused) == 12, sorted(_fused)
    assert {v for k, v in _chained if k == "reconcile"} == RECONCILE_VARIANTS, sorted(_chained)
    assert {v for k, v in _chained if k == "check"} == CHECK_VARIANTS, sorted(_chained)
    assert any(L == 32 for _, L, _ in _worlds_ran) and any(h for _, _, h in _worlds_ran)
