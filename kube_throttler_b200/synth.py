"""Deterministic synthetic snapshots for the BASELINE.json configs (SURVEY.md section 8d).

Pure data generation (numpy, seeded PCG64): pods, namespaces, Throttle/ClusterThrottle specs with
selector tables, thresholds calibrated against the true matched sums, overrides, reservations.
The numpy matcher in here (`match_matrix_numpy`) exists only to calibrate thresholds and to give the
tests a third, independent implementation; it is not on the product path.

Configs (BASELINE.json):
  C1  1 Throttle, 10 running, 1 pending, cpu-only threshold (example/throttle.yaml shape)
  C2  1k Throttles x 100k running x 10k pending, R=4                      (1 GPU; the bench workload)
  C3  600 Throttle + 400 ClusterThrottle, ns selectors, R=8               (2 GPUs)
  C4  5k throttles, 20% with active temporaryThresholdOverrides           (4 GPUs)
  C5  10k x 1M x 100k, R=4                                                (8 GPUs)
"""
from __future__ import annotations

import numpy as np

from . import abi

NOW_2026 = 1767225600 * 10**9  # 2026-01-01T00:00:00Z in unix ns

K_POD_KEYS = 16
V_VALUES = 64
NS_KEY_NAME, NS_KEY_TEAM, NS_KEY_ENV = 100, 101, 102  # namespace label key ids
N_TEAMS, N_ENVS = 8, 4

CONFIGS = {
    "C1": dict(seed=1, m=1, n=10, p=1, R=1),
    "C2": dict(seed=2, m=1000, n=100_000, p=10_000, R=4),
    "C3": dict(seed=3, m=1000, n=100_000, p=10_000, R=8, cluster_frac=0.4, n_ns=50),
    "C4": dict(seed=4, m=5000, n=200_000, p=20_000, R=4, override_frac=0.2),
    "C5": dict(seed=5, m=10_000, n=1_000_000, p=100_000, R=4),
}


def _zipf_p(n: int, s: float = 1.1) -> np.ndarray:
    w = 1.0 / np.arange(1, n + 1) ** s
    return w / w.sum()


def _lab(key, val):
    return (np.asarray(key, np.int64) << 32) | np.asarray(val, np.int64)


def _gen_pods(rng, n: int, n_ns: int, R: int, L: int, running: bool, sort_by_namespace: bool) -> abi.PodCols:
    ns = rng.choice(n_ns, size=n, p=_zipf_p(n_ns)).astype(np.int32)
    if sort_by_namespace:
        ns = np.sort(ns)
    # each pod: ell in [2, L] distinct keys out of K, values Zipf(1.1)
    ell = rng.integers(2, L + 1, size=n)
    keys = np.argsort(rng.random((n, K_POD_KEYS)), axis=1)[:, :L]  # random distinct keys per pod
    keys = np.sort(np.where(np.arange(L)[None, :] < ell[:, None], keys, K_POD_KEYS + 1), axis=1)
    vals = rng.choice(V_VALUES, size=(n, L), p=_zipf_p(V_VALUES))
    labels = np.where(keys <= K_POD_KEYS, _lab(keys, vals), abi.LABEL_EMPTY).astype(np.int64)
    labels = np.ascontiguousarray(labels.T)  # [L][n]

    req = np.zeros((R, n), np.int64)
    present = np.zeros(n, np.uint32)
    # r0 cpu (milli): 50m..4000m step 50m
    req[0] = rng.integers(1, 81, size=n) * 50
    present |= 1
    if R > 1:  # r1 memory (bytes): 64Mi..16Gi powers of two
        req[1] = (64 << 20) << rng.integers(0, 9, size=n)
        present |= 2
    if R > 2:  # r2 nvidia.com/gpu: {0,1,2,4,8}; 0 => 30% absent / 10% explicit zero / rest small
        g = rng.choice([0, 1, 2, 4, 8], size=n, p=[0.4, 0.3, 0.15, 0.1, 0.05])
        u = rng.random(n)
        absent = (g == 0) & (u < 0.75)  # ~30% of all pods
        req[2] = g
        present |= np.where(absent, 0, 4).astype(np.uint32)
    if R > 3:  # r3 ephemeral-storage (bytes): 0..100Gi in 1Gi steps, half of the pods
        has = rng.random(n) < 0.5
        req[3] = np.where(has, rng.integers(0, 101, size=n) << 30, 0)
        present |= np.where(has, 8, 0).astype(np.uint32)
    for r in range(4, R):  # extended resources: sparse small integers
        has = rng.random(n) < 0.15
        req[r] = np.where(has, rng.integers(0, 5, size=n), 0)
        present |= np.where(has, 1 << r, 0).astype(np.uint32)
    req *= ((present[None, :] >> np.arange(R, dtype=np.uint32)[:, None]) & 1).astype(np.int64)

    if running:
        u = rng.random(n)
        flags = np.full(n, abi.POD_SCHEDULER_MATCH | abi.POD_SCHEDULED | abi.POD_NOT_FINISHED, np.uint32)
        flags = np.where(u < 0.05, flags & ~np.uint32(abi.POD_NOT_FINISHED), flags)            # 5% finished
        flags = np.where((u >= 0.05) & (u < 0.08), flags & ~np.uint32(abi.POD_SCHEDULER_MATCH), flags)  # 3% other scheduler
        flags = np.where((u >= 0.08) & (u < 0.10), flags & ~np.uint32(abi.POD_SCHEDULED), flags)        # 2% unscheduled
    else:
        flags = np.full(n, abi.POD_SCHEDULER_MATCH | abi.POD_NOT_FINISHED, np.uint32)
    return abi.PodCols(labels, req, present.astype(np.uint32), flags.astype(np.uint32), ns)


def _namespace_set(ns_reqs_of_terms, ns_labels) -> str:
    """One character per namespace: does some term's namespaceSelector admit it?  (What kt_host.cc orders its ClusterThrottle
    columns by: reorder_columns.)"""
    LN, n_ns = ns_labels.shape
    out = []
    for ns in range(n_ns):
        have = {int(v) >> 32: int(v) & 0xFFFFFFFF for v in ns_labels[:, ns] if int(v) != abi.LABEL_EMPTY}
        ok_any = False
        for reqs in ns_reqs_of_terms:
            ok = True
            for key, op, vals in reqs:
                present = key in have
                if op == abi.OP_IN: ok = present and have[key] in vals
                elif op == abi.OP_NOTIN: ok = (not present) or have[key] not in vals
                elif op == abi.OP_EXISTS: ok = present
                else: ok = not present
                if not ok:
                    break
            if ok:
                ok_any = True
                break
        out.append("1" if ok_any else "0")
    return "".join(out)


def _gen_selectors(rng, m: int, kind: np.ndarray, q_max: int = 0, layout_ns_labels=None, terms=None):
    """CSR selector table: T in {1,2} (80/20), Q in {1,2,3} (60/30/10); 85% equality, 5% each
    In(2-3 values) / NotIn / Exists / DoesNotExist.  ClusterThrottle terms get 0-2 namespace requirements.
    terms=k: T = 1 for k = 1, else uniform in 1..k with the last throttle at exactly k (so k fixes the table's term planes).
    Requirement pool layout: all podSelector requirements (term order), then all namespaceSelector ones."""
    zp = _zipf_p(V_VALUES)
    term_off = [0]
    pod_reqs, ns_reqs = [], []  # per term: list of (key, op, [vals])
    for t in range(m):
        u = rng.random()
        if terms is None:
            T = 1 if u < 0.8 else 2
        else:
            T = terms if t == m - 1 else 1 + int(u * terms)
        for _ in range(T):
            Q = int(rng.integers(1, q_max + 1)) if q_max else int(rng.choice([1, 2, 3], p=[0.6, 0.3, 0.1]))
            keys = rng.choice(K_POD_KEYS, size=Q, replace=False)
            pr = []
            for k in keys:
                u = rng.random()
                if u < 0.85:
                    pr.append((int(k), abi.OP_IN, [int(rng.choice(V_VALUES, p=zp))]))
                elif u < 0.90:
                    pr.append((int(k), abi.OP_IN, [int(v) for v in rng.choice(V_VALUES, size=int(rng.integers(2, 4)), replace=False, p=zp)]))
                elif u < 0.95:
                    pr.append((int(k), abi.OP_NOTIN, [int(v) for v in rng.choice(V_VALUES, size=int(rng.integers(1, 3)), replace=False, p=zp)]))
                elif u < 0.975:
                    pr.append((int(k), abi.OP_EXISTS, []))
                else:
                    pr.append((int(k), abi.OP_DOESNOTEXIST, []))
            nr = []
            if kind[t] == abi.KIND_CLUSTERTHROTTLE:
                u = rng.random()
                if u < 0.5:
                    nr.append((NS_KEY_TEAM, abi.OP_IN, [int(rng.integers(0, N_TEAMS))]))
                elif u < 0.8:
                    nr.append((NS_KEY_ENV, abi.OP_IN, [int(rng.integers(0, N_ENVS))]))
                elif u < 0.9:
                    nr.append((NS_KEY_TEAM, abi.OP_IN, [int(rng.integers(0, N_TEAMS))]))
                    nr.append((NS_KEY_ENV, abi.OP_NOTIN, [int(rng.integers(0, N_ENVS))]))
                # else: empty namespaceSelector == Everything
            pod_reqs.append(pr)
            ns_reqs.append(nr)
        term_off.append(len(pod_reqs))
    if layout_ns_labels is not None:
        # the ClusterThrottles in the order the product's host layer lays its device columns out in: by the set of namespaces
        # their namespaceSelectors admit (only WHICH selector goes to which ClusterThrottle index changes; everything else of a
        # throttle is drawn independently of it)
        blocks = [(pod_reqs[term_off[t]:term_off[t + 1]], ns_reqs[term_off[t]:term_off[t + 1]]) for t in range(m)]
        ct = [t for t in range(m) if kind[t] == abi.KIND_CLUSTERTHROTTLE]
        order = sorted(ct, key=lambda t: (_namespace_set(blocks[t][1], layout_ns_labels), t))
        laid = list(blocks)
        for dst, src in zip(ct, order):
            laid[dst] = blocks[src]
        term_off, pod_reqs, ns_reqs = [0], [], []
        for pr, nr in laid:
            pod_reqs.extend(pr)
            ns_reqs.extend(nr)
            term_off.append(len(pod_reqs))
    return build_selector_csr(term_off, pod_reqs, ns_reqs)


def build_selector_csr(term_off, pod_reqs, ns_reqs, term_flags=None):
    """Pack per-term requirement lists [(key, op, [vals]), ...] into the kt_selector_table CSR arrays."""
    n_terms = len(pod_reqs)
    req_key, req_op, req_val_off, req_vals = [], [], [0], []
    pod_off, ns_off = [0], []
    for pr in pod_reqs:
        for (k, op, vals) in pr:
            req_key.append(k); req_op.append(op); req_vals.extend(vals); req_val_off.append(len(req_vals))
        pod_off.append(len(req_key))
    ns_off.append(len(req_key))
    for nr in ns_reqs:
        for (k, op, vals) in nr:
            req_key.append(k); req_op.append(op); req_vals.extend(vals); req_val_off.append(len(req_vals))
        ns_off.append(len(req_key))
    return dict(term_off=np.array(term_off, np.int32),
                term_flags=np.array(term_flags if term_flags is not None else [0] * n_terms, np.uint8),
                pod_req_off=np.array(pod_off, np.int32), ns_req_off=np.array(ns_off, np.int32),
                req_key=np.array(req_key, np.uint32), req_op=np.array(req_op, np.uint8),
                req_val_off=np.array(req_val_off, np.int32), req_vals=np.array(req_vals, np.uint32))


def match_matrix_numpy(snap: abi.Snapshot, pods: abi.PodCols, t: int, rows: np.ndarray) -> np.ndarray:
    """Selector match of throttle t against pod rows `rows` (numpy, vectorised over rows)."""
    L = snap.L
    lab = pods.labels[:, rows]  # [L][k]
    keys = np.where(lab == abi.LABEL_EMPTY, -1, lab >> 32)
    vals = lab & 0xFFFFFFFF
    ns = pods.ns_id[rows]
    out = np.zeros(rows.shape[0], bool)

    def req_ok(q, keys_, vals_):
        k = int(snap.req_key[q])
        hit = keys_ == k  # [slots][k]
        has = hit.any(axis=0)
        v = np.where(hit, vals_, 0).sum(axis=0)
        vs = snap.req_vals[snap.req_val_off[q]:snap.req_val_off[q + 1]]
        inset = np.isin(v, vs) & has
        op = int(snap.req_op[q])
        if op == abi.OP_IN:
            return inset
        if op == abi.OP_NOTIN:
            return ~inset
        if op == abi.OP_EXISTS:
            return has
        return ~has

    nslab = snap.ns_labels
    nskeys = np.where(nslab == abi.LABEL_EMPTY, -1, nslab >> 32)
    nsvals = nslab & 0xFFFFFFFF
    for term in range(int(snap.term_off[t]), int(snap.term_off[t + 1])):
        ok = np.ones(rows.shape[0], bool)
        if snap.kind[t] == abi.KIND_THROTTLE:
            ok &= ns == snap.thr_ns[t]
        else:
            if snap.term_flags[term] & abi.TERM_NS_INVALID:
                continue
            nsok = np.ones(snap.n_ns, bool)
            for q in range(int(snap.ns_req_off[term]), int(snap.ns_req_off[term + 1])):
                nsok &= req_ok(q, nskeys, nsvals)
            valid = (ns >= 0) & (ns < snap.n_ns)
            ok &= valid & nsok[np.clip(ns, 0, max(snap.n_ns - 1, 0))]
        for q in range(int(snap.pod_req_off[term]), int(snap.pod_req_off[term + 1])):
            if not ok.any():
                break
            ok &= req_ok(q, keys, vals)
        out |= ok
    return out


def _candidate_rows(snap: abi.Snapshot, pods: abi.PodCols, t: int, ns_sorted_bounds):
    if snap.kind[t] == abi.KIND_THROTTLE and ns_sorted_bounds is not None:
        lo, hi = ns_sorted_bounds[int(snap.thr_ns[t])], ns_sorted_bounds[int(snap.thr_ns[t]) + 1]
        return np.arange(lo, hi)
    if snap.kind[t] == abi.KIND_THROTTLE:
        return np.nonzero(pods.ns_id == snap.thr_ns[t])[0]
    return np.arange(pods.n)


def true_used_numpy(snap: abi.Snapshot):
    """Per-throttle used sums / presence / counts over the running pods (numpy)."""
    m, R = snap.m, snap.R
    pods = snap.running
    used = np.zeros((R, m), np.int64)
    present = np.zeros(m, np.uint32)
    cnt = np.zeros(m, np.int64)
    bounds = None
    if np.all(np.diff(pods.ns_id) >= 0):
        bounds = np.searchsorted(pods.ns_id, np.arange(snap.n_ns + 1))
    counted = (pods.flags & (abi.POD_SCHEDULER_MATCH | abi.POD_SCHEDULED)) == (abi.POD_SCHEDULER_MATCH | abi.POD_SCHEDULED)
    alive = counted & ((pods.flags & abi.POD_NOT_FINISHED) != 0)
    for t in range(m):
        if not (snap.thr_flags[t] & abi.THR_RESPONSIBLE) or (snap.thr_flags[t] & abi.THR_SELECTOR_ERROR):
            continue
        rows = _candidate_rows(snap, pods, t, bounds)
        if rows.size == 0:
            continue
        sel = match_matrix_numpy(snap, pods, t, rows) & alive[rows]
        rr = rows[sel]
        if rr.size == 0:
            continue
        cnt[t] = rr.size
        pm = np.uint32(abi.COUNT_BIT)
        for r in range(R):
            has = (pods.present[rr] >> np.uint32(r)) & 1
            if has.any():
                pm |= np.uint32(1 << r)
                used[r, t] = int((pods.req[r, rr] * has).sum())
        present[t] = pm
    return used, present, cnt


VALUE_REGIMES = ("wide", "carry", "signed")
HIGH_LIMB = 1 << 44  # warp_sum_u64 adds bits 44-63 as its third limb


def _rewrite_values(pods: abi.PodCols, rng, regime: str, bound: int) -> None:
    """Replace every present request by a value of the regime (absent ones stay 0)."""
    R, n = pods.req.shape
    has = ((pods.present[None, :] >> np.arange(R, dtype=np.uint32)[:, None]) & 1).astype(bool)
    if regime == "wide":      # [2^44, bound) with random low bits: the high limb of every warp sum is busy
        v = rng.integers(HIGH_LIMB, bound, size=(R, n), dtype=np.int64)
    elif regime == "carry":   # low 32 bits all ones (so the low 22 too): every limb and every 32-bit half carries
        v = (rng.integers(0, min(1 << 14, bound >> 32), size=(R, n), dtype=np.int64) << 32) | 0xFFFFFFFF
    elif regime == "signed":  # both signs, a tenth present with value zero
        v = rng.integers(-(1 << 40), 1 << 40, size=(R, n), dtype=np.int64)
        v = np.where(rng.random((R, n)) < 0.1, 0, v)
    else:
        raise ValueError(f"values={regime!r}: expected one of {VALUE_REGIMES}")
    pods.req = np.ascontiguousarray(np.where(has, v, 0).astype(np.int64))


def _equality_thresholds(snap: abi.Snapshot, rng, frac: float = 0.12) -> None:
    """Thresholds exactly at the edges of the check, from the exact matched sums (Python ints): on about half of the chosen
    throttles S3's alreadyUsed == threshold (a resource column and the count), on the others S4's alreadyUsed + the request of one
    matched pending pod == threshold (a column the pod requests non-zero, and the count).  A `>` / `>=` mix-up then changes
    codes under both isThrottledOnEqual settings.  Throttles with overrides are left alone (their spec threshold is not the
    calculated one)."""
    used, _, ucnt = true_used_numpy(snap)
    m, R = snap.m, snap.R
    pend = snap.pending
    live = ((snap.thr_flags & abi.THR_RESPONSIBLE) != 0) & ((snap.thr_flags & abi.THR_SELECTOR_ERROR) == 0)
    pick = np.nonzero((rng.random(m) < frac) & live & (np.diff(snap.ovr_off) == 0))[0]
    thr, thr_present, thr_cnt = snap.thr.copy(), snap.thr_present.copy(), snap.thr_cnt.copy()
    s4 = False
    for t in pick.tolist():
        already = [int(used[r, t]) + int(snap.reserved[r, t]) for r in range(R)]  # Python ints: exact
        cnt = int(ucnt[t]) + int(snap.reserved_cnt[t])
        rows = _candidate_rows(snap, pend, t, None)
        rows = rows[match_matrix_numpy(snap, pend, t, rows)] if rows.size else rows
        s4 = not s4 and rows.size > 0  # alternate, among the throttles some pending pod affects
        if not s4:      # S3
            r = int(rng.integers(R))
            thr[r, t], thr_cnt[t] = already[r], cnt
        else:           # S4: one pending pod the throttle affects
            i = int(rows[rng.integers(rows.size)])
            cols = [r for r in range(R) if (int(pend.present[i]) >> r) & 1 and int(pend.req[r, i]) != 0]
            r = cols[int(rng.integers(len(cols)))] if cols else int(rng.integers(R))
            thr[r, t], thr_cnt[t] = already[r] + int(pend.req[r, i]), cnt + 1
        thr_present[t] |= np.uint32((1 << r) | abi.COUNT_BIT)
    snap.thr, snap.thr_present, snap.thr_cnt = thr, thr_present, thr_cnt


def generate(config: str = "C2", *, seed=None, m=None, n=None, p=None, R=None, n_ns=None, cluster_frac=None,
             override_frac=None, L: int = 8, sort_by_namespace: bool = True, now: int = NOW_2026,
             calibrate: bool = True, q_max: int = 0, column_layout: bool = False, values=None, terms=None) -> abi.Snapshot:
    """Build the snapshot of a BASELINE config (or a scaled variant via keyword overrides).

    terms: None draws one or two selector terms per throttle (80/20); 1 gives every throttle one term (one term plane per
    table entry); 2, 3 or 4 draw 1..terms terms, with the last throttle at exactly `terms` (3: two plane pairs, one of them a
    padded empty plane; 4: two full plane pairs).

    values: None keeps the requests of the config (cpu milli, memory bytes, ...); "wide", "carry" or "signed" rewrites the
    request columns of the running and pending pods (VALUE_REGIMES, _rewrite_values) before the thresholds are calibrated, within
    the domain the host layer guarantees (per column, sum of |v| over running + pending + reservations + status below 2^62), and
    adds exact-equality thresholds (_equality_thresholds)."""
    if terms not in (None, 1, 2, 3, 4):
        raise ValueError(f"terms={terms!r}: expected None or 1..4")
    base = dict(CONFIGS[config])
    for k, v in dict(seed=seed, m=m, n=n, p=p, R=R, n_ns=n_ns, cluster_frac=cluster_frac, override_frac=override_frac).items():
        if v is not None:
            base[k] = v
    if config == "C1" and m is None and n is None:
        return _generate_c1(now)
    seed, m, n, p, R = base["seed"], base["m"], base["n"], base["p"], base["R"]
    cluster_frac = base.get("cluster_frac", 0.0)
    override_frac = base.get("override_frac", 0.0)
    n_ns = base.get("n_ns") or max(1, m // 20)
    rng = np.random.Generator(np.random.PCG64(seed))
    LN = 4

    # namespaces: kubernetes.io/metadata.name=<ns>, team, env
    ns_labels = np.full((LN, n_ns), abi.LABEL_EMPTY, np.int64)
    ns_labels[0] = _lab(NS_KEY_NAME, 1000 + np.arange(n_ns))
    ns_labels[1] = _lab(NS_KEY_TEAM, rng.integers(0, N_TEAMS, size=n_ns))
    ns_labels[2] = _lab(NS_KEY_ENV, rng.integers(0, N_ENVS, size=n_ns))

    running = _gen_pods(rng, n, n_ns, R, L, True, sort_by_namespace)
    pending = _gen_pods(rng, p, n_ns, R, L, False, sort_by_namespace)
    vrng = None
    if values is not None:  # its own stream: the default snapshots stay byte-identical
        vrng = np.random.Generator(np.random.PCG64([seed, VALUE_REGIMES.index(values) if values in VALUE_REGIMES else 99]))
        # running + pending at most 2^60, status used at most as much again, reservations small: below 2^62 per column
        bound = (1 << 60) // (n + p)
        if bound <= HIGH_LIMB + (1 << 40):
            raise ValueError(f"values={values!r}: {n + p} pods leave no room above 2^44 under the 2^62 column bound")
        for pods in (running, pending):
            _rewrite_values(pods, vrng, values, bound)

    # throttles: Throttles grouped by namespace first, then ClusterThrottles
    m_c = int(round(m * cluster_frac))
    m_t = m - m_c
    kind = np.concatenate([np.full(m_t, abi.KIND_THROTTLE, np.uint8), np.full(m_c, abi.KIND_CLUSTERTHROTTLE, np.uint8)])
    thr_ns = np.concatenate([np.sort(rng.integers(0, n_ns, size=m_t)), np.full(m_c, -1)]).astype(np.int32)
    thr_flags = np.full(m, abi.THR_RESPONSIBLE, np.uint8)
    thr_flags[rng.random(m) < 0.01] = 0  # 1% belong to another throttler instance

    # q_max > 3: terms needing > 3 keys present (6-bit counters); column_layout: ClusterThrottles ordered as kt_host.cc orders them
    sel = _gen_selectors(rng, m, kind, q_max, layout_ns_labels=ns_labels if column_layout else None, terms=terms)

    snap = abi.Snapshot(
        R=R, L=L, LN=LN, running=running, pending=pending, ns_labels=ns_labels, kind=kind, thr_ns=thr_ns,
        thr_flags=thr_flags, thr=np.zeros((R, m), np.int64), thr_present=np.zeros(m, np.uint32),
        thr_cnt=np.zeros(m, np.int64), ovr_off=np.zeros(m + 1, np.int32), ovr_begin=np.zeros(0, np.int64),
        ovr_end=np.zeros(0, np.int64), ovr_flags=np.zeros(0, np.uint8), ovr_thr=np.zeros((R, 0), np.int64),
        ovr_present=np.zeros(0, np.uint32), ovr_cnt=np.zeros(0, np.int64), now=now, **sel,
        meta=dict(config=config, seed=seed, m=m, n=n, p=p, R=R, n_ns=n_ns, L=L))
    snap.normalize()

    # ---- thresholds: q in U[0.5,1.5] x true matched sum; 1% pod:0 (Q4); 2% exact equality (Q1/Q2) ----
    if calibrate:
        used, upresent, ucnt = true_used_numpy(snap)
    else:
        used, upresent, ucnt = np.zeros((R, m), np.int64), np.zeros(m, np.uint32), np.zeros(m, np.int64)
    snap.meta["true_used"] = (used, upresent, ucnt)
    # three equally likely regimes per throttle so pending pods spread over active / insufficient / not-throttled:
    #   0: threshold below the used sum (q in [0.5,1))   1: about one pod of headroom   2: ample headroom (q in [1.2,2])
    typical = np.array([4000, 8 << 30, 8, 100 << 30] + [4] * max(0, R - 4), np.int64)[:R]
    one_pod = np.array([2000, 1 << 30, 2, 50 << 30] + [2] * max(0, R - 4), np.int64)[:R]
    if values is not None:  # the same regimes of headroom, in units of the rewritten requests
        one_pod = np.array([max(1, int(np.median(np.abs(pods_r[pods_r != 0])))) if (pods_r != 0).any() else 1
                            for pods_r in pending.req], np.int64)
        typical = 4 * one_pod
    regime = rng.integers(0, 3, size=m)
    base_amt = np.where(used > 0, used, typical[:, None])
    q = np.where(regime[None, :] == 0, rng.uniform(0.5, 1.0, size=(R, m)), rng.uniform(1.2, 2.0, size=(R, m)))
    thr = (base_amt * q).astype(np.int64)
    near = (used + (rng.uniform(0.0, 1.5, size=(R, m)) * one_pod[:, None]).astype(np.int64))
    thr = np.maximum(1, np.where(regime[None, :] == 1, near, thr))
    p_has = np.array([0.9, 0.7, 0.3, 0.2] + [0.1] * max(0, R - 4))[:R]
    has = rng.random((R, m)) < p_has[:, None]
    thr_present = (has.astype(np.uint32) << np.arange(R, dtype=np.uint32)[:, None]).sum(axis=0).astype(np.uint32)
    has_cnt = rng.random(m) < 0.5
    qc = np.where(regime == 0, rng.uniform(0.5, 1.0, size=m), rng.uniform(1.2, 2.0, size=m))
    thr_cnt = (np.where(ucnt > 0, ucnt, 10) * qc).astype(np.int64)
    thr_cnt = np.maximum(1, np.where(regime == 1, ucnt + rng.integers(0, 3, size=m), thr_cnt))
    u = rng.random(m)
    exact = u < 0.02  # threshold == used exactly on cpu (and the count when present)
    thr[0] = np.where(exact & (used[0] > 0), used[0], thr[0])
    thr_present = np.where(exact, thr_present | 1, thr_present).astype(np.uint32)
    thr_cnt = np.where(exact & (ucnt > 0), ucnt, thr_cnt)
    zero_pod = (u >= 0.02) & (u < 0.03)
    has_cnt = has_cnt | zero_pod
    thr_cnt = np.where(zero_pod, 0, thr_cnt)
    thr_present = np.where(has_cnt, thr_present | abi.COUNT_BIT, thr_present).astype(np.uint32)
    snap.thr = (thr * has).astype(np.int64)
    snap.thr_present = thr_present
    snap.thr_cnt = np.where(has_cnt, thr_cnt, 0).astype(np.int64)

    # ---- temporaryThresholdOverrides (C4): 1-3 per chosen throttle, >=1 active at `now` ----
    if override_frac > 0:
        chosen = rng.random(m) < override_frac
        counts = np.where(chosen, rng.integers(1, 4, size=m), 0)
        ovr_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
        n_ovr = int(ovr_off[-1])
        day = 86400 * 10**9
        begin = np.empty(n_ovr, np.int64)
        end = np.empty(n_ovr, np.int64)
        oflags = np.zeros(n_ovr, np.uint8)
        othr = np.zeros((R, n_ovr), np.int64)
        opresent = np.zeros(n_ovr, np.uint32)
        ocnt = np.zeros(n_ovr, np.int64)
        for t in np.nonzero(chosen)[0]:
            lo, hi = ovr_off[t], ovr_off[t + 1]
            for j, i in enumerate(range(lo, hi)):
                active = j == 0 or rng.random() < 0.5  # first one always active -> overlapping pairs happen
                if active:
                    begin[i] = now - int(rng.integers(0, 30)) * day
                    end[i] = now + int(rng.integers(0, 30)) * day
                else:
                    begin[i] = now + int(rng.integers(1, 30)) * day
                    end[i] = begin[i] + 5 * day
                uu = rng.random()
                if uu < 0.1:
                    begin[i] = abi.TIME_OPEN_BEGIN
                elif uu < 0.2:
                    end[i] = abi.TIME_OPEN_END if active else end[i]
                if rng.random() < 0.01:
                    oflags[i] = abi.OVR_PARSE_ERROR
                pm = 0
                for r in range(R):
                    if rng.random() < 0.5:
                        pm |= 1 << r
                        othr[r, i] = max(1, int(snap.thr[r, t] * rng.uniform(0.5, 2.0)) if snap.thr[r, t] else int(typical[r]))
                if rng.random() < 0.4:
                    pm |= abi.COUNT_BIT
                    ocnt[i] = int(rng.integers(0, 50))
                opresent[i] = pm
        snap.ovr_off, snap.ovr_begin, snap.ovr_end, snap.ovr_flags = ovr_off, begin, end, oflags
        snap.ovr_thr, snap.ovr_present, snap.ovr_cnt = othr, opresent, ocnt

    # ---- reservations: 5% of throttles carry reserved-but-unobserved pods ----
    rsv = rng.random(m) < 0.05
    rcnt = np.where(rsv, rng.integers(1, 4, size=m), 0).astype(np.int64)
    reserved = np.zeros((R, m), np.int64)
    rpresent = np.where(rsv, abi.COUNT_BIT | 1, 0).astype(np.uint32)
    reserved[0] = rcnt * 250
    if R > 1:
        mem = rsv & (rng.random(m) < 0.5)
        reserved[1] = np.where(mem, rcnt * (256 << 20), 0)
        rpresent = np.where(mem, rpresent | 2, rpresent).astype(np.uint32)
    snap.reserved, snap.reserved_present, snap.reserved_cnt = reserved, rpresent, rcnt
    if vrng is not None:
        snap.meta["values"] = values
        _equality_thresholds(snap.normalize(), vrng)
    return snap.normalize()


def _generate_c1(now: int) -> abi.Snapshot:
    """BASELINE config 1: example/throttle.yaml reduced to a cpu-only threshold of 200m, 10 running pods
    labelled throttle=t1 at 10m each, pending pods at 100m / 101m / 300m (admit / insufficient / exceeds)."""
    L, R, LN = 2, 1, 1
    KEY_THROTTLE, VAL_T1 = 0, 0
    n, p = 10, 3
    lab = np.full((L, n), abi.LABEL_EMPTY, np.int64)
    lab[0] = _lab(KEY_THROTTLE, VAL_T1)
    running = abi.PodCols(lab, np.full((R, n), 10, np.int64), np.ones(n, np.uint32),
                          np.full(n, 7, np.uint32), np.zeros(n, np.int32))
    plab = np.full((L, p), abi.LABEL_EMPTY, np.int64)
    plab[0] = _lab(KEY_THROTTLE, VAL_T1)
    pending = abi.PodCols(plab, np.array([[100, 101, 300]], np.int64), np.ones(p, np.uint32),
                          np.full(p, 5, np.uint32), np.zeros(p, np.int32))
    snap = abi.Snapshot(
        R=R, L=L, LN=LN, running=running, pending=pending, ns_labels=np.full((LN, 1), abi.LABEL_EMPTY, np.int64),
        kind=np.zeros(1, np.uint8), thr_ns=np.zeros(1, np.int32), thr_flags=np.ones(1, np.uint8),
        thr=np.array([[200]], np.int64), thr_present=np.array([1], np.uint32), thr_cnt=np.zeros(1, np.int64),
        ovr_off=np.zeros(2, np.int32), ovr_begin=np.zeros(0, np.int64), ovr_end=np.zeros(0, np.int64),
        ovr_flags=np.zeros(0, np.uint8), ovr_thr=np.zeros((R, 0), np.int64), ovr_present=np.zeros(0, np.uint32),
        ovr_cnt=np.zeros(0, np.int64), term_off=np.array([0, 1], np.int32), term_flags=np.zeros(1, np.uint8),
        pod_req_off=np.array([0, 1], np.int32), ns_req_off=np.array([1, 1], np.int32),
        req_key=np.array([KEY_THROTTLE], np.uint32), req_op=np.array([abi.OP_IN], np.uint8),
        req_val_off=np.array([0, 1], np.int32), req_vals=np.array([VAL_T1], np.uint32), now=now,
        meta=dict(config="C1", m=1, n=n, p=p, R=R))
    return snap.normalize()
