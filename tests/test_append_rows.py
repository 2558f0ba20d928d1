"""kt_append_throttle_rows: new throttle columns appended at [M, M+k) on the device -- Throttle and ClusterThrottle creations --
without recompiling the selector tables when the new columns fit them.

Two engines hold the same pods, namespaces, throttles, observed status and reservations.  One gets every change as a whole
kt_upload_throttles of the grown spec followed by the status and reservations widened by zero columns; the other gets the new
columns through kt_append_throttle_rows, k = 1, 16 or 256 columns a step cut into random batches without a pass in between,
then status and reservation row deltas for some of the new columns.  Appends start from M = 0 and from M a multiple of 32, stay
inside the last 32-throttle word, cross word boundaries and 128-column boundaries (the bitmap row width Wp), and carry
temporaryThresholdOverrides.  Appends that need a new table row, more term planes or more counter planes than the resident
tables have must compile the tables again (recompiled = 1) and answer the same; the others must not.  Hole fills through the
selector and threshold deltas, deletions, status, reservation and namespace-row deltas and kt_upload_namespaces are mixed in.
After every step both engines must answer bit for bit alike (FRESH, GIVEN and ON_EQUAL passes queued back to back under every
forced pass plan, the status diff, the check summary and the keyed calls, kt_admit_queue, the check rows), equal the columnar
oracle, and hold the namespace word lists kt_debug_compile_tables builds for the grown spec (and its masks where the two
term-plane counts agree)."""
import copy
import ctypes as C

import numpy as np
import pytest

from kube_throttler_b200 import KtError, abi, synth
from test_namespace_rows import GIVEN, PLANS, WORLDS, assert_oracle, assert_same, batches, observe, synth_words
from test_partial_passes import observed_status
from test_selector_rows import columns, edit, ns_tables_match, pack
from test_tables_cpu import compile_tables
from test_threshold_rows import rand_override

pytestmark = pytest.mark.gpu

STATUS = ("calculated", "calc_thr", "calc_present", "calc_cnt", "used", "used_present", "used_cnt", "throttled")


def thr_columns(snap):
    """Per throttle column: (thr[R], present, cnt, overrides), an override being (begin, end, flags, thr[R], present, cnt)."""
    out = []
    for t in range(snap.m):
        ovr = [(int(snap.ovr_begin[e]), int(snap.ovr_end[e]), int(snap.ovr_flags[e]), snap.ovr_thr[:, e].copy(), int(snap.ovr_present[e]),
                int(snap.ovr_cnt[e])) for e in range(snap.ovr_off[t], snap.ovr_off[t + 1])]
        out.append((snap.thr[:, t].copy(), int(snap.thr_present[t]), int(snap.thr_cnt[t]), ovr))
    return out


def pack_thr(tcols, R):
    """The columns' thresholds and their override CSR, named like the Snapshot fields."""
    ovr = [o for c in tcols for o in c[3]]
    return dict(thr=np.array([c[0] for c in tcols], np.int64).reshape(len(tcols), R).T.copy(), thr_present=np.array([c[1] for c in tcols], np.uint32),
                thr_cnt=np.array([c[2] for c in tcols], np.int64), ovr_off=np.cumsum([0] + [len(c[3]) for c in tcols]).astype(np.int32),
                ovr_begin=np.array([o[0] for o in ovr], np.int64), ovr_end=np.array([o[1] for o in ovr], np.int64),
                ovr_flags=np.array([o[2] for o in ovr], np.uint8), ovr_thr=np.array([o[3] for o in ovr], np.int64).reshape(len(ovr), R).T.copy(),
                ovr_present=np.array([o[4] for o in ovr], np.uint32), ovr_cnt=np.array([o[5] for o in ovr], np.int64))


def zero_status(R, m):
    return {f: np.zeros((R, m) if f in ("calc_thr", "used") else m, np.uint8 if f == "calculated" else np.int64) for f in STATUS}


class World:
    """The current throttle side (selector columns, threshold columns, status, reservations) over a fixed pod and namespace side."""

    def __init__(self, base, cols, tcols, status, reserved):
        self.base, self.cols, self.tcols, self.status, self.reserved = base, cols, tcols, status, reserved

    def snap(self):
        s = copy.copy(self.base)
        for f, v in dict(pack(self.cols), **pack_thr(self.tcols, s.R)).items():
            setattr(s, f, v)
        s.status = self.status
        s.reserved, s.reserved_present, s.reserved_cnt = self.reserved
        return s.normalize()

    def append(self, cols, tcols):
        R, k = self.base.R, len(cols)
        self.cols += cols
        self.tcols += tcols
        if self.status is not None:
            self.status = {f: np.concatenate([v, np.zeros((R, k) if v.ndim == 2 else k, v.dtype)], axis=v.ndim - 1) for f, v in self.status.items()}
        r, p, c = self.reserved
        self.reserved = (np.concatenate([r, np.zeros((R, k), np.int64)], axis=1), np.concatenate([p, np.zeros(k, np.uint32)]),
                         np.concatenate([c, np.zeros(k, np.int64)]))


def engines(kt, snap):
    out = []
    for _ in range(2):
        e = kt.Engine(snap.R, snap.L, snap.LN)
        e.upload_namespaces(snap.ns_labels)
        e.upload_throttles(snap)
        if snap.status is not None:
            e.upload_status(snap)
        e.set_reserved(snap)
        e.upload_pods(abi.PODS_RUNNING, snap.running)
        e.upload_pods(abi.PODS_PENDING, snap.pending)
        e.set_sparse_check(1 << 16)
        out.append(e)
    return out


def vocab_of(cols):
    """The podSelector keys and (key, value) pairs the tables compiled from these columns have rows for."""
    keys, pairs = set(), set()
    for c in cols:
        for tm in c[3]:
            for key, _, vals in tm[1]:
                keys.add(key)
                pairs.update((key, v) for v in vals)
    return keys, pairs


def fits(c, vocab, res, L):
    """Does a new column fit the resident tables: rows for its keys and pairs, terms within TPpad, need within the counter
    planes (a term needing more keys than a pod row holds needs none), a Throttle's namespace below NS?"""
    keys, pairs = vocab
    if len(c[3]) > res["TPpad"] or (c[0] == abi.KIND_THROTTLE and c[1] >= res["NS"]):
        return False
    for tm in c[3]:
        if any(key not in keys or any((key, v) not in pairs for v in vals) for key, _, vals in tm[1]):
            return False
        need = len({key for key, op, _ in tm[1] if op in (abi.OP_IN, abi.OP_EXISTS)})
        if need <= L and need >= 1 << res["B"]:
            return False
    return True


def code(fn):
    with pytest.raises(KtError) as ex:
        fn()
    return ex.value.code


# (operation, k): "append" takes the next pool columns; "beyond" edits them past the resident tables; "hole" deletes columns and
# fills them again through the selector and threshold deltas; "mixed" adds namespace, threshold, status and reservation row
# deltas; "reupload_ns" a whole namespace upload.
STEPS = [("append", 1), ("append", 16), ("append", 256), ("beyond:new_key", 1), ("hole", 16), ("append", 16), ("mixed", 1),
         ("beyond:more_terms", 16), ("append", 1), ("beyond:wide_need", 16), ("reupload_ns", 256), ("append", 16)]


@pytest.mark.parametrize("start", ["zero", "word"])
@pytest.mark.parametrize("world", list(WORLDS))
def test_appends_equal_full_uploads(kt, oracle, world, start):
    full_snap = WORLDS[world]()
    rng = np.random.default_rng(sum(map(ord, world + start)) + 23)
    pool_cols, pool_thr = columns(full_snap), thr_columns(full_snap)
    pool_status = observed_status(oracle.columnar_evaluate(full_snap, abi.EVAL_FRESH_STATUS, words_per_row=synth_words(full_snap)), full_snap, rng)
    R, L, n_pool = full_snap.R, full_snap.L, full_snap.m
    for t in range(0, n_pool, 3):  # temporaryThresholdOverrides on every third column
        pool_thr[t] = pool_thr[t][:3] + ([rand_override(rng, R, full_snap.now, False) for _ in range(1 + (t // 3) % 3)],)
    m0 = 0 if start == "zero" else min(64, n_pool // 32 * 32)
    reserved = (full_snap.reserved[:, :m0].copy(), full_snap.reserved_present[:m0].copy(), full_snap.reserved_cnt[:m0].copy()) \
        if full_snap.reserved is not None else (np.zeros((R, m0), np.int64), np.zeros(m0, np.uint32), np.zeros(m0, np.int64))
    status = {f: (v[:, :m0] if v.ndim == 2 else v[:m0]).copy() for f, v in pool_status.items()} if m0 else None
    w = World(full_snap, [list(c) for c in pool_cols[:m0]], list(pool_thr[:m0]), status, reserved)
    full, delta = engines(kt, w.snap())
    # what the resident tables were last compiled with: the fit test of a new column is against it
    res, vocab = compile_tables(kt, w.snap()), vocab_of(w.cols)
    seen = {0: 0, 1: 0}
    nxt = m0
    for step, (op, k) in enumerate(STEPS):
        m = len(w.cols)
        where = f"{world} from {start} step {step} {op} k={k} m={m}"
        if op in ("append", "mixed", "reupload_ns") or op.startswith("beyond"):
            how = op.split(":")[1] if op.startswith("beyond") else None
            ok = [t for t in range(n_pool) if fits(pool_cols[t], vocab, res, L)] if how is None else []
            src = [ok[(nxt + i) % len(ok)] for i in range(k)] if ok else [(nxt + i) % n_pool for i in range(k)]
            nxt += k
            new_cols, new_thr = [list(pool_cols[t]) for t in src], [pool_thr[t] for t in src]
            all_cols = w.cols + new_cols
            if how is not None and (how != "wide_need" or (res["B"] == 2 and L >= 4 and len(vocab[0]) >= 4)):
                for i in range(k):
                    edit(rng, all_cols, m + i, how, res["TPpad"])
            new_cols = all_cols[m:]
            beyond = not all(fits(c, vocab, res, L) for c in new_cols)
            w.append(new_cols, new_thr)
            snap = w.snap()
            full.upload_throttles(snap)
            if snap.status is not None:
                full.upload_status(snap)
            full.set_reserved(snap)
            got, at = set(), m
            for b in batches(rng, np.arange(k)):  # several appends, no pass in between
                b = np.sort(b)
                n = len(b)
                cols = dict(pack(new_cols[at - m:at - m + n]), **pack_thr(new_thr[at - m:at - m + n], R))
                got.add(delta.append_throttle_rows(cols))
                at += n
            assert delta.m == snap.m == m + k, where
            if beyond:
                assert True in got, where
                res, vocab = compile_tables(kt, snap), vocab_of(w.cols)
            else:
                assert got == {False}, where
            seen[int(beyond)] += 1
            if w.status is None:  # no status before the call: still none after it
                assert code(lambda: delta.evaluate(0, GIVEN)) == abi.ERR_STATE, where
                w.status = {f: (v[:, :len(w.cols)] if v.ndim == 2 else v[:len(w.cols)]).copy() for f, v in pool_status.items()} \
                    if len(w.cols) <= n_pool else None
                if w.status is None:
                    w.status = zero_status(R, len(w.cols))
                snap = w.snap()
                for e in (full, delta):
                    e.upload_status(snap)
            else:  # an informer's status and a Reserve for some of the new columns: row deltas against whole uploads
                sc = np.sort(rng.choice(np.arange(m, m + k), size=max(1, k // 3), replace=False)).astype(np.int32)
                like = rng.integers(0, n_pool, size=len(sc))
                for f, v in w.status.items():
                    v[..., sc] = pool_status[f][..., like]
                r, p, cnt = w.reserved
                r[0, sc] = rng.integers(0, 3000, size=len(sc))
                p[sc] |= 1
                cnt[sc] = rng.integers(0, 4, size=len(sc))
                snap = w.snap()
                full.upload_status(snap)
                full.set_reserved(snap)
                delta.update_status_rows(sc, {f: (v[:, sc] if v.ndim == 2 else v[sc]) for f, v in w.status.items()})
                delta.update_reserved_rows(sc, r[:, sc], p[sc], cnt[sc])
        if op == "hole":  # deletions, then the holes filled with other columns through the existing deltas
            k = min(k, m)
            holes = np.sort(rng.choice(m, size=k, replace=False)).astype(np.int32)
            for t in holes:
                w.cols[t] = [w.cols[t][0], w.cols[t][1], 0, []]
            snap = w.snap()
            full.upload_throttles(snap)
            full.upload_status(snap)
            full.set_reserved(snap)
            delta.update_selector_rows(holes, pack([w.cols[t] for t in holes]))
            fill = [(nxt + i) % n_pool for i in range(k)]
            nxt += k
            for t, s in zip(holes, fill):
                w.cols[t] = list(pool_cols[s])
                w.tcols[t] = pool_thr[s]
                for f, v in w.status.items():
                    v[..., t] = 0
                w.reserved[0][:, t] = 0
                w.reserved[1][t] = 0
                w.reserved[2][t] = 0
            snap = w.snap()
            full.upload_throttles(snap)
            full.upload_status(snap)
            full.set_reserved(snap)
            recompiled = delta.update_selector_rows(holes, pack([w.cols[t] for t in holes]))
            delta.update_threshold_rows(holes, pack_thr([w.tcols[t] for t in holes], R))
            delta.update_status_rows(holes, {f: (v[:, holes] if v.ndim == 2 else v[holes]) for f, v in w.status.items()})
            delta.update_reserved_rows(holes, w.reserved[0][:, holes], w.reserved[1][holes], w.reserved[2][holes])
            if recompiled:
                res, vocab = compile_tables(kt, snap), vocab_of(w.cols)
        if op == "mixed":  # a namespace-row delta and a threshold edit of a new column on both engines after the append
            nsr = np.array([0], np.int32)
            base = w.base
            base.ns_labels = base.ns_labels.copy()
            base.ns_labels[:, 0] = base.ns_labels[:, min(1, base.n_ns - 1)]
            t = len(w.cols) - 1
            thr = w.tcols[t][0].copy()
            thr[0] = int(rng.integers(0, 4000))
            w.tcols[t] = (thr, w.tcols[t][1] | 1, w.tcols[t][2], w.tcols[t][3])
            snap = w.snap()
            for e in (full, delta):
                e.update_namespace_rows(snap.n_ns, nsr, snap.ns_labels[:, nsr])
                e.update_threshold_rows(np.array([t], np.int32), pack_thr([w.tcols[t]], R))
        if op == "reupload_ns":  # a whole namespace upload after the appends: the tables compiled from the grown spec
            snap = w.snap()
            for e in (full, delta):
                e.upload_namespaces(snap.ns_labels)
            res, vocab = compile_tables(kt, snap), vocab_of(w.cols)
        snap = w.snap()
        assert full.words_per_row == delta.words_per_row, where
        ns_tables_match(kt, delta, snap, where)
        assert_oracle(delta, snap, oracle, where)
        m = snap.m
        rows = rng.integers(0, snap.pending.n, size=min(snap.pending.n, 19))
        idx = rng.choice(m, size=min(m, 9), replace=False).astype(np.int32)
        probe = (rows, idx, snap.pending.labels[:, rows], snap.pending.ns_id[rows].astype(np.int32))
        plan = PLANS[step % len(PLANS)]
        assert_same(observe(full, snap, plan, probe), observe(delta, snap, plan, probe), where + f" plan {plan}")
    assert seen[0] >= 6 and seen[1] >= 2, seen
    full.close()
    delta.close()


def test_argument_and_state_errors(kt):
    snap = synth.generate("C3", m=40, n=200, p=50, n_ns=6).normalize()
    e = kt.Engine(snap.R, snap.L, snap.LN)
    L, h = e._L, e._h
    cols, tcols = columns(snap), thr_columns(snap)
    two = dict(pack(cols[1:3]), **pack_thr(tcols[1:3], snap.R))

    assert code(lambda: e.append_throttle_rows(two)) == abi.ERR_STATE  # before kt_upload_throttles
    e.upload_namespaces(snap.ns_labels)
    e.upload_throttles(snap)
    assert e.m == snap.m
    a = {f: np.ascontiguousarray(v) for f, v in two.items()}

    def structs(**over):
        x = dict(a, **over)
        tc = abi.ThrottleCols(*(abi.ptr(x[f]) for f in ("kind", "thr_ns", "thr_flags", "thr", "thr_present", "thr_cnt", "ovr_off")),
                              int(x["ovr_off"][-1]), *(abi.ptr(x[f]) for f in ("ovr_begin", "ovr_end", "ovr_flags", "ovr_thr", "ovr_present", "ovr_cnt")))
        st = abi.SelectorTable(int(x["term_off"][-1]), int(x["req_key"].shape[0]), int(x["req_vals"].shape[0]),
                               *(abi.ptr(x[f]) for f in ("term_off", "term_flags", "pod_req_off", "ns_req_off", "req_key", "req_op", "req_val_off", "req_vals")))
        return tc, st

    def call(k, tc, st):
        out = np.full(1, 7, np.int32)
        rc = L.kt_append_throttle_rows(h, k, C.byref(tc) if tc else None, C.byref(st) if st else None, abi.ptr(out))
        return rc, int(out[0])

    tc, st = structs()
    assert call(-1, tc, st)[0] == abi.ERR_INVALID
    assert call(2, None, st)[0] == abi.ERR_INVALID
    assert call(2, tc, None)[0] == abi.ERR_INVALID
    for f in ("kind", "ns_id", "flags", "thr", "thr_present", "thr_cnt", "ovr_off"):
        bad, st = structs()
        setattr(bad, f, None)
        assert call(2, bad, st)[0] == abi.ERR_INVALID, f
    # ovr_off not from 0 / not monotone / not ending at n_ovr
    n = int(a["ovr_off"][-1])
    for off in ([1, n, n], [0, n + 1, n], [0, 0, n + 1]):
        tc, st = structs(ovr_off=np.array(off, np.int32))
        tc.n_ovr = n
        assert call(2, tc, st)[0] == abi.ERR_INVALID, off
    # a malformed CSR
    nt = int(a["term_off"][-1])
    for off in ([1, nt, nt], [0, nt + 1, nt] if nt else [0, 1, 0], [0, 0, nt + 1]):
        tc, st = structs(term_off=np.array(off, np.int32))
        assert call(2, tc, st)[0] == abi.ERR_INVALID, off
    if len(a["req_op"]):
        tc, st = structs(req_op=np.full(len(a["req_op"]), 9, np.uint8))
        assert call(2, tc, st)[0] == abi.ERR_INVALID
    tc, st = structs(kind=np.array([0, 7], np.uint8))
    assert call(2, tc, st)[0] == abi.ERR_INVALID
    # k = 0: a no-op, null columns allowed
    assert call(0, None, None) == (abi.OK, 0)
    # nothing was appended by the rejected calls
    assert e.words_per_row == 4
    dims = np.zeros(5, np.int32)
    assert L.kt_debug_get_ns_tables(h, abi.ptr(dims), None, None, None) == 0
    assert int(dims[3]) == (snap.m + 31) // 32
    # no status before the call: still none after it; a status held before it is kept and a pass is needed again
    assert e.append_throttle_rows(two) is False
    assert code(lambda: e.evaluate(0, GIVEN)) == abi.ERR_STATE
    m = snap.m + 2
    s2 = copy.copy(snap)
    s2.status = zero_status(snap.R, m)
    for f, v in dict(pack(cols + cols[1:3]), **pack_thr(tcols + tcols[1:3], snap.R)).items():
        setattr(s2, f, v)
    s2.reserved, s2.reserved_present, s2.reserved_cnt = np.zeros((snap.R, m), np.int64), np.zeros(m, np.uint32), np.zeros(m, np.int64)
    s2.normalize()
    e.upload_status(s2)
    e.evaluate(s2.now, abi.EVAL_FRESH_STATUS)
    e.get_changed()
    assert e.append_throttle_rows(two) is False
    assert e.m == m + 2
    assert code(lambda: e.get_changed()) == abi.ERR_STATE
    e.evaluate(0, GIVEN)  # (GIVEN needs the status: still held)
    e.close()
