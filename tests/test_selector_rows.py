"""kt_update_selector_rows: kind, ns_id, flags and selector terms of listed throttle columns replaced on the device -- deletions
(no terms, flags 0), selector swaps within the resident vocabulary and responsibility flips -- with M and every column's position
kept, without recompiling the selector tables when the new terms fit them.

Two engines hold the same pods, namespaces, throttles, observed status and reservations.  One gets every change as a whole
kt_upload_throttles of the patched spec followed by the same status and reservation uploads; the other gets the same columns
through kt_update_selector_rows, k = 1, 16 or 256 columns a step cut into random batches without a pass in between.  After every
step both must answer bit for bit alike (FRESH, GIVEN and ON_EQUAL passes queued back to back under every forced pass plan, the
status diff, the check summary, kt_check_pending_rows, kt_check_pods, kt_match_pods, kt_reconcile_throttles,
kt_get_match_columns, kt_admit_queue, the check rows), equal the columnar oracle, and hold the namespace masks and word lists
kt_debug_compile_tables builds for the patched spec (the masks wherever the two term-plane counts agree).  Edits that need a new
table row, more term planes or more counter planes than the resident tables have must compile the tables again (recompiled = 1)
and answer the same; the others must not.  Namespace-row, threshold-row and status-row deltas and kt_upload_namespaces are mixed
in.  Worlds: ClusterThrottle-heavy and mixed C3 slices, and selector edge worlds with broken namespace and pod selectors, terms
needing more keys than a pod row holds and both counter-plane widths; both pod row layouts (clustered and not) come from them."""
import ctypes as C

import numpy as np
import pytest

from kube_throttler_b200 import KtError, abi, synth
from test_namespace_rows import PLANS, WORLDS, assert_oracle, assert_same, batches, observe, setup
from test_tables_cpu import compile_tables

pytestmark = pytest.mark.gpu


def columns(snap):
    """Per throttle column: [kind, ns_id, flags, terms]; a term is (term flags, podSelector reqs, namespaceSelector reqs) and a
    requirement (key, op, values)."""
    def reqs(q0, q1):
        return [(int(snap.req_key[q]), int(snap.req_op[q]), tuple(int(v) for v in snap.req_vals[snap.req_val_off[q]:snap.req_val_off[q + 1]]))
                for q in range(q0, q1)]

    return [[int(snap.kind[t]), int(snap.thr_ns[t]), int(snap.thr_flags[t]),
             [(int(snap.term_flags[j]), reqs(snap.pod_req_off[j], snap.pod_req_off[j + 1]), reqs(snap.ns_req_off[j], snap.ns_req_off[j + 1]))
              for j in range(snap.term_off[t], snap.term_off[t + 1])]] for t in range(snap.m)]


def pack(cols):
    """The columns as kind / thr_ns / thr_flags and a selector CSR over them (podSelector requirements first)."""
    terms = [tm for c in cols for tm in c[3]]
    key, op, vals, val_off = [], [], [], [0]

    def push(rs):
        for k, o, vs in rs:
            key.append(k)
            op.append(o)
            vals.extend(vs)
            val_off.append(len(vals))

    pod_off, ns_off = [0], []
    for tm in terms:
        push(tm[1])
        pod_off.append(len(key))
    ns_off.append(len(key))
    for tm in terms:
        push(tm[2])
        ns_off.append(len(key))
    return dict(kind=np.array([c[0] for c in cols], np.uint8), thr_ns=np.array([c[1] for c in cols], np.int32),
                thr_flags=np.array([c[2] for c in cols], np.uint8), term_off=np.cumsum([0] + [len(c[3]) for c in cols]).astype(np.int32),
                term_flags=np.array([tm[0] for tm in terms], np.uint8), pod_req_off=np.array(pod_off, np.int32),
                ns_req_off=np.array(ns_off, np.int32), req_key=np.array(key, np.uint32), req_op=np.array(op, np.uint8),
                req_val_off=np.array(val_off, np.int32), req_vals=np.array(vals, np.uint32))


def set_spec(snap, cols):
    for f, v in pack(cols).items():
        setattr(snap, f, v)
    snap.normalize()


def edit(rng, cols, t, how, tp_pad):
    """Column t edited in place: a deletion, another column's terms (same kind), a responsibility flip, or -- beyond the resident
    tables -- a key no table row has, more terms than tp_pad, or a term with four positive keys."""
    kind, ns, flags, terms = cols[t]
    if how == "delete":
        cols[t] = [kind, ns, 0, []]
    elif how == "swap":
        same = [u for u in range(len(cols)) if cols[u][0] == kind and cols[u][3]] or [t]
        u = int(rng.choice(same))
        cols[t] = [kind, ns, (flags & abi.THR_RESPONSIBLE) | (cols[u][2] & ~abi.THR_RESPONSIBLE), list(cols[u][3])]
    elif how == "flip":
        cols[t] = [kind, ns, flags ^ abi.THR_RESPONSIBLE, terms]
    elif how == "new_key":
        top = max([r[0] for c in cols for tm in c[3] for r in tm[1]] + [0])
        cols[t] = [kind, ns, abi.THR_RESPONSIBLE, [(0, [(top + 1 + t, abi.OP_EXISTS, ())], [])]]
    elif how == "more_terms":
        pool = [tm for c in cols for tm in c[3] if not tm[0]] or [(0, [], [])]
        cols[t] = [kind, ns, abi.THR_RESPONSIBLE, [pool[int(rng.integers(len(pool)))] for _ in range(tp_pad + 1)]]
    elif how == "wide_need":
        keys = sorted({r[0] for c in cols for tm in c[3] for r in tm[1]})[:4]
        cols[t] = [kind, ns, abi.THR_RESPONSIBLE, [(0, [(k, abi.OP_EXISTS, ()) for k in keys], [])]]


def ns_tables_match(kt, eng, snap, where):
    """The resident word lists equal the table compiler's for the patched spec; the masks too when the term planes agree."""
    got, want = eng.ns_tables(), compile_tables(kt, snap)
    n = int(want["nsw_off"][-1])
    np.testing.assert_array_equal(got["nsw_off"], want["nsw_off"], err_msg=where)
    np.testing.assert_array_equal(got["nsw_idx"], want["nsw_idx"][:n], err_msg=where)
    if got["nsmask"].shape == want["nsmask"].shape:
        np.testing.assert_array_equal(got["nsmask"], want["nsmask"], err_msg=where)
    return want


OPS = ["delete", "swap", "flip", "swap", "mixed", "delete", "new_key", "swap", "more_terms", "flip", "wide_need", "reupload_ns", "swap"]


@pytest.mark.parametrize("world", list(WORLDS))
def test_selector_deltas_equal_full_uploads(kt, oracle, world):
    snap = WORLDS[world]()
    rng = np.random.default_rng(sum(map(ord, world)) + 11)
    full, delta = setup(kt, oracle, snap, np.ascontiguousarray(snap.ns_labels), rng)
    m, P = snap.m, snap.pending.n
    probe_rows = rng.integers(0, P, size=min(P, 19))
    probe_idx = rng.choice(m, size=min(m, 9), replace=False).astype(np.int32)
    probe = (probe_rows, probe_idx, snap.pending.labels[:, probe_rows], snap.pending.ns_id[probe_rows].astype(np.int32))
    cols = columns(snap)
    res = compile_tables(kt, snap)
    tp_pad, b_planes = res["TPpad"], res["B"]
    seen = {0: 0, 1: 0}
    for step, op in enumerate(OPS):
        k = min(m, [1, 16, 256][step % 3])
        listed = rng.choice(m, size=k, replace=False).astype(np.int32)
        how = op if op not in ("mixed", "reupload_ns") else "swap"
        n_keys = len({r[0] for c in cols for tm in c[3] for r in tm[1]})
        beyond = how in ("new_key", "more_terms") or (how == "wide_need" and b_planes == 2 and snap.L >= 4 and n_keys >= 4)
        if how == "wide_need" and not beyond:
            how = "swap"
        for t in listed:
            edit(rng, cols, int(t), how, tp_pad)
        set_spec(snap, cols)
        full.upload_throttles(snap)
        full.upload_status(snap)
        full.set_reserved(snap)
        got = set()
        for b in batches(rng, listed):  # several deltas, no pass in between
            got.add(delta.update_selector_rows(b, pack([cols[t] for t in b])))
        if beyond:
            assert True in got, (world, step, op)
            res = compile_tables(kt, snap)
            tp_pad, b_planes = res["TPpad"], res["B"]
        else:
            assert got == {False}, (world, step, op)
        seen[int(beyond)] += 1
        if op == "mixed":  # namespace-row, threshold-row and status-row deltas on both engines after the selector delta
            nsr = np.array([0], np.int32)
            snap.ns_labels[:, 0] = snap.ns_labels[:, min(1, snap.n_ns - 1)]
            sc = np.array([t for t in rng.permutation(m) if snap.ovr_off[t] == snap.ovr_off[t + 1]][:4], np.int32)
            snap.thr[:, sc] = rng.integers(0, 4000, size=(snap.R, len(sc)))
            snap.status["used"][:, sc] = rng.integers(0, 4000, size=(snap.R, len(sc)))
            snap.normalize()
            thr = dict(thr=snap.thr[:, sc], thr_present=snap.thr_present[sc], thr_cnt=snap.thr_cnt[sc], ovr_off=np.zeros(len(sc) + 1, np.int32),
                       ovr_begin=[], ovr_end=[], ovr_flags=[], ovr_thr=np.zeros((snap.R, 0)), ovr_present=[], ovr_cnt=[])
            for e in (full, delta):
                e.update_namespace_rows(snap.n_ns, nsr, snap.ns_labels[:, nsr])
                e.update_threshold_rows(sc, thr)
                e.update_status_rows(sc, {f: (v[:, sc] if v.ndim == 2 else v[sc]) for f, v in snap.status.items()})
        if op == "reupload_ns":  # a whole namespace upload after the deltas: the tables compiled from the patched spec
            for e in (full, delta):
                e.upload_namespaces(snap.ns_labels)
            res = compile_tables(kt, snap)
            tp_pad, b_planes = res["TPpad"], res["B"]
        where = f"{world} step {step} {op} k={k}"
        ns_tables_match(kt, delta, snap, where)
        assert_oracle(delta, snap, oracle, where)
        plan = PLANS[step % len(PLANS)]
        assert_same(observe(full, snap, plan, probe), observe(delta, snap, plan, probe), where + f" plan {plan}")
    assert seen[0] >= 8 and seen[1] >= 2, seen
    full.close()
    delta.close()


def test_argument_and_state_errors(kt):
    snap = synth.generate("C3", m=40, n=200, p=50, n_ns=6).normalize()
    e = kt.Engine(snap.R, snap.L, snap.LN)
    L, h = e._L, e._h
    cols = columns(snap)
    idx = np.array([1, 2], np.int32)
    two = pack([cols[1], cols[2]])

    def code(fn):
        with pytest.raises(KtError) as ex:
            fn()
        return ex.value.code

    assert code(lambda: e.update_selector_rows(idx, two)) == abi.ERR_STATE  # before kt_upload_throttles
    e.upload_namespaces(snap.ns_labels)
    e.upload_throttles(snap)
    assert e.update_selector_rows(idx, two) is False  # the same columns: they fit
    for bad in ([snap.m, 0], [-1, 0], [3, 3]):  # out of range, negative, duplicate
        assert code(lambda: e.update_selector_rows(np.array(bad, np.int32), two)) == abi.ERR_INVALID
    a = {f: np.ascontiguousarray(v) for f, v in two.items()}

    def structs(**over):
        x = dict(a, **over)
        tc = abi.ThrottleCols(abi.ptr(x["kind"]), abi.ptr(x["thr_ns"]), abi.ptr(x["thr_flags"]), None, None, None, None, 0, None, None, None,
                              None, None, None)
        st = abi.SelectorTable(int(x["term_off"][-1]), int(x["req_key"].shape[0]), int(x["req_vals"].shape[0]),
                               *(abi.ptr(x[f]) for f in ("term_off", "term_flags", "pod_req_off", "ns_req_off", "req_key", "req_op", "req_val_off", "req_vals")))
        return tc, st

    def call(k, ix, tc, st):
        out = np.full(1, 7, np.int32)
        rc = L.kt_update_selector_rows(h, k, abi.ptr(ix), C.byref(tc) if tc else None, C.byref(st) if st else None, abi.ptr(out))
        return rc, int(out[0])

    tc, st = structs()
    assert call(2, idx, tc, st) == (abi.OK, 0)
    assert call(-1, idx, tc, st)[0] == abi.ERR_INVALID
    assert call(2, None, tc, st)[0] == abi.ERR_INVALID
    assert call(2, idx, None, st)[0] == abi.ERR_INVALID
    assert call(2, idx, tc, None)[0] == abi.ERR_INVALID
    for f in ("kind", "ns_id", "flags"):
        bad, st = structs()
        setattr(bad, f, None)
        assert call(2, idx, bad, st)[0] == abi.ERR_INVALID, f
    for f in ("thr", "thr_present", "thr_cnt", "ovr_off", "ovr_begin", "ovr_thr"):  # the threshold columns are another call's
        bad, st = structs()
        setattr(bad, f, abi.ptr(np.zeros(4, np.int64)))
        assert call(2, idx, bad, st)[0] == abi.ERR_INVALID, f
        assert call(0, None, bad, None)[0] == abi.ERR_INVALID, f
    # a malformed CSR: term_off not from 0 / not monotone / not ending at n_terms, a requirement range out of bounds, a bad op
    n = int(a["term_off"][-1])
    for off in ([1, n, n], [0, n + 1, n] if n else [0, 1, 0], [0, 0, n + 1]):
        tc, st = structs(term_off=np.array(off, np.int32))
        assert call(2, idx, tc, st)[0] == abi.ERR_INVALID, off
    if n:
        tc, st = structs(pod_req_off=np.full(n + 1, len(a["req_key"]) + 5, np.int32))
        assert call(2, idx, tc, st)[0] == abi.ERR_INVALID
    if len(a["req_op"]):
        tc, st = structs(req_op=np.full(len(a["req_op"]), 9, np.uint8))
        assert call(2, idx, tc, st)[0] == abi.ERR_INVALID
    tc, st = structs(kind=np.array([0, 7], np.uint8))
    assert call(2, idx, tc, st)[0] == abi.ERR_INVALID
    # k = 0: a no-op, null columns allowed
    assert call(0, None, None, None) == (abi.OK, 0)
    # the status held before the call is kept; a pass is needed again before the getters that read one
    snap.status = {f: np.zeros((snap.R, snap.m) if f in ("calc_thr", "used") else snap.m) for f in
                   ("calculated", "calc_thr", "calc_present", "calc_cnt", "used", "used_present", "used_cnt", "throttled")}
    snap.normalize()
    e.upload_status(snap)
    e.evaluate(snap.now, abi.EVAL_FRESH_STATUS)
    e.get_changed()
    e.update_selector_rows(np.array([0], np.int32), pack([[cols[0][0], cols[0][1], 0, []]]))
    assert code(lambda: e.get_changed()) == abi.ERR_STATE
    e.evaluate(0, abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE)  # (GIVEN needs the status: still held)
    e.close()
