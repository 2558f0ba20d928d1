"""kt_update_namespace_rows: namespace rows replaced (and the namespace count grown) on the device, without recompiling the
selector tables.

Two engines hold the same pods, throttles and observed status.  One gets every namespace change as a whole kt_upload_namespaces;
the other gets the same final rows through row deltas, in random batches, several of them without a pass in between.  Steps:
relabels that flip ClusterThrottle namespaceSelectors both ways (rows mixed from other namespaces' labels), deletions (every slot
empty), creations that grow the count -- by one, and past the allocation -- with pods already in the new namespaces, re-creation,
and kt_upload_throttles after a run of deltas.  After every step both engines must answer bit for bit alike (FRESH and GIVEN
passes queued back to back with a forced pass plan, the status diff, the check summary, kt_check_pending_rows, kt_check_pods,
kt_match_pods, kt_reconcile_throttles, kt_get_match_columns, kt_admit_queue, the check rows), equal the columnar oracle, and hold
the namespace masks and word lists kt_debug_compile_tables builds for the same rows.  Worlds: ClusterThrottle-heavy C3 slices
(several words per namespace) and selector edge worlds with broken namespace and pod selectors."""
import ctypes as C

import numpy as np
import pytest

from kube_throttler_b200 import KtError, abi, synth
from test_partial_passes import observed_status
from test_selector_edges import world as edge_world_named
from test_tables_cpu import compile_tables

pytestmark = pytest.mark.gpu

FRESH = abi.EVAL_FRESH_STATUS
GIVEN = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE
PLANS = [(0, 0), (512, abi.PLAN_DECIDE_QUAD), (512, abi.PLAN_DECIDE_PER_POD), (768, abi.PLAN_DECIDE_QUAD), (768, abi.PLAN_DECIDE_PER_POD)]


def c3_world(**kw):
    return synth.generate("C3", **kw)


WORLDS = {
    "c3_cluster_heavy": lambda: c3_world(m=700, n=3000, p=800, n_ns=40, cluster_frac=0.9),
    "c3_mixed": lambda: c3_world(m=300, n=2500, p=600, n_ns=30),
    "edge_general_t2_b2": lambda: edge_world_named("general_t2_b2", small=True),
    "edge_fast256_t2_r4": lambda: edge_world_named("fast256_t2_r4", small=True),
    "edge_general_t2_b6": lambda: edge_world_named("general_t2_b6", small=True),
}


def setup(kt, oracle, snap, rows, rng):
    """The full-upload engine and the row-delta engine on the first `rows` namespace rows, with an observed status."""
    snap.ns_labels = np.ascontiguousarray(rows)
    fresh = oracle.columnar_evaluate(snap, FRESH, words_per_row=synth_words(snap))
    snap.status = observed_status(fresh, snap, rng)
    snap.normalize()
    out = []
    for _ in range(2):
        e = kt.Engine(snap.R, snap.L, snap.LN)
        e.upload_namespaces(snap.ns_labels)
        e.upload_throttles(snap)
        e.upload_status(snap)
        e.set_reserved(snap)
        e.upload_pods(abi.PODS_RUNNING, snap.running)
        e.upload_pods(abi.PODS_PENDING, snap.pending)
        e.set_sparse_check(1 << 16)
        out.append(e)
    return out


def synth_words(snap):
    w = (snap.m + 31) // 32
    return max(4, (w + 3) // 4 * 4)


def observe(eng, snap, plan, probe):
    """Everything the namespace rows feed, in one list of arrays."""
    rows, idx, labels, ns = probe
    P = snap.pending.n
    out = []
    eng.set_pass_plan(*plan)
    eng.evaluate(snap.now, FRESH)
    eng.evaluate(0, GIVEN)  # queued right behind: starts its first phase while the first pass decides
    r = eng.download()
    out += [r.run_bitmap, r.pend_bitmap, r.codes, r.admit]
    out += list(eng.check_summary(0, P))
    eng.evaluate(snap.now, FRESH)
    r = eng.download()
    out += [r.run_bitmap, r.used, r.used_present, r.used_cnt, r.throttled, r.calc_thr, r.calc_present, r.calc_cnt, r.codes, r.admit]
    out += list(eng.get_changed())
    eng.evaluate(0, GIVEN | abi.EVAL_ON_EQUAL)
    r = eng.download()
    out += [r.codes, r.admit]
    eng.set_pass_plan()
    for on_equal in (False, True):
        out += list(eng.check_pending_rows(rows, on_equal))
    out.append(eng.match_pods(labels, ns))
    out += list(eng.check_pods(labels, snap.pending.req[:, rows], snap.pending.present[rows], ns))
    st, off, rrows = eng.reconcile_throttles(snap.now, idx)
    out += [st.used, st.used_present, st.used_cnt, st.throttled, st.calc_thr, off, rrows]
    eng.evaluate(0, GIVEN)
    for kind in (abi.PODS_RUNNING, abi.PODS_PENDING):
        out += [x for x in eng.match_columns(kind, idx) if x is not None]
    out += list(eng.get_check_rows(np.arange(P)))
    out += list(eng.admit_queue(0, P))
    return out


def assert_same(a, b, where):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        np.testing.assert_array_equal(np.asarray(x), np.asarray(y), err_msg=f"{where}: output {i}")


def assert_oracle(eng, snap, oracle, where, modes=(FRESH, GIVEN)):
    for flags in modes:
        eng.evaluate(snap.now if flags == FRESH else 0, flags)
        got = eng.download()
        want = oracle.columnar_evaluate(snap, flags, words_per_row=eng.words_per_row)
        np.testing.assert_array_equal(got.pend_bitmap, want.pend_bitmap, err_msg=where)
        np.testing.assert_array_equal(got.codes, want.codes, err_msg=where)
        np.testing.assert_array_equal(got.admit, want.admit, err_msg=where)
        if flags == FRESH:
            live = (snap.thr_flags & abi.THR_RESPONSIBLE) != 0
            np.testing.assert_array_equal(got.run_bitmap, want.run_bitmap, err_msg=where)
            np.testing.assert_array_equal(got.used[:, live], want.used[:, live], err_msg=where)


def assert_tables(kt, eng, snap, where):
    """The resident namespace masks and word lists equal the table compiler's for the same rows."""
    got, want = eng.ns_tables(), compile_tables(kt, snap)
    np.testing.assert_array_equal(got["nsmask"], want["nsmask"], err_msg=where)
    np.testing.assert_array_equal(got["nsw_off"], want["nsw_off"], err_msg=where)
    n = int(want["nsw_off"][-1])
    np.testing.assert_array_equal(got["nsw_idx"], want["nsw_idx"][:n], err_msg=where)
    counts = np.diff(want["nsw_off"])
    assert got["max_ns_words"] == (int(counts.max()) if counts.size else 0), where
    return got["max_ns_words"], n


def new_rows(rng, pool, k):
    """k namespace rows [LN][k]: copies of rows in the pool, rows mixed slot by slot from two of them, and empty rows."""
    LN, n = pool.shape
    out = np.full((LN, k), abi.LABEL_EMPTY, np.int64)
    for i in range(k):
        r = rng.random()
        if r < 0.15 or n == 0:
            continue  # deleted: no label at all
        a, b = pool[:, rng.integers(n)], pool[:, rng.integers(n)]
        out[:, i] = a if r < 0.5 else np.where(rng.random(LN) < 0.5, a, b)
        out[rng.random(LN) < 0.15, i] = abi.LABEL_EMPTY
    return out


def batches(rng, idx):
    idx = rng.permutation(idx)
    out, i = [], 0
    while i < len(idx):
        k = int(rng.integers(1, len(idx) - i + 1))
        out.append(idx[i:i + k])
        i += k
    return out


@pytest.mark.parametrize("world", list(WORLDS))
def test_row_deltas_equal_full_uploads(kt, oracle, world):
    snap = WORLDS[world]()
    rng = np.random.default_rng(sum(map(ord, world)))
    pool = np.ascontiguousarray(snap.ns_labels)
    LN, n_all = pool.shape
    # the last namespaces are created during the test; some pods already live there (ids past the namespace count)
    n0 = max(1, n_all - max(2, n_all // 3))
    grow_to = n_all + 2 * n_all + 5
    # (Throttles name namespaces that exist from the start: the oracle's view of a Throttle whose namespace has no row is not
    # what this test is about)
    snap.thr_ns = np.where(snap.thr_ns >= n0, snap.thr_ns % n0, snap.thr_ns).astype(np.int32)
    for pods in (snap.running, snap.pending):
        move = rng.random(pods.n) < 0.15
        pods.ns_id[move] = rng.integers(n0, grow_to, size=int(move.sum()))
    cur = pool[:, :n0].copy()
    full, delta = setup(kt, oracle, snap, cur, rng)
    P = snap.pending.n
    probe_rows = rng.integers(0, P, size=min(P, 19))
    probe_idx = rng.choice(snap.m, size=min(snap.m, 9), replace=False).astype(np.int32)
    probe_ns = np.concatenate([snap.pending.ns_id[probe_rows][:-2], [grow_to - 1, grow_to + 3]]).astype(np.int32)  # and out of range
    probe = (probe_rows, probe_idx, snap.pending.labels[:, probe_rows], probe_ns)
    words_seen = {assert_tables(kt, delta, snap, f"{world} start")}
    ops = ["relabel", "grow1", "relabel_many", "grow_far", "delete", "delete_all", "relabel", "reupload", "recreate"]
    for step, op in enumerate(ops):
        n = cur.shape[1]
        if op == "grow1":  # one new namespace, listed
            n_new, listed = n + 1, np.array([n])
        elif op == "grow_far":  # past the allocation; only some of the new rows listed (the others are label-less)
            n_new = grow_to
            listed = np.union1d(rng.choice(np.arange(n, n_new), size=(n_new - n) // 2, replace=False), rng.integers(0, n, size=2))
        elif op == "relabel":
            n_new, listed = n, rng.choice(n, size=min(n, int(rng.choice([1, 2, 3]))), replace=False)
        elif op == "relabel_many":
            n_new, listed = n, rng.choice(n, size=max(1, n // 2), replace=False)
        elif op == "delete":
            n_new, listed = n, rng.choice(n, size=min(n, 4), replace=False)
        elif op == "delete_all":  # only the Throttles' words are left: the longest word list shrinks
            n_new, listed = n, np.arange(n)
        else:  # reupload / recreate: relabel a few, then (reupload) the throttles again
            n_new, listed = n, rng.choice(n, size=min(n, 5), replace=False)
        nxt = np.full((LN, n_new), abi.LABEL_EMPTY, np.int64)
        nxt[:, :n] = cur
        vals = new_rows(rng, pool, len(listed))
        if op in ("delete", "delete_all"):
            vals[:] = abi.LABEL_EMPTY
        if op == "recreate":
            vals = pool[:, rng.integers(0, n_all, size=len(listed))]
        nxt[:, listed] = vals
        cur = nxt
        snap.ns_labels = np.ascontiguousarray(cur)
        full.upload_namespaces(snap.ns_labels)
        for b in batches(rng, np.asarray(listed)):  # several deltas, no pass in between
            delta.update_namespace_rows(n_new, b.astype(np.int32), cur[:, b])
        if op == "reupload":
            for e in (full, delta):
                e.upload_throttles(snap)
                e.upload_status(snap)
                e.set_reserved(snap)
        where = f"{world} step {step} {op}"
        words_seen.add(assert_tables(kt, delta, snap, where))
        assert_oracle(delta, snap, oracle, where)
        plan = PLANS[step % len(PLANS)]
        assert_same(observe(full, snap, plan, probe), observe(delta, snap, plan, probe), where + f" plan {plan}")
    if world == "c3_cluster_heavy":  # several words per namespace, and word lists that changed on the way
        assert len(words_seen) > 1 and max(words_seen)[0] > 2, words_seen
    full.close()
    delta.close()


def test_deltas_before_the_throttles(kt, oracle):
    """Before kt_upload_throttles the call only stores the rows: the tables compiled later are the ones of those rows."""
    snap = synth.generate("C3", m=200, n=1000, p=300, n_ns=12, cluster_frac=0.8)
    rng = np.random.default_rng(5)
    pool = np.ascontiguousarray(snap.ns_labels)
    e = kt.Engine(snap.R, snap.L, snap.LN)
    e.upload_namespaces(np.ascontiguousarray(pool[:, :8]))
    rows = new_rows(rng, pool, 6)
    e.update_namespace_rows(12, np.array([1, 9, 11, 3], np.int32), rows[:, :4])
    e.update_namespace_rows(12, np.array([0], np.int32), rows[:, 4:5])
    want = np.full_like(pool, abi.LABEL_EMPTY)
    want[:, :8] = pool[:, :8]
    want[:, [1, 9, 11, 3]] = rows[:, :4]
    want[:, 0] = rows[:, 4]
    snap.ns_labels = want
    e.upload_throttles(snap)
    assert_tables(kt, e, snap, "before throttles")
    e.set_reserved(snap)
    e.upload_pods(abi.PODS_RUNNING, snap.running)
    e.upload_pods(abi.PODS_PENDING, snap.pending)
    assert_oracle(e, snap, oracle, "before throttles", (FRESH,))
    e.close()


def test_argument_and_state_errors(kt, oracle):
    snap = synth.generate("C3", m=60, n=300, p=80, n_ns=6, cluster_frac=0.7)
    e = kt.Engine(snap.R, snap.L, snap.LN)
    L, h = e._L, e._h
    LN = snap.LN
    lab = np.full((LN, 2), abi.LABEL_EMPTY, np.int64)
    idx = np.array([1, 2], np.int32)

    def code(fn):
        with pytest.raises(KtError) as ex:
            fn()
        return ex.value.code

    e.upload_namespaces(snap.ns_labels)
    n = snap.n_ns
    for bad in ([n, 0], [-1, 0], [3, 3]):  # out of range, negative, duplicate
        assert code(lambda: e.update_namespace_rows(n, np.array(bad, np.int32), lab)) == abi.ERR_INVALID
    assert code(lambda: e.update_namespace_rows(n - 1, idx, lab)) == abi.ERR_INVALID  # the count never shrinks
    assert L.kt_update_namespace_rows(h, n, -1, abi.ptr(idx), abi.ptr(lab)) == abi.ERR_INVALID
    assert L.kt_update_namespace_rows(h, n, 2, None, abi.ptr(lab)) == abi.ERR_INVALID
    assert L.kt_update_namespace_rows(h, n, 2, abi.ptr(idx), None) == abi.ERR_INVALID
    e.upload_throttles(snap)
    e.set_reserved(snap)
    e.upload_pods(abi.PODS_RUNNING, snap.running)
    e.upload_pods(abi.PODS_PENDING, snap.pending)
    e.evaluate(snap.now, FRESH)
    before = e.download()
    # k = 0 with the same count: a no-op (null arrays allowed), the last pass still answers
    assert L.kt_update_namespace_rows(h, n, 0, None, None) == abi.OK
    np.testing.assert_array_equal(e.download().pend_bitmap, before.pend_bitmap)
    # a delta needs a pass before the getters that read one
    e.update_namespace_rows(n, idx, lab)
    assert code(lambda: e.download()) == abi.ERR_STATE
    # k = 0 with a larger count: label-less rows appended
    e.update_namespace_rows(n + 3, np.zeros(0, np.int32), np.zeros((LN, 0), np.int64))
    rows = np.full((LN, n + 3), abi.LABEL_EMPTY, np.int64)
    rows[:, :n] = snap.ns_labels
    rows[:, idx] = lab
    snap.ns_labels = rows
    assert_tables(kt, e, snap, "k = 0 growth")
    assert_oracle(e, snap, oracle, "k = 0 growth", (FRESH,))
    e.close()
