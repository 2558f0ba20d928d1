"""kt_check_pending_rows: PreFilter of listed pending rows on the device, without a pass over the pending table.

Every answer is compared bit for bit with the columnar oracle's GIVEN_STATUS | SKIP_RECONCILE pass (the listed rows of its pending
match bitmap, codes and admit bits) and with the engine's own pass over the same state (kt_get_match_rows / kt_get_check_rows),
for both values of isThrottledOnEqual.  The call must work on rows, tables, statuses and reservations as they are -- right after
uploads, row deltas, status and reservation changes and table re-uploads, with no pass in between -- and must leave every getter's
answer, and the next pass, as they would be without it."""
import numpy as np
import pytest

from kube_throttler_b200 import KtError, abi, synth
from test_partial_passes import observed_status, random_reserved, set_reserved

pytestmark = pytest.mark.gpu

FRESH = abi.EVAL_FRESH_STATUS
GIVEN = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE
_variants = set()  # (tpc, b, rt) of the tables the listed-row check ran on: with_variant picks its kernel from the same tables


def row_lists(p, rng):
    """one row at both ends, a few, duplicates, every row, and k = 0"""
    return [np.array([0]), np.array([p - 1]), rng.integers(0, p, size=max(1, min(p, 9))), np.concatenate([rng.integers(0, p, size=4)] * 3),
            np.arange(p), np.zeros(0, np.int64)]


def with_status(eng, snap, oracle, rng):
    """Upload the snapshot with an observed status that lags behind the truth and random reservations."""
    eng.upload_snapshot(snap)
    fresh = oracle.columnar_evaluate(snap, FRESH, words_per_row=eng.words_per_row)
    snap.status = observed_status(fresh, snap, rng)
    snap.normalize()
    eng.upload_status(snap)
    set_reserved(eng, snap, random_reserved(snap, rng))


def assert_rows(eng, snap, oracle, rows, on_equal, note=""):
    """The listed-row answer == the oracle's GIVEN_STATUS pass over the snapshot as it is now."""
    flags = GIVEN | (abi.EVAL_ON_EQUAL if on_equal else 0)
    want = oracle.columnar_evaluate(snap, flags, words_per_row=eng.words_per_row)
    words, codes, admit = eng.check_pending_rows(rows, on_equal)
    rows = np.asarray(rows, np.int64)
    np.testing.assert_array_equal(words, want.pend_bitmap[rows], err_msg=f"{note} words on_equal={on_equal}")
    np.testing.assert_array_equal(codes, want.codes[rows], err_msg=f"{note} codes on_equal={on_equal}")
    np.testing.assert_array_equal(admit, want.admit[rows], err_msg=f"{note} admit on_equal={on_equal}")
    return words, codes, admit


def assert_equals_pass(eng, snap, rows, on_equal, got):
    """The same rows from the engine's own GIVEN_STATUS | SKIP_RECONCILE pass."""
    eng.evaluate(0, GIVEN | (abi.EVAL_ON_EQUAL if on_equal else 0))
    words, codes, admit = got
    np.testing.assert_array_equal(words, eng.match_rows(abi.PODS_PENDING, rows))
    c, a = eng.get_check_rows(rows)
    np.testing.assert_array_equal(codes, c)
    np.testing.assert_array_equal(admit, a)


def record_variant(eng, snap):
    eng.evaluate(snap.now)  # a fused pass: it reports the variant of these tables
    plan = eng.pass_plan()
    _variants.add((plan.tpc, plan.b, plan.rt))


SHAPES = [
    dict(config="C1"),
    dict(config="C2", m=200, n=3000, p=1500),
    dict(config="C3", m=300, n=3000, p=1200),
    dict(config="C4", m=500, n=4000, p=1000),
    dict(config="C2", m=333, n=3000, p=1111, sort_by_namespace=False),  # rows in arrival order
    dict(config="C2", m=40, n=70, p=33, R=1),                            # ragged: a partial tile, a partial last word
    dict(config="C2", m=150, n=2000, p=600, R=12),
    dict(config="C2", m=120, n=2000, p=500, R=31, L=12),
    dict(config="C2", m=200, n=2000, p=500, L=3),
]


@pytest.mark.parametrize("kw", SHAPES)
def test_rows_equal_oracle_and_pass(kt, oracle, kw):
    kw = dict(kw)
    snap = synth.generate(kw.pop("config"), **kw)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(snap.m)
    with_status(eng, snap, oracle, rng)
    P = snap.pending.n
    for on_equal in (False, True):
        for rows in row_lists(P, rng):  # no pass has run: the row offsets are translated by the call itself
            assert_rows(eng, snap, oracle, rows, on_equal, "before any pass")
    for on_equal in (False, True):
        for rows in row_lists(P, rng)[:5]:
            assert_equals_pass(eng, snap, rows, on_equal, assert_rows(eng, snap, oracle, rows, on_equal))
    record_variant(eng, snap)
    eng.close()


@pytest.mark.parametrize("name", ["fast128_t1_r4", "fast128_t1_r8", "fast128_t2_r4", "fast128_t2_r8", "general_t1_b2", "general_t1_b6",
                                  "general_t2_b2", "general_t2_b6", "limits_r31_l32"])
def test_rows_on_edge_worlds(kt, oracle, name):
    """The selector edge worlds, one per kernel variant (6-bit counters at L = 32, sparse and hashed ids, duplicate keys)."""
    from test_selector_edges import world

    snap = world(name, small=True)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(7)
    with_status(eng, snap, oracle, rng)
    for on_equal in (False, True):
        for rows in row_lists(snap.pending.n, rng):
            assert_rows(eng, snap, oracle, rows, on_equal, name)
    record_variant(eng, snap)
    eng.close()


@pytest.mark.parametrize("mode", ["sparse_keys", "sparse_values"])
def test_rows_with_sparse_dictionary_ids(kt, oracle, mode):
    from test_gpu_parity import _remap_label_ids

    snap = synth.generate("C3", m=300, n=3000, p=800)
    if mode == "sparse_keys":
        snap = _remap_label_ids(snap, lambda k: k * 7919 + 70000, lambda v: v * 1009 + 5)
    else:
        snap = _remap_label_ids(snap, lambda k: k, lambda v: v * 1000003 % (1 << 31))
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(3)
    with_status(eng, snap, oracle, rng)
    for on_equal in (False, True):
        for rows in row_lists(snap.pending.n, rng):
            assert_rows(eng, snap, oracle, rows, on_equal, mode)
    eng.close()


@pytest.mark.parametrize("mode", [abi.ROW_ORDER_BY_NAMESPACE, abi.ROW_ORDER_AS_GIVEN])
def test_rows_are_caller_rows_in_either_row_order(kt, oracle, mode):
    """Pending rows stored sorted by namespace (or as given): the listed rows are the caller's, in and out."""
    snap = synth.generate("C2", m=300, n=3000, p=2000, sort_by_namespace=False)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.set_row_order(abi.PODS_PENDING, mode)
    rng = np.random.default_rng(13)
    with_status(eng, snap, oracle, rng)
    clustered, _ = eng.row_order(abi.PODS_PENDING)
    assert bool(clustered) == (mode == abi.ROW_ORDER_BY_NAMESPACE)
    for on_equal in (False, True):
        for rows in row_lists(snap.pending.n, rng):
            assert_equals_pass(eng, snap, rows, on_equal, assert_rows(eng, snap, oracle, rows, on_equal, f"order {mode}"))
    eng.close()


def test_rows_after_deltas_status_reservations_and_tables_without_a_pass(kt, oracle):
    snap = synth.generate("C3", m=300, n=3000, p=1500)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(11)
    with_status(eng, snap, oracle, rng)
    eng.evaluate(0, GIVEN)
    rows = rng.integers(0, snap.pending.n, size=40)
    assert_rows(eng, snap, oracle, rows, False)
    # row deltas: pods move namespace, get relabelled and new requests -- no pass in between
    d_rows = np.sort(rng.choice(snap.pending.n, size=300, replace=False)).astype(np.int64)
    delta = snap.pending.rows(d_rows)
    delta.ns_id = ((delta.ns_id + 1 + rng.integers(0, snap.n_ns - 1, size=len(d_rows))) % snap.n_ns).astype(np.int32)
    delta.labels = np.ascontiguousarray(np.roll(delta.labels, 1, axis=1))
    delta.req = np.ascontiguousarray(delta.req[:, ::-1])
    eng.update_pod_rows(abi.PODS_PENDING, d_rows, delta)
    snap.pending.ns_id[d_rows] = delta.ns_id
    snap.pending.labels[:, d_rows] = delta.labels
    snap.pending.req[:, d_rows] = delta.req
    for on_equal in (False, True):
        assert_rows(eng, snap, oracle, np.concatenate([rows, d_rows[:50]]), on_equal, "after a row delta")
    # another observed status, other reservations, then none
    fresh = oracle.columnar_evaluate(snap, FRESH, words_per_row=eng.words_per_row)
    snap.status = observed_status(fresh, snap, rng)
    snap.normalize()
    eng.upload_status(snap)
    assert_rows(eng, snap, oracle, d_rows, False, "after a status upload")
    set_reserved(eng, snap, random_reserved(snap, rng))
    assert_rows(eng, snap, oracle, d_rows, True, "after new reservations")
    set_reserved(eng, snap, (None, None, None))
    assert_rows(eng, snap, oracle, d_rows, False, "after the reservations were cleared")
    # new throttle columns: other selectors and thresholds, and more words per row (Wp changes) -- uploaded without a pass
    snap2 = synth.generate("C3", m=700, n=3000, p=1500, seed=99)
    assert snap2.n_ns == snap.n_ns
    snap2.running, snap2.pending = snap.running, snap.pending
    w0 = eng.words_per_row
    eng.upload_namespaces(snap2.ns_labels)
    eng.upload_throttles(snap2)
    assert eng.words_per_row != w0
    with pytest.raises(KtError):
        eng.check_pending_rows(rows)  # a throttle upload drops the status of the old columns
    fresh = oracle.columnar_evaluate(snap2, FRESH, words_per_row=eng.words_per_row)
    snap2.status = observed_status(fresh, snap2, rng)
    snap2.reserved = snap2.reserved_present = snap2.reserved_cnt = None
    snap2.normalize()
    eng.upload_status(snap2)
    for on_equal in (False, True):
        for r in row_lists(snap2.pending.n, rng):
            assert_rows(eng, snap2, oracle, r, on_equal, "after a table upload")
    eng.close()


def getters(eng, snap):
    """Everything a getter answers after the last pass."""
    d = eng.download()
    out = {f: getattr(d, f).copy() for f in ("used", "used_present", "used_cnt", "throttled", "calc_thr", "calc_present", "calc_cnt",
                                             "override_active", "run_bitmap", "pend_bitmap", "codes", "admit")}
    out["changed"] = eng.get_changed()
    idx = np.arange(snap.m)
    out["cols_run"] = eng.match_columns(abi.PODS_RUNNING, idx)
    out["cols_pend"] = eng.match_columns(abi.PODS_PENDING, idx)
    rows = np.arange(snap.pending.n)
    out["check_rows"] = eng.get_check_rows(rows)
    out["match_rows"] = eng.match_rows(abi.PODS_PENDING, rows)
    return out


def assert_same_getters(a, b):
    assert a.keys() == b.keys()
    for k in a:
        x, y = a[k], b[k]
        for u, v in (zip(x, y) if isinstance(x, tuple) else [(x, y)]):
            np.testing.assert_array_equal(u, v, err_msg=k)


def test_rows_leave_every_getter_and_the_next_pass_unchanged(kt, oracle):
    snap = synth.generate("C2", m=300, n=3000, p=1500)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(5)
    with_status(eng, snap, oracle, rng)
    eng.evaluate(snap.now)  # a fused FRESH pass: status columns, diff, bitmaps, codes of its own
    before = getters(eng, snap)
    for on_equal in (False, True):
        for rows in row_lists(snap.pending.n, rng):
            eng.check_pending_rows(rows, on_equal)
    assert_same_getters(before, getters(eng, snap))
    # a row delta, the listed-row call, then the next pass: as without the call
    d_rows = np.sort(rng.choice(snap.pending.n, size=200, replace=False)).astype(np.int64)
    delta = snap.pending.rows(d_rows)
    delta.ns_id = ((delta.ns_id + 1) % snap.n_ns).astype(np.int32)
    eng.update_pod_rows(abi.PODS_PENDING, d_rows, delta)
    snap.pending.ns_id[d_rows] = delta.ns_id
    with pytest.raises(KtError):
        eng.get_check_rows(d_rows)  # no pass since the delta: the getters fail ...
    eng.check_pending_rows(np.arange(snap.pending.n))
    with pytest.raises(KtError):
        eng.get_check_rows(d_rows)  # ... and the call does not make them answer
    eng.evaluate(0, GIVEN)
    after = eng.download()
    want = oracle.columnar_evaluate(snap, GIVEN, words_per_row=eng.words_per_row)
    for f in ("pend_bitmap", "codes", "admit"):
        np.testing.assert_array_equal(getattr(after, f), getattr(want, f), err_msg=f)
    eng.close()


def test_arguments_and_state(kt, oracle):
    snap = synth.generate("C2", m=200, n=2000, p=700)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    L, h = eng._L, eng._h
    rows = np.array([0, 5], np.int64)
    out = np.zeros((2, 64), np.uint32)
    call = lambda flags, k, r: L.kt_check_pending_rows(h, flags, k, abi.ptr(r), abi.ptr(out), None, None)
    assert call(0, 2, rows) == abi.ERR_STATE  # no throttles yet
    snap.status = snap.reserved = snap.reserved_present = snap.reserved_cnt = None
    eng.upload_snapshot(snap)
    assert call(0, 2, rows) == abi.ERR_STATE  # no observed status yet
    with_status(eng, snap, oracle, np.random.default_rng(1))
    assert call(0, 2, rows) == abi.OK
    assert call(abi.EVAL_ON_EQUAL, 2, rows) == abi.OK
    for bad in (abi.EVAL_GIVEN_STATUS, abi.EVAL_SKIP_RECONCILE, abi.EVAL_SKIP_CHECK, 16):
        assert call(bad, 2, rows) == abi.ERR_INVALID
    for bad in (np.array([-1], np.int64), np.array([snap.pending.n], np.int64), np.array([0, snap.pending.n + 5], np.int64)):
        assert call(0, len(bad), bad) == abi.ERR_INVALID
    assert L.kt_check_pending_rows(h, 0, 1, None, None, None, None) == abi.ERR_INVALID
    assert L.kt_check_pending_rows(h, 0, 0, None, None, None, None) == abi.OK
    # each output alone
    want_w, want_c, want_a = eng.check_pending_rows(rows)
    adm = np.zeros(2, np.uint8)
    assert L.kt_check_pending_rows(h, 0, 2, abi.ptr(rows), None, None, abi.ptr(adm)) == abi.OK
    np.testing.assert_array_equal(adm, want_a)
    codes = np.zeros_like(want_c)
    assert L.kt_check_pending_rows(h, 0, 2, abi.ptr(rows), None, abi.ptr(codes), None) == abi.OK
    np.testing.assert_array_equal(codes, want_c)
    eng.close()


def test_every_variant_reached():
    """Runs after the tests above: the listed-row check ran on tables of all 8 (tpc, b, rt) variants with_variant chooses -- the
    fast family (register label rows, rt 4 and 8) and the general family (rt 0, 2- and 6-bit counters), each with 1 and 2 term
    planes.  (The check keeps no per-resource registers: its kernel is the (tpc, b, register rows) of the same tables.)"""
    want = {(tpc, 2, rt) for tpc in (1, 2) for rt in (4, 8)} | {(tpc, b, 0) for tpc in (1, 2) for b in (2, 6)}
    assert _variants == want, sorted(_variants)
