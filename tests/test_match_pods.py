"""kt_match_pods: the affected throttles of pods given by value (the versions an informer event carries), matched on the device
against the throttle tables as they are, with no resident pod row read or written.

Every answer is compared bit for bit with the columnar oracle's GIVEN_STATUS | SKIP_RECONCILE pass over a snapshot whose pending
rows hold the same labels and namespaces, and with the engine's own pass over those rows uploaded as pending rows (the PENDING
relation of kt_get_match_rows).  Worlds: synthetic ones at several widths (ClusterThrottle-heavy tables with more than two words
per namespace included), the selector edge worlds of test_selector_edges.py, sparse dictionary ids, namespaces out of range,
throttles without terms, broken terms and other throttlers' throttles.  Sizes k = 0, 1, 31, 32, 33 and 10^4 with duplicates."""
import numpy as np
import pytest

from kube_throttler_b200 import KtError, abi, synth
from test_check_rows import assert_same_getters, getters, with_status

pytestmark = pytest.mark.gpu

GIVEN = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE
_variants = set()  # (tpc, b, rt) of the tables kt_match_pods ran on: with_variant picks its kernel from the same tables


def pod_lists(p, rng):
    """row picks of k = 1, 31, 32, 33 and 10^4 pods (duplicates included), both ends, and k = 0"""
    return [np.array([0]), np.array([p - 1]), rng.integers(0, p, size=31), rng.integers(0, p, size=32), rng.integers(0, p, size=33),
            rng.integers(0, p, size=10_000), np.zeros(0, np.int64)]


def pods_of(snap, rows):
    rows = np.asarray(rows, np.int64)
    return np.ascontiguousarray(snap.pending.labels[:, rows]), np.ascontiguousarray(snap.pending.ns_id[rows])


def assert_match(eng, snap, oracle, rows, note="", want=None):
    """match_pods of the pending rows' labels and namespaces == the oracle's pending match bitmap of those rows."""
    if want is None:
        want = oracle.columnar_evaluate(snap, GIVEN, words_per_row=eng.words_per_row).pend_bitmap
    labels, ns = pods_of(snap, rows)
    got = eng.match_pods(labels, ns)
    np.testing.assert_array_equal(got, want[np.asarray(rows, np.int64)], err_msg=note)
    return got, want


def assert_equals_pass(eng, rows, got):
    """The same rows from the engine's own GIVEN_STATUS | SKIP_RECONCILE pass over the uploaded pending table."""
    eng.evaluate(0, GIVEN)
    np.testing.assert_array_equal(got, eng.match_rows(abi.PODS_PENDING, np.asarray(rows, np.int64)))


def record_variant(eng, snap):
    eng.evaluate(snap.now)  # a fused pass: it reports the variant of these tables
    plan = eng.pass_plan()
    _variants.add((plan.tpc, plan.b, plan.rt))


SHAPES = [
    dict(config="C1"),
    dict(config="C2", m=200, n=3000, p=1500),
    dict(config="C3", m=300, n=3000, p=1200),          # ClusterThrottle-heavy: long word lists per namespace
    dict(config="C4", m=500, n=4000, p=1000),
    dict(config="C3", m=1400, n=2000, p=800),          # more than 32 words
    dict(config="C2", m=40, n=70, p=33, R=1),
    dict(config="C2", m=120, n=2000, p=500, R=31, L=12),
    dict(config="C2", m=200, n=2000, p=500, L=3),
]


@pytest.mark.parametrize("kw", SHAPES)
def test_match_equals_oracle_and_pass(kt, oracle, kw):
    kw = dict(kw)
    snap = synth.generate(kw.pop("config"), **kw)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(snap.m)
    with_status(eng, snap, oracle, rng)
    want = None
    for rows in pod_lists(snap.pending.n, rng):  # no pass has run
        got, want = assert_match(eng, snap, oracle, rows, f"{kw} k={len(rows)}", want)
    for rows in pod_lists(snap.pending.n, rng)[:5]:
        got, _ = assert_match(eng, snap, oracle, rows, "", want)
        assert_equals_pass(eng, rows, got)
    record_variant(eng, snap)
    eng.close()


@pytest.mark.parametrize("name", ["fast128_t1_r4", "fast128_t1_r8", "fast128_t2_r4", "fast128_t2_r8", "general_t1_b2", "general_t1_b6",
                                  "general_t2_b2", "general_t2_b6", "limits_r31_l32"])
def test_match_on_edge_worlds(kt, oracle, name):
    """The selector edge worlds, one per kernel variant (6-bit counters at L = 32, sparse and hashed ids, duplicate keys)."""
    from test_selector_edges import world

    snap = world(name, small=True)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    with_status(eng, snap, oracle, np.random.default_rng(7))
    want = None
    for rows in pod_lists(snap.pending.n, np.random.default_rng(8)):
        got, want = assert_match(eng, snap, oracle, rows, name, want)
    assert_equals_pass(eng, np.arange(snap.pending.n), eng.match_pods(*pods_of(snap, np.arange(snap.pending.n))))
    record_variant(eng, snap)
    eng.close()


@pytest.mark.parametrize("mode", ["sparse_keys", "sparse_values"])
def test_match_with_sparse_dictionary_ids(kt, oracle, mode):
    from test_gpu_parity import _remap_label_ids

    snap = synth.generate("C3", m=300, n=3000, p=800)
    if mode == "sparse_keys":
        snap = _remap_label_ids(snap, lambda k: k * 7919 + 70000, lambda v: v * 1009 + 5)
    else:
        snap = _remap_label_ids(snap, lambda k: k, lambda v: v * 1000003 % (1 << 31))
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    with_status(eng, snap, oracle, np.random.default_rng(3))
    want = None
    for rows in pod_lists(snap.pending.n, np.random.default_rng(4)):
        _, want = assert_match(eng, snap, oracle, rows, mode, want)
    eng.close()


def test_namespaces_out_of_range_terms_and_throttlers(kt, oracle):
    """Namespace ids no table row covers (negative, or beyond n_ns and every Throttle's namespace id) give all-zero rows; ids just
    above n_ns match as in the pass (a namespaced Throttle may name a namespace the namespace table does not hold).  The edge
    world carries throttles without terms, broken terms (KT_TERM_POD_INVALID switches the later terms off), selector errors and
    other throttlers' throttles."""
    from test_selector_edges import world

    snap = world("general_t2_b2", small=True)
    rng = np.random.default_rng(21)
    rows = rng.integers(0, snap.pending.n, size=500)
    snap.pending.ns_id[np.unique(rows)[::4]] = snap.n_ns + 1
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    with_status(eng, snap, oracle, rng)
    assert not (snap.thr_flags & abi.THR_RESPONSIBLE).all()
    want = oracle.columnar_evaluate(snap, GIVEN, words_per_row=eng.words_per_row).pend_bitmap
    labels, ns = pods_of(snap, rows)
    got = eng.match_pods(labels, ns)
    np.testing.assert_array_equal(got, want[rows])
    assert_equals_pass(eng, rows, got)
    bad = ns.copy()
    bad[::3] = -1
    bad[1::3] = 1 << 20
    got = eng.match_pods(labels, bad)
    off = (bad < 0) | (bad >= 1 << 20)
    assert not got[off].any()
    np.testing.assert_array_equal(got[~off], want[rows][~off])
    eng.close()


def test_after_table_changes(kt, oracle):
    """After a throttle upload that changes the words per row, and after a namespace relabel -- with no pass in between."""
    snap = synth.generate("C3", m=300, n=3000, p=1500)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(11)
    with_status(eng, snap, oracle, rng)
    rows = rng.integers(0, snap.pending.n, size=700)
    assert_match(eng, snap, oracle, rows, "before")
    snap2 = synth.generate("C3", m=700, n=3000, p=1500, seed=99)
    assert snap2.n_ns == snap.n_ns
    snap2.running, snap2.pending = snap.running, snap.pending
    w0 = eng.words_per_row
    eng.upload_namespaces(snap2.ns_labels)
    eng.upload_throttles(snap2)  # (the status of the old columns is dropped: the match needs none)
    assert eng.words_per_row != w0
    labels, ns = pods_of(snap2, rows)
    got = eng.match_pods(labels, ns)
    with_status(eng, snap2, oracle, rng)
    assert_match(eng, snap2, oracle, rows, "after a throttle upload")
    np.testing.assert_array_equal(got, eng.match_pods(labels, ns))
    # a namespace relabel: the labels of half the namespaces rotate
    nsl = snap2.ns_labels.copy()
    half = np.arange(0, snap2.n_ns, 2)
    nsl[:, half] = np.roll(nsl[:, half], 1, axis=1)
    snap2.ns_labels = np.ascontiguousarray(nsl)
    eng.upload_namespaces(snap2.ns_labels)
    assert_match(eng, snap2, oracle, rows, "after a namespace relabel")
    eng.close()


def test_match_leaves_every_getter_unchanged(kt, oracle):
    snap = synth.generate("C2", m=300, n=3000, p=1500)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(5)
    with_status(eng, snap, oracle, rng)
    eng.evaluate(snap.now)
    before = getters(eng, snap)
    for rows in pod_lists(snap.pending.n, rng):
        eng.match_pods(*pods_of(snap, rows))
    assert_same_getters(before, getters(eng, snap))
    # a fresh engine with tables but no pass: the call does not make the getters answer
    eng2 = kt.Engine(snap.R, snap.L, snap.LN)
    eng2.upload_namespaces(snap.ns_labels)
    eng2.upload_throttles(snap)
    eng2.match_pods(*pods_of(snap, np.arange(50)))
    with pytest.raises(KtError):
        eng2.match_rows(abi.PODS_PENDING, np.arange(1))
    eng2.close()
    eng.close()


def test_arguments_and_state(kt):
    snap = synth.generate("C2", m=200, n=2000, p=700)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    L, h = eng._L, eng._h
    labels, ns = pods_of(snap, np.array([0, 5]))
    out = np.zeros((2, 64), np.uint32)
    assert L.kt_match_pods(h, 2, abi.ptr(labels), abi.ptr(ns), abi.ptr(out)) == abi.ERR_STATE  # no throttles yet
    eng.upload_namespaces(snap.ns_labels)
    eng.upload_throttles(snap)  # throttles only: no pods, status or reservations
    out = np.zeros((2, eng.words_per_row), np.uint32)
    assert L.kt_match_pods(h, 2, abi.ptr(labels), abi.ptr(ns), abi.ptr(out)) == abi.OK
    assert L.kt_match_pods(h, -1, abi.ptr(labels), abi.ptr(ns), abi.ptr(out)) == abi.ERR_INVALID
    assert L.kt_match_pods(h, 2, None, abi.ptr(ns), abi.ptr(out)) == abi.ERR_INVALID
    assert L.kt_match_pods(h, 2, abi.ptr(labels), None, abi.ptr(out)) == abi.ERR_INVALID
    assert L.kt_match_pods(h, 2, abi.ptr(labels), abi.ptr(ns), None) == abi.ERR_INVALID
    assert L.kt_match_pods(h, 0, None, None, None) == abi.OK
    assert L.kt_match_pods(None, 0, None, None, None) == abi.ERR_INVALID
    eng.close()


def test_every_variant_reached():
    """Runs after the tests above: kt_match_pods ran on tables of all 8 (tpc, b, rt) variants with_variant chooses (its kernel is
    the (tpc, b, register rows) of the same tables)."""
    want = {(tpc, 2, rt) for tpc in (1, 2) for rt in (4, 8)} | {(tpc, b, 0) for tpc in (1, 2) for b in (2, 6)}
    assert want <= _variants, sorted(want - _variants)
