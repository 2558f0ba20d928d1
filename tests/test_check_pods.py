"""kt_check_pods: PreFilter of pods given by value on the device, with no pending row read and no pass over the pending table.

Every answer is compared bit for bit with the columnar oracle's GIVEN_STATUS | SKIP_RECONCILE pass over a pending table that
holds exactly the given pods (its match bitmap, codes and admit bits), and with the engine's own pass over the same pods
uploaded as pending rows (the scratch-row path the host layer used before), for both values of isThrottledOnEqual.  The call
must work on tables, statuses and reservations as they are -- right after uploads, column deltas and table re-uploads, with no
pass in between and with no pod table at all -- and must leave every getter's answer, and the next pass, as they would be
without it."""
import copy

import numpy as np
import pytest

from kube_throttler_b200 import KtError, abi, synth
from test_check_rows import SHAPES, assert_same_getters, getters, with_status
from test_partial_passes import observed_status, random_reserved, set_reserved

pytestmark = pytest.mark.gpu

FRESH = abi.EVAL_FRESH_STATUS
GIVEN = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE
_variants = set()  # (tpc, b, rt) of the tables the by-value check ran on: with_variant picks its kernel from the same tables


def pod_lists(pend, rng):
    """pods taken from the snapshot's pending rows: one, a few, duplicates, every row, and k = 0"""
    p = pend.n
    picks = [np.array([0]), np.array([p - 1]), rng.integers(0, p, size=max(1, min(p, 9))), np.concatenate([rng.integers(0, p, size=4)] * 3),
             np.arange(p), np.zeros(0, np.int64)]
    return [pend.rows(r) for r in picks]


def assert_pods(eng, snap, oracle, pods, on_equal, note="", scratch_pass=False):
    """check_pods == the oracle's GIVEN_STATUS pass over a pending table holding exactly `pods`; optionally also == the engine's
    own pass over the same pods uploaded as its pending rows (which replaces the engine's pending table)."""
    flags = GIVEN | (abi.EVAL_ON_EQUAL if on_equal else 0)
    s = copy.copy(snap)
    s.pending = pods
    want = oracle.columnar_evaluate(s, flags, words_per_row=eng.words_per_row)
    got = eng.check_pods(pods.labels, pods.req, pods.present, pods.ns_id, on_equal)
    for name, g, w in zip(("words", "codes", "admit"), got, (want.pend_bitmap, want.codes, want.admit)):
        np.testing.assert_array_equal(g, w[:pods.n], err_msg=f"{note} {name} on_equal={on_equal}")
    if scratch_pass and pods.n:
        eng.upload_pods(abi.PODS_PENDING, pods)
        eng.evaluate(0, flags)
        d = eng.download()
        for name, g, w in zip(("words", "codes", "admit"), got, (d.pend_bitmap, d.codes, d.admit)):
            np.testing.assert_array_equal(g, w, err_msg=f"{note} {name} against the pass, on_equal={on_equal}")
    return got


def record_variant(eng, snap):
    eng.evaluate(snap.now)  # a fused pass: it reports the variant of these tables
    plan = eng.pass_plan()
    _variants.add((plan.tpc, plan.b, plan.rt))


@pytest.mark.parametrize("kw", SHAPES)
def test_pods_equal_oracle_and_pass(kt, oracle, kw):
    kw = dict(kw)
    snap = synth.generate(kw.pop("config"), **kw)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(snap.m)
    with_status(eng, snap, oracle, rng)
    record_variant(eng, snap)
    for on_equal in (False, True):
        for pods in pod_lists(snap.pending, rng):
            assert_pods(eng, snap, oracle, pods, on_equal, str(kw), scratch_pass=True)
    eng.close()


@pytest.mark.parametrize("name", ["fast128_t1_r4", "fast128_t1_r8", "fast128_t2_r4", "fast128_t2_r8", "general_t1_b2", "general_t1_b6",
                                  "general_t2_b2", "general_t2_b6", "limits_r31_l32"])
def test_pods_on_edge_worlds(kt, oracle, name):
    """The selector edge worlds, one per kernel variant (6-bit counters at L = 32, sparse and hashed ids, duplicate keys, broken
    podSelectors that shadow the later terms)."""
    from test_selector_edges import world

    snap = world(name, small=True)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(7)
    with_status(eng, snap, oracle, rng)
    record_variant(eng, snap)
    for on_equal in (False, True):
        for pods in pod_lists(snap.pending, rng):
            assert_pods(eng, snap, oracle, pods, on_equal, name, scratch_pass=True)
    eng.close()


@pytest.mark.parametrize("mode", ["sparse_keys", "sparse_values"])
def test_pods_with_sparse_dictionary_ids(kt, oracle, mode):
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
        for pods in pod_lists(snap.pending, rng):
            assert_pods(eng, snap, oracle, pods, on_equal, mode)
    eng.close()


def test_pods_value_edges_and_foreign_namespaces(kt, oracle):
    """Negative, zero and large requests, presence bits that hide a value, and namespace ids the tables do not cover (negative,
    at n_ns, far beyond): such a pod gets an all-zero row with admit = 1, as in the pass."""
    snap = synth.generate("C2", m=200, n=2000, p=600)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(17)
    with_status(eng, snap, oracle, rng)
    pods = snap.pending.rows(rng.integers(0, snap.pending.n, size=300))
    edges = np.array([-(1 << 40), -7, -1, 0, 1, 3, 1 << 40], np.int64)
    pods.req[:] = rng.choice(edges, size=pods.req.shape)
    pods.present[:] = rng.integers(0, 1 << snap.R, size=pods.n).astype(np.uint32) | (rng.integers(0, 2, size=pods.n).astype(np.uint32) << 31)
    pods.ns_id[::7] = -1
    pods.ns_id[1::11] = snap.n_ns
    pods.ns_id[2::13] = 1 << 20
    for on_equal in (False, True):
        words, codes, admit = assert_pods(eng, snap, oracle, pods, on_equal, "value edges")
        out = (pods.ns_id < 0) | (pods.ns_id >= (1 << 20))
        assert not words[out].any() and not codes[out].any() and admit[out].all()
    assert_pods(eng, snap, oracle, pods, False, "value edges", scratch_pass=True)
    eng.close()


def test_pods_clusterthrottle_heavy(kt, oracle):
    """Long namespace word lists: ClusterThrottles whose namespaceSelectors reach most namespaces."""
    snap = synth.generate("C3", m=800, n=3000, p=1000, cluster_frac=0.9)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(23)
    with_status(eng, snap, oracle, rng)
    assert (snap.kind == abi.KIND_CLUSTERTHROTTLE).sum() > snap.m // 4
    for on_equal in (False, True):
        for pods in pod_lists(snap.pending, rng)[2:5]:
            assert_pods(eng, snap, oracle, pods, on_equal, "cluster-heavy", scratch_pass=True)
    eng.close()


def test_pods_without_pod_tables_and_after_column_deltas(kt, oracle):
    """No pod table uploaded at all; then status and reservation column deltas and a table re-upload take effect at once."""
    snap = synth.generate("C3", m=300, n=3000, p=1500)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(11)
    eng.upload_namespaces(snap.ns_labels)
    eng.upload_throttles(snap)
    fresh = oracle.columnar_evaluate(snap, FRESH)
    snap.status = observed_status(fresh, snap, rng)
    snap.reserved = snap.reserved_present = snap.reserved_cnt = None
    snap.normalize()
    eng.upload_status(snap)
    pods = snap.pending.rows(rng.integers(0, snap.pending.n, size=200))
    for on_equal in (False, True):
        assert_pods(eng, snap, oracle, pods, on_equal, "no pod tables")
    set_reserved(eng, snap, random_reserved(snap, rng))
    assert_pods(eng, snap, oracle, pods, True, "after new reservations")
    # column deltas of status and reservations, no pass in between
    idx = np.sort(rng.choice(snap.m, size=40, replace=False)).astype(np.int32)
    fresh2 = oracle.columnar_evaluate(snap, FRESH, words_per_row=eng.words_per_row)
    st2 = observed_status(fresh2, snap, rng)
    cols = {f: np.ascontiguousarray(np.asarray(st2[f])[..., idx]) for f in st2}
    eng.update_status_rows(idx, cols)
    for f in cols:
        snap.status[f][..., idx] = cols[f]
    res, pres, cnt = random_reserved(snap, rng)
    eng.update_reserved_rows(idx, res[:, idx], pres[idx], cnt[idx])
    snap.reserved[:, idx], snap.reserved_present[idx], snap.reserved_cnt[idx] = res[:, idx], pres[idx], cnt[idx]
    for on_equal in (False, True):
        assert_pods(eng, snap, oracle, pods, on_equal, "after column deltas")
    # new throttle columns (Wp changes): the status of the old columns is gone until the next upload
    snap2 = synth.generate("C3", m=700, n=3000, p=1500, seed=99)
    eng.upload_namespaces(snap2.ns_labels)
    eng.upload_throttles(snap2)
    with pytest.raises(KtError):
        eng.check_pods(pods.labels, pods.req, pods.present, pods.ns_id)
    fresh = oracle.columnar_evaluate(snap2, FRESH, words_per_row=eng.words_per_row)
    snap2.status = observed_status(fresh, snap2, rng)
    snap2.reserved = snap2.reserved_present = snap2.reserved_cnt = None
    snap2.normalize()
    eng.upload_status(snap2)
    for on_equal in (False, True):
        for p in pod_lists(snap2.pending, rng):
            assert_pods(eng, snap2, oracle, p, on_equal, "after a table upload")
    eng.close()


def test_pods_leave_every_getter_and_the_next_pass_unchanged(kt, oracle):
    snap = synth.generate("C2", m=300, n=3000, p=1500)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(5)
    with_status(eng, snap, oracle, rng)
    eng.set_pass_plan(threads=512)  # a forced plan: the pass poisons every output it writes before it writes it
    eng.evaluate(snap.now)
    before = getters(eng, snap)
    for on_equal in (False, True):
        for pods in pod_lists(snap.pending, rng):
            eng.check_pods(pods.labels, pods.req, pods.present, pods.ns_id, on_equal)
    assert_same_getters(before, getters(eng, snap))
    # a row delta, the call, then the next pass: as without the call
    d_rows = np.sort(rng.choice(snap.pending.n, size=200, replace=False)).astype(np.int64)
    delta = snap.pending.rows(d_rows)
    delta.ns_id = ((delta.ns_id + 1) % snap.n_ns).astype(np.int32)
    eng.update_pod_rows(abi.PODS_PENDING, d_rows, delta)
    snap.pending.ns_id[d_rows] = delta.ns_id
    with pytest.raises(KtError):
        eng.get_check_rows(d_rows)  # no pass since the delta: the getters fail ...
    eng.check_pods(delta.labels, delta.req, delta.present, delta.ns_id)
    with pytest.raises(KtError):
        eng.get_check_rows(d_rows)  # ... and the call does not make them answer
    eng.evaluate(0, GIVEN)
    after = eng.download()
    want = oracle.columnar_evaluate(snap, GIVEN, words_per_row=eng.words_per_row)
    for f in ("pend_bitmap", "codes", "admit"):
        np.testing.assert_array_equal(getattr(after, f), getattr(want, f), err_msg=f)
    eng.set_pass_plan()
    eng.close()


def test_arguments_and_state(kt, oracle):
    snap = synth.generate("C2", m=200, n=2000, p=700)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    L, h = eng._L, eng._h
    pods = snap.pending.rows(np.array([0, 5]))
    out = np.zeros((2, 64), np.uint32)
    lab, req, pres, ns = (abi.ptr(np.ascontiguousarray(x)) for x in (pods.labels, pods.req, pods.present, pods.ns_id))
    call = lambda flags, k, *cols: L.kt_check_pods(h, flags, k, *(cols or (lab, req, pres, ns)), abi.ptr(out), None, None)
    assert call(0, 2) == abi.ERR_STATE  # no throttles yet
    snap.status = snap.reserved = snap.reserved_present = snap.reserved_cnt = None
    eng.upload_snapshot(snap)
    assert call(0, 2) == abi.ERR_STATE  # no observed status yet
    with_status(eng, snap, oracle, np.random.default_rng(1))
    assert call(0, 2) == abi.OK
    assert call(abi.EVAL_ON_EQUAL, 2) == abi.OK
    for bad in (abi.EVAL_GIVEN_STATUS, abi.EVAL_SKIP_RECONCILE, abi.EVAL_SKIP_CHECK, 16):
        assert call(bad, 2) == abi.ERR_INVALID
    assert call(0, -1) == abi.ERR_INVALID
    for i in range(4):  # each input column missing
        cols = [lab, req, pres, ns]
        cols[i] = None
        assert call(0, 2, *cols) == abi.ERR_INVALID
    assert L.kt_check_pods(h, 0, 0, None, None, None, None, None, None, None) == abi.OK
    # each output alone
    want_w, want_c, want_a = eng.check_pods(pods.labels, pods.req, pods.present, pods.ns_id)
    adm = np.zeros(2, np.uint8)
    assert L.kt_check_pods(h, 0, 2, lab, req, pres, ns, None, None, abi.ptr(adm)) == abi.OK
    np.testing.assert_array_equal(adm, want_a)
    codes = np.zeros_like(want_c)
    assert L.kt_check_pods(h, 0, 2, lab, req, pres, ns, None, abi.ptr(codes), None) == abi.OK
    np.testing.assert_array_equal(codes, want_c)
    eng.close()


def test_every_variant_reached():
    """Runs after the tests above: the by-value check ran on tables of all 8 (tpc, b, rt) variants with_variant chooses."""
    want = {(tpc, 2, rt) for tpc in (1, 2) for rt in (4, 8)} | {(tpc, b, 0) for tpc in (1, 2) for b in (2, 6)}
    assert _variants == want, sorted(_variants)
