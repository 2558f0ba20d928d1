"""kt_reconcile_throttles: reconcile(key) of listed throttles on the device.

Every answer is compared bit for bit with the columnar oracle's FRESH_STATUS pass (status columns of the listed throttles, and
their matched running rows transposed) and with the engine's own full reconcile pass over the same state (kt_get_reconcile_rows /
kt_get_match_columns).  The call must work on rows and tables as they are -- right after uploads, row deltas and table
re-uploads, with no pass in between -- and must leave every getter's answer, and the next pass, as they would be without it."""
import numpy as np
import pytest

from kube_throttler_b200 import abi, synth
from test_match_columns import numpy_columns

pytestmark = pytest.mark.gpu

FRESH = abi.EVAL_FRESH_STATUS
REC_ONLY = abi.EVAL_FRESH_STATUS | abi.EVAL_SKIP_CHECK
STATUS_FIELDS = ("used", "used_present", "used_cnt", "throttled", "calc_thr", "calc_present", "calc_cnt", "override_active")
_variants = set()  # (tpc, b, rt) of the tables the keyed calls ran on: with_variant picks the same for k_keyed_rows as for the pass


def index_lists(m, rng):
    """k = 1 at both ends, random subsets with duplicates, every throttle, and k = 0"""
    return [np.array([0]), np.array([m - 1]), rng.integers(0, m, size=max(1, m // 7)), np.concatenate([rng.integers(0, m, size=5)] * 2),
            np.arange(m), np.zeros(0, np.int64)]


def assert_keyed(eng, snap, oracle, idx, note=""):
    """The keyed answer for idx == the oracle's FRESH_STATUS pass over the snapshot as it is now."""
    want = oracle.columnar_evaluate(snap, FRESH, words_per_row=eng.words_per_row)
    got, off, rows = eng.reconcile_throttles(snap.now, idx)
    idx = np.asarray(idx, np.int64)
    for f in STATUS_FIELDS:
        w = getattr(want, f)
        np.testing.assert_array_equal(getattr(got, f), w[..., idx], err_msg=f"{note} {f}")
    w_off, w_rows, _ = numpy_columns(want.run_bitmap, snap.m, idx)
    np.testing.assert_array_equal(off, w_off, err_msg=note)
    np.testing.assert_array_equal(rows, w_rows, err_msg=note)
    return got, off, rows


def assert_equals_full_pass(eng, snap, idx, keyed):
    """The same columns from a full reconcile pass of the engine itself."""
    got, off, rows = keyed
    eng.evaluate(snap.now, REC_ONLY)
    full = eng.get_reconcile_rows(np.asarray(idx, np.int32))
    for f in STATUS_FIELDS:
        np.testing.assert_array_equal(getattr(got, f), getattr(full, f), err_msg=f)
    f_off, f_rows, _ = eng.match_columns(abi.PODS_RUNNING, idx)
    np.testing.assert_array_equal(off, f_off)
    np.testing.assert_array_equal(rows, f_rows)


def getters(eng, snap, with_status):
    """Everything a getter answers after the last pass."""
    d = eng.download()
    out = {f: getattr(d, f).copy() for f in STATUS_FIELDS + ("run_bitmap", "pend_bitmap", "codes", "admit")}
    if with_status:
        out["changed"] = eng.get_changed()
    idx = np.arange(snap.m)
    out["cols_run"] = eng.match_columns(abi.PODS_RUNNING, idx)
    out["cols_pend"] = eng.match_columns(abi.PODS_PENDING, idx)
    return out


def assert_same_getters(a, b):
    assert a.keys() == b.keys()
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, tuple):
            for u, v in zip(x, y):
                np.testing.assert_array_equal(u, v, err_msg=k)
        else:
            np.testing.assert_array_equal(x, y, err_msg=k)


def record_variant(eng, snap):
    eng.evaluate(snap.now)  # a fused pass: it reports the variant
    plan = eng.pass_plan()
    _variants.add((plan.tpc, plan.b, plan.rt))


SHAPES = [
    dict(config="C1"),
    dict(config="C2", m=200, n=5000, p=700),
    dict(config="C3", m=300, n=6000, p=800),
    dict(config="C4", m=500, n=8000, p=1000),
    dict(config="C2", m=333, n=7777, p=1111, sort_by_namespace=False),  # rows in arrival order
    dict(config="C2", m=40, n=70, p=33, R=1),                            # ragged: a partial tile, a partial last word
    dict(config="C3", m=200, n=3000, p=800, R=5),
    dict(config="C2", m=150, n=4000, p=600, R=12),
    dict(config="C2", m=120, n=3000, p=500, R=31, L=12),
    dict(config="C2", m=200, n=3000, p=500, L=3),
    dict(config="C2", m=200, n=3000, p=500, L=12),
    dict(config="C4", m=2500, n=5000, p=900),                            # k = M: 79 listed words, accumulators in HBM
]


@pytest.mark.parametrize("kw", SHAPES)
def test_keyed_equals_oracle_and_full_pass(kt, oracle, kw):
    kw = dict(kw)
    snap = synth.generate(kw.pop("config"), **kw)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    rng = np.random.default_rng(snap.m)
    for idx in index_lists(snap.m, rng):  # no pass has run: the row offsets are translated by the call itself
        assert_keyed(eng, snap, oracle, idx, "before any pass")
    for idx in index_lists(snap.m, rng)[:4]:
        assert_equals_full_pass(eng, snap, idx, assert_keyed(eng, snap, oracle, idx))
    record_variant(eng, snap)
    eng.close()


@pytest.mark.parametrize("name", ["fast128_t1_r4", "fast128_t1_r8", "fast128_t2_r4", "fast128_t2_r8", "general_t1_b2", "general_t1_b6",
                                  "general_t2_b2", "general_t2_b6", "limits_r31_l32"])
def test_keyed_on_edge_worlds(kt, oracle, name):
    """The selector edge worlds, one per kernel variant (6-bit counters at L = 32, sparse and hashed ids, duplicate keys)."""
    from test_selector_edges import world

    snap = world(name, small=True)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    rng = np.random.default_rng(7)
    for idx in index_lists(snap.m, rng):
        assert_keyed(eng, snap, oracle, idx, name)
    record_variant(eng, snap)
    eng.close()


@pytest.mark.parametrize("mode", ["sparse_keys", "sparse_values"])
def test_keyed_with_sparse_dictionary_ids(kt, oracle, mode):
    from test_gpu_parity import _remap_label_ids

    snap = synth.generate("C3", m=300, n=6000, p=800)
    if mode == "sparse_keys":
        snap = _remap_label_ids(snap, lambda k: k * 7919 + 70000, lambda v: v * 1009 + 5)
    else:
        snap = _remap_label_ids(snap, lambda k: k, lambda v: v * 1000003 % (1 << 31))
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    for idx in index_lists(snap.m, np.random.default_rng(3)):
        assert_keyed(eng, snap, oracle, idx, mode)
    eng.close()


def test_keyed_after_row_deltas_and_table_uploads_without_a_pass(kt, oracle):
    snap = synth.generate("C3", m=300, n=6000, p=800)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    eng.evaluate(snap.now)
    rng = np.random.default_rng(11)
    idx = rng.integers(0, snap.m, size=20)
    assert_keyed(eng, snap, oracle, idx)
    # row deltas: pods move namespace, finish, get relabelled -- no pass in between
    rows = np.sort(rng.choice(snap.running.n, size=500, replace=False)).astype(np.int64)
    delta = snap.running.rows(rows)
    delta.ns_id = ((delta.ns_id + 1 + rng.integers(0, snap.n_ns - 1, size=len(rows))) % snap.n_ns).astype(np.int32)
    delta.flags = (delta.flags ^ np.where(rng.random(len(rows)) < 0.3, abi.POD_NOT_FINISHED, 0)).astype(np.uint32)
    delta.labels = np.ascontiguousarray(np.roll(delta.labels, 1, axis=1))
    eng.update_pod_rows(abi.PODS_RUNNING, rows, delta)
    snap.running.ns_id[rows] = delta.ns_id
    snap.running.flags[rows] = delta.flags
    snap.running.labels[:, rows] = delta.labels
    assert_keyed(eng, snap, oracle, idx, "after a row delta")
    # new namespaces and throttle columns (other selectors and thresholds), uploaded without a pass
    snap2 = synth.generate("C3", m=400, n=6000, p=800, seed=99)
    assert snap2.n_ns == snap.n_ns
    snap2.running, snap2.pending = snap.running, snap.pending
    eng.upload_namespaces(snap2.ns_labels)
    eng.upload_throttles(snap2)
    assert_keyed(eng, snap2, oracle, rng.integers(0, snap2.m, size=30), "after a table upload")
    assert_keyed(eng, snap2, oracle, np.arange(snap2.m), "after a table upload, every column")
    eng.close()


def test_keyed_leaves_every_getter_and_the_next_pass_unchanged(kt, oracle):
    from test_partial_passes import observed_status

    snap = synth.generate("C2", m=300, n=6000, p=900)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    fresh = oracle.columnar_evaluate(snap, FRESH, words_per_row=eng.words_per_row)
    snap.status = observed_status(fresh, snap, np.random.default_rng(2))
    snap.normalize()
    eng.upload_status(snap)
    eng.evaluate(snap.now)
    before = getters(eng, snap, True)
    rng = np.random.default_rng(5)
    for idx in index_lists(snap.m, rng):
        eng.reconcile_throttles(snap.now + 10**12, idx)  # another clock: nothing of it may show in the getters
    assert_same_getters(before, getters(eng, snap, True))
    # a row delta, a keyed call, then the next pass: as without the keyed call
    rows = np.sort(rng.choice(snap.running.n, size=300, replace=False)).astype(np.int64)
    delta = snap.running.rows(rows)
    delta.ns_id = ((delta.ns_id + 1) % snap.n_ns).astype(np.int32)
    eng.update_pod_rows(abi.PODS_RUNNING, rows, delta)
    snap.running.ns_id[rows] = delta.ns_id
    eng.reconcile_throttles(snap.now, np.arange(snap.m))
    eng.evaluate(snap.now)
    after = eng.download()
    want = oracle.columnar_evaluate(snap, FRESH, words_per_row=eng.words_per_row)
    for f in STATUS_FIELDS + ("run_bitmap", "pend_bitmap", "codes", "admit"):
        np.testing.assert_array_equal(getattr(after, f), getattr(want, f), err_msg=f)
    eng.close()


def test_cap_arguments_and_state(kt):
    snap = synth.generate("C2", m=200, n=5000, p=700)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    L, h = eng._L, eng._h
    idx = np.arange(snap.m, dtype=np.int32)
    off = np.zeros(snap.m + 1, np.int64)
    rows = np.zeros(8, np.int64)
    z = np.zeros
    out = abi.PassResult(4, z((snap.R, snap.m), np.int64), z(snap.m, np.uint32), z(snap.m, np.int64), z(snap.m, np.uint32),
                         z((snap.R, snap.m), np.int64), z(snap.m, np.uint32), z(snap.m, np.int64), z(snap.m, np.uint8),
                         z((0, 1), np.uint32), z((0, 1), np.uint32), z((0, 1), np.uint32), z(0, np.uint8))
    rec = out.reconcile_out()
    import ctypes as C

    call = lambda k, ix, o, r, cap: L.kt_reconcile_throttles(h, snap.now, k, abi.ptr(ix), C.byref(rec), abi.ptr(o), abi.ptr(r), cap)
    assert call(snap.m, idx, off, rows, 8) == abi.ERR_STATE  # no throttles yet
    eng.upload_snapshot(snap)
    _, want_off, want_rows = eng.reconcile_throttles(snap.now, idx)
    total = int(want_off[-1])
    assert total > 1
    rows = np.full(total - 1, -7, np.int64)  # one row too little room: off is written, the rows are not
    assert call(snap.m, idx, off, rows, total - 1) == abi.OK
    np.testing.assert_array_equal(off, want_off)
    assert (rows == -7).all()
    rows = np.zeros(total, np.int64)
    assert call(snap.m, idx, off, rows, total) == abi.OK
    np.testing.assert_array_equal(rows, want_rows)
    for bad in (np.array([-1], np.int32), np.array([snap.m], np.int32), np.array([0, snap.m + 5], np.int32)):
        assert call(len(bad), bad, off, rows, total) == abi.ERR_INVALID
    assert call(1, idx, None, rows, total) == abi.ERR_INVALID
    assert call(1, idx, off, rows, -1) == abi.ERR_INVALID
    off[:] = 5
    assert call(0, None, off, None, 0) == abi.OK
    assert off[0] == 0 and off[1] == 5
    eng.close()


def test_every_variant_reached():
    """Runs after the tests above: the keyed kernel ran on tables of all 8 (tpc, b, rt) variants with_variant chooses -- the fast
    family (register label rows, rt 4 and 8) and the general family (rt 0, 2- and 6-bit counters), each with 1 and 2 term planes."""
    want = {(tpc, 2, rt) for tpc in (1, 2) for rt in (4, 8)} | {(tpc, b, 0) for tpc in (1, 2) for b in (2, 6)}
    assert _variants == want, sorted(_variants)
