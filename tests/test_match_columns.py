"""kt_get_match_columns: the match relation transposed per throttle on the device (affectedPods from the throttles' side).

Every answer is compared with a numpy transposition of what kt_get_match_bitmap / kt_get_check deliver for the same pass, and
the relation itself with the columnar oracle's."""
import numpy as np
import pytest

from kube_throttler_b200 import abi, synth

pytestmark = pytest.mark.gpu


def numpy_columns(bitmap, m, idx, codes=None):
    """(off, rows, codes) from the pod-major bitmap [n][W] (and codes [n][2W]) the way kt_get_match_columns defines them."""
    idx = np.asarray(idx, np.int64)
    bits = (bitmap[:, idx >> 5] >> (idx & 31).astype(np.uint32)) & 1  # [n][k]
    off = np.zeros(len(idx) + 1, np.int64)
    rows, cs = [], []
    for j, t in enumerate(idx):
        r = np.flatnonzero(bits[:, j]).astype(np.int64)
        rows.append(r)
        if codes is not None:
            cs.append(((codes[r, t >> 4] >> np.uint32(2 * (t & 15))) & 3).astype(np.uint8))
        off[j + 1] = off[j] + len(r)
    cat = lambda v, dt: np.concatenate(v).astype(dt) if v else np.zeros(0, dt)
    return off, cat(rows, np.int64), (cat(cs, np.uint8) if codes is not None else None)


def index_lists(m, rng):
    """all throttles, random subsets with duplicates, k = 1 and k = 0"""
    return [np.arange(m), rng.integers(0, m, size=max(1, m // 3)), np.concatenate([rng.integers(0, m, size=7)] * 2),
            np.array([m - 1]), np.array([0]), np.zeros(0, np.int64)]


def check_engine(eng, m, want=None, seed=0):
    """Every index list of both kinds against the engine's own dense downloads (and the oracle's relation, when given)."""
    got = eng.download()
    if want is not None:
        np.testing.assert_array_equal(got.run_bitmap, want.run_bitmap)
        np.testing.assert_array_equal(got.pend_bitmap, want.pend_bitmap)
        np.testing.assert_array_equal(got.codes, want.codes)
    rng = np.random.default_rng(seed)
    for idx in index_lists(m, rng):
        for kind, bitmap, codes in ((abi.PODS_RUNNING, got.run_bitmap, None), (abi.PODS_PENDING, got.pend_bitmap, got.codes)):
            off, rows, cs = eng.match_columns(kind, idx)
            w_off, w_rows, w_cs = numpy_columns(bitmap, m, idx, codes)
            np.testing.assert_array_equal(off, w_off)
            np.testing.assert_array_equal(rows, w_rows)
            if codes is not None:
                np.testing.assert_array_equal(cs, w_cs)
            else:
                assert cs is None
    return got


def evaluate(kt, oracle, snap, flags=abi.EVAL_FRESH_STATUS):
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    eng.evaluate(snap.now, flags)
    want = oracle.columnar_evaluate(snap, flags, words_per_row=eng.words_per_row)
    return eng, want


@pytest.mark.parametrize("kw", [
    dict(config="C1"),
    dict(config="C2", m=200, n=5000, p=700),
    dict(config="C2", m=1000, n=20000, p=2000),
    dict(config="C3", m=300, n=6000, p=800),
    dict(config="C4", m=500, n=8000, p=1000),
    dict(config="C2", m=333, n=7777, p=1111, sort_by_namespace=False),   # rows in arrival order
    dict(config="C3", m=1000, n=20000, p=2000, sort_by_namespace=False),
    dict(config="C2", m=40, n=70, p=33, R=1),                             # ragged: a partial block, a partial last word
    dict(config="C3", m=200, n=3000, p=800, R=5),
    dict(config="C2", m=150, n=4000, p=600, R=12),
    dict(config="C4", m=2500, n=5000, p=900),                             # k > 1024: the scan of the lengths walks ranges
])
def test_columns_equal_the_transposed_bitmap(kt, oracle, kw):
    kw = dict(kw)
    snap = synth.generate(kw.pop("config"), **kw)
    eng, want = evaluate(kt, oracle, snap)
    got = check_engine(eng, snap.m, want)
    assert got.run_bitmap.any() and got.pend_bitmap.any()
    eng.close()


@pytest.mark.parametrize("mode", ["sparse_keys", "sparse_values"])
def test_columns_with_sparse_dictionary_ids(kt, oracle, mode):
    from test_gpu_parity import _remap_label_ids

    snap = synth.generate("C3", m=300, n=6000, p=800)
    if mode == "sparse_keys":
        snap = _remap_label_ids(snap, lambda k: k * 7919 + 70000, lambda v: v * 1009 + 5)
    else:
        snap = _remap_label_ids(snap, lambda k: k, lambda v: v * 1000003 % (1 << 31))
    eng, want = evaluate(kt, oracle, snap)
    check_engine(eng, snap.m, want)
    eng.close()


def test_columns_after_a_row_delta_that_moves_pods_to_another_namespace(kt, oracle):
    """A pod that changes namespace leaves words of its old namespace's list behind; the next pass clears them."""
    snap = synth.generate("C3", m=300, n=6000, p=800)
    eng, want = evaluate(kt, oracle, snap)
    check_engine(eng, snap.m, want)
    rng = np.random.default_rng(5)
    rows = np.sort(rng.choice(snap.running.n, size=400, replace=False)).astype(np.int64)
    delta = snap.running.rows(rows)
    delta.ns_id = ((delta.ns_id + 1 + rng.integers(0, snap.n_ns - 1, size=len(rows))) % snap.n_ns).astype(np.int32)
    eng.update_pod_rows(abi.PODS_RUNNING, rows, delta)
    snap.running.ns_id[rows] = delta.ns_id
    eng.evaluate(snap.now)
    want = oracle.columnar_evaluate(snap, words_per_row=eng.words_per_row)
    check_engine(eng, snap.m, want, seed=1)
    eng.close()


def test_columns_carry_the_codes_of_queue_admission(kt, oracle):
    from test_oracle_admission import admission_world

    snap = admission_world(oracle, "C2", m=200, n=4000, p=1500)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    eng.admit_queue(100, 1200, 0)
    want, _, _ = oracle.columnar_admit_queue(snap, 100, 1200, 0, words_per_row=eng.words_per_row)
    got = check_engine(eng, snap.m)
    np.testing.assert_array_equal(got.codes, want.codes)
    _, _, cs = eng.match_columns(abi.PODS_PENDING, np.arange(snap.m))
    assert (cs != 0).any()  # the rejected pods' codes are in the columns
    eng.close()


def test_cap_arguments_and_call_order(kt):
    snap = synth.generate("C2", m=200, n=5000, p=700)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    L, h = eng._L, eng._h
    idx = np.arange(snap.m, dtype=np.int32)
    off = np.zeros(snap.m + 1, np.int64)
    rows = np.zeros(8, np.int64)
    assert L.kt_get_match_columns(h, abi.PODS_RUNNING, snap.m, abi.ptr(idx), abi.ptr(off), abi.ptr(rows), None, 8) == abi.ERR_STATE
    eng.evaluate(snap.now)
    want_off, want_rows, want_cs = eng.match_columns(abi.PODS_PENDING, idx)
    total = int(want_off[-1])
    assert total > 1
    # one row too little room: off is written, the rows are not
    rows = np.full(total - 1, -7, np.int64)
    codes = np.full(total - 1, 9, np.uint8)
    assert L.kt_get_match_columns(h, abi.PODS_PENDING, snap.m, abi.ptr(idx), abi.ptr(off), abi.ptr(rows), abi.ptr(codes), total - 1) == abi.OK
    np.testing.assert_array_equal(off, want_off)
    assert (rows == -7).all() and (codes == 9).all()
    # exactly enough room
    rows = np.zeros(total, np.int64)
    codes = np.zeros(total, np.uint8)
    assert L.kt_get_match_columns(h, abi.PODS_PENDING, snap.m, abi.ptr(idx), abi.ptr(off), abi.ptr(rows), abi.ptr(codes), total) == abi.OK
    np.testing.assert_array_equal(rows, want_rows)
    np.testing.assert_array_equal(codes, want_cs)
    # argument errors
    for bad in (np.array([-1], np.int32), np.array([snap.m], np.int32), np.array([0, snap.m + 5], np.int32)):
        assert L.kt_get_match_columns(h, abi.PODS_RUNNING, len(bad), abi.ptr(bad), abi.ptr(off), abi.ptr(rows), None, total) == abi.ERR_INVALID
    assert L.kt_get_match_columns(h, 2, 1, abi.ptr(idx), abi.ptr(off), abi.ptr(rows), None, total) == abi.ERR_INVALID
    assert L.kt_get_match_columns(h, abi.PODS_RUNNING, 1, abi.ptr(idx), abi.ptr(off), abi.ptr(rows), abi.ptr(codes), total) == abi.ERR_INVALID
    assert L.kt_get_match_columns(h, abi.PODS_RUNNING, 1, abi.ptr(idx), None, abi.ptr(rows), None, total) == abi.ERR_INVALID
    assert L.kt_get_match_columns(h, abi.PODS_RUNNING, 1, abi.ptr(idx), abi.ptr(off), abi.ptr(rows), None, -1) == abi.ERR_INVALID
    # k = 0 writes off[0] only
    off[:] = 5
    assert L.kt_get_match_columns(h, abi.PODS_RUNNING, 0, None, abi.ptr(off), None, None, 0) == abi.OK
    assert off[0] == 0 and off[1] == 5
    eng.close()
