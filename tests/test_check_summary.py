"""kt_get_check_summary: the pending rows of the last checking pass summarised per throttle on the device.

Every answer is compared exactly with a numpy reduction of the columnar oracle's codes over the snapshot's pending columns, and
with the same reduction of what kt_get_check delivers on the same context: per-status counts, the rows a throttle alone rejects,
the request sums and their presence, over row ranges and random row classes, in both row layouts, after a full pass, a check-only
pass and kt_admit_queue.  The call must leave every getter as it was."""
import numpy as np
import pytest

from kube_throttler_b200 import KtError, abi, synth
from test_check_rows import assert_same_getters, getters, with_status

pytestmark = pytest.mark.gpu

FRESH = abi.EVAL_FRESH_STATUS
GIVEN = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE


def expected(snap, codes, admit, first, count, row_class=None):
    """(status_cnt[3][m], sole_cnt[m], held[R][m], held_present[m]) of the dense codes / admit bytes of a pass, in numpy."""
    m, R = snap.m, snap.R
    rows = np.arange(first, first + count)
    cls = np.ones(count, np.uint8) if row_class is None else np.asarray(row_class, np.uint8)
    assert not codes[admit.astype(bool)].any(), "an admitted row carries a non-zero code"
    t = np.arange(m)
    c = ((codes[rows][:, t >> 4] >> (2 * (t & 15)).astype(np.uint32)) & 3).astype(np.int64)  # [count][m]
    c[cls == 0] = 0
    on = c != 0
    status_cnt = np.stack([(c == k).sum(0) for k in (1, 2, 3)]).astype(np.int64)
    sole = (cls == 1) & (on.sum(1) == 1)
    sole_cnt = (on & sole[:, None]).sum(0).astype(np.int64)
    present = snap.pending.present[rows].astype(np.uint32) & np.uint32(~abi.COUNT_BIT & 0xFFFFFFFF)
    held = np.zeros((R, m), np.int64)
    for r in range(R):
        v = np.where((present >> np.uint32(r)) & 1, snap.pending.req[r, rows], 0).astype(np.int64)
        held[r] = (on * v[:, None]).sum(0, dtype=np.int64)
    held_present = np.zeros(m, np.uint32)
    for i in np.nonzero(on.any(1))[0]:
        held_present[on[i]] |= present[i] | np.uint32(abi.COUNT_BIT)
    return status_cnt, sole_cnt, held, held_present


def assert_summary(got, want, note=""):
    for name, a, b in zip(("status_cnt", "sole_cnt", "held", "held_present"), got, want):
        np.testing.assert_array_equal(a, b, err_msg=f"{note}: {name}")


def ranges(P, rng):
    """the whole table, a prefix, a suffix, a middle slice, one row at either end, and count = 0"""
    out = [(0, P)]
    if P:
        a, b = sorted(rng.integers(0, P + 1, size=2))
        out += [(0, max(1, P // 3)), (P // 2, P - P // 2), (int(a), int(b - a)), (0, 1), (P - 1, 1), (int(rng.integers(0, P)), 0)]
    return out + [(P, 0)]


def check_all(eng, snap, want_codes, want_admit, rng, note):
    """Every range, with no classes and with random ones, against the oracle's codes and against kt_get_check's."""
    P = snap.pending.n
    codes = np.zeros((P, 2 * eng.words_per_row), np.uint32)
    admit = np.zeros(P, np.uint8)
    eng.get_check(codes, admit)
    np.testing.assert_array_equal(codes, want_codes, err_msg=f"{note}: kt_get_check codes")
    np.testing.assert_array_equal(admit, want_admit, err_msg=f"{note}: kt_get_check admit")
    for first, count in ranges(P, rng):
        for cls in (None, rng.integers(0, 3, size=count).astype(np.uint8), np.full(count, 2, np.uint8)):
            want = expected(snap, want_codes, want_admit, first, count, cls)
            assert_summary(eng.check_summary(first, count, cls), want, f"{note} [{first}, +{count}) classes={cls is not None}")
    status_cnt, _, _, _ = eng.check_summary(0, P)
    return int(status_cnt.sum())


SHAPES = [
    dict(config="C1"),
    dict(config="C2", m=200, n=3000, p=1500),
    dict(config="C3", m=300, n=3000, p=1200),                          # ClusterThrottles
    dict(config="C4", m=500, n=4000, p=1000),                          # overrides
    dict(config="C2", m=333, n=3000, p=1111, sort_by_namespace=False),  # M not a multiple of 16 or 32, rows in arrival order
    dict(config="C2", m=40, n=70, p=33, R=1),                          # R = 1, a partial warp, a partial last word
    dict(config="C2", m=150, n=2000, p=600, R=12),
    dict(config="C2", m=120, n=2000, p=500, R=31, L=12),                # the widest R
    dict(config="C3", m=300, n=3000, p=800, values="signed"),          # negative requests
    dict(config="C4", m=200, n=3000, p=700, values="wide"),            # values beyond 2^44 (every limb of the warp sums)
]


@pytest.mark.parametrize("kw", SHAPES)
def test_summary_equals_oracle_and_get_check(kt, oracle, kw):
    kw = dict(kw)
    snap = synth.generate(kw.pop("config"), **kw)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(snap.m + snap.pending.n)
    with_status(eng, snap, oracle, rng)
    eng.evaluate(0, GIVEN)  # what every PreFilter pass of the plugin runs
    want = oracle.columnar_evaluate(snap, GIVEN, words_per_row=eng.words_per_row)
    assert check_all(eng, snap, want.codes, want.admit, rng, "check-only pass") > 0
    eng.evaluate(snap.now, FRESH)  # a whole pass (the fused kernel): its own codes
    want = oracle.columnar_evaluate(snap, FRESH, words_per_row=eng.words_per_row)
    check_all(eng, snap, want.codes, want.admit, rng, "fresh pass")
    eng.close()


def test_summary_on_golden_value_edges(kt, oracle):
    from test_golden import load

    meta, snap, gold = load("c2_value_edges")
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    eng.evaluate(snap.now, meta["flags"])
    assert eng.words_per_row == meta["words_per_row"]
    check_all(eng, snap, gold["codes"], gold["admit"], np.random.default_rng(4), "c2_value_edges")
    eng.close()


@pytest.mark.parametrize("mode", [abi.ROW_ORDER_BY_NAMESPACE, abi.ROW_ORDER_AS_GIVEN])
def test_summary_in_either_row_order(kt, oracle, mode):
    snap = synth.generate("C2", m=300, n=3000, p=2000, sort_by_namespace=False)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.set_row_order(abi.PODS_PENDING, mode)
    rng = np.random.default_rng(13)
    with_status(eng, snap, oracle, rng)
    assert eng.row_order(abi.PODS_PENDING)[0] == (mode == abi.ROW_ORDER_BY_NAMESPACE)
    eng.evaluate(0, GIVEN)
    want = oracle.columnar_evaluate(snap, GIVEN, words_per_row=eng.words_per_row)
    check_all(eng, snap, want.codes, want.admit, rng, f"order {mode}")
    eng.close()


def test_summary_of_admit_queue_codes(kt, oracle):
    """kt_admit_queue leaves the codes each rejected queue row saw at its turn, and a check-only pass's outside the queue."""
    snap = synth.generate("C2", m=200, n=3000, p=1500)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(21)
    with_status(eng, snap, oracle, rng)
    eng.admit_queue(200, 900)
    P = snap.pending.n
    codes, admit = np.zeros((P, 2 * eng.words_per_row), np.uint32), np.zeros(P, np.uint8)
    eng.get_check(codes, admit)
    assert codes[200:1100].any() and admit[200:1100].any()
    for first, count in ranges(P, rng):
        cls = rng.integers(0, 3, size=count).astype(np.uint8)
        assert_summary(eng.check_summary(first, count, cls), expected(snap, codes, admit, first, count, cls), f"admit_queue [{first}, +{count})")
    eng.close()


def _crowded_world(P, m, hot, seed=0):
    """P pending pods in one namespace, m Throttles; column `hot` matches every pod (one term, no requirements) with a pod-count
    threshold of 0, so it rejects every row; the others select one value of k0 each with a random cpu threshold.  Requests
    are signed."""
    rng = np.random.default_rng(seed)
    L, R, LN = 2, 2, 1
    lab = np.full((L, P), abi.LABEL_EMPTY, np.int64)
    lab[0] = rng.integers(0, 4, size=P).astype(np.int64)  # k0 = v0..v3
    req = rng.integers(-50, 400, size=(R, P)).astype(np.int64)
    present = rng.integers(0, 4, size=P).astype(np.uint32)
    pending = abi.PodCols(lab, req, present, np.full(P, abi.POD_SCHEDULER_MATCH | abi.POD_NOT_FINISHED, np.uint32), np.zeros(P, np.int32))
    running = abi.PodCols(np.full((L, 0), abi.LABEL_EMPTY, np.int64), np.zeros((R, 0), np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint32),
                          np.zeros(0, np.int32))
    terms = [[] if t == hot else [(0, abi.OP_IN, [t % 4])] for t in range(m)]
    sel = synth.build_selector_csr(list(range(m + 1)), terms, [[] for _ in range(m)])
    thr = np.zeros((R, m), np.int64)
    thr[0] = rng.integers(0, 300, size=m)
    thr_present = np.ones(m, np.uint32)
    thr_present[hot] = abi.COUNT_BIT
    snap = abi.Snapshot(
        R=R, L=L, LN=LN, running=running, pending=pending, ns_labels=np.full((LN, 1), abi.LABEL_EMPTY, np.int64),
        kind=np.zeros(m, np.uint8), thr_ns=np.zeros(m, np.int32), thr_flags=np.full(m, abi.THR_RESPONSIBLE, np.uint8),
        thr=thr, thr_present=thr_present, thr_cnt=np.zeros(m, np.int64),
        ovr_off=np.zeros(m + 1, np.int32), ovr_begin=np.zeros(0, np.int64), ovr_end=np.zeros(0, np.int64),
        ovr_flags=np.zeros(0, np.uint8), ovr_thr=np.zeros((R, 0), np.int64), ovr_present=np.zeros(0, np.uint32),
        ovr_cnt=np.zeros(0, np.int64), now=synth.NOW_2026, **sel)
    return snap.normalize()


def test_one_throttle_rejects_every_row(kt, oracle):
    """One throttle rejects all 120k pending rows, each warp's lanes crediting it at once: the sums stay exact."""
    P, m, hot = 120_000, 35, 20
    snap = _crowded_world(P, m, hot)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    eng.evaluate(snap.now, FRESH)
    want = oracle.columnar_evaluate(snap, FRESH, words_per_row=eng.words_per_row)
    hot_codes = (want.codes[:, hot >> 4] >> np.uint32(2 * (hot & 15))) & 3
    assert (hot_codes != 0).all()
    got = eng.check_summary(0, P)
    assert_summary(got, expected(snap, want.codes, want.admit, 0, P), "crowded")
    assert got[0][:, hot].sum() == P
    cls = np.random.default_rng(1).integers(0, 3, size=P).astype(np.uint8)
    assert_summary(eng.check_summary(0, P, cls), expected(snap, want.codes, want.admit, 0, P, cls), "crowded, classes")
    eng.close()


def test_summary_leaves_every_getter_unchanged(kt, oracle):
    snap = synth.generate("C2", m=300, n=3000, p=1500)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    rng = np.random.default_rng(5)
    with_status(eng, snap, oracle, rng)
    eng.evaluate(snap.now)  # a fused FRESH pass: status columns, diff, bitmaps, codes of its own
    eng.set_sparse_check(1 << 16)
    eng.evaluate(snap.now)
    before = getters(eng, snap)
    sparse = np.zeros((1 << 16, 3), np.uint32)
    n_before = eng.get_check_sparse(None, sparse)
    for first, count in ranges(snap.pending.n, rng):
        eng.check_summary(first, count, rng.integers(0, 3, size=count).astype(np.uint8))
    assert_same_getters(before, getters(eng, snap))
    sparse2 = np.zeros_like(sparse)
    assert eng.get_check_sparse(None, sparse2) == n_before
    np.testing.assert_array_equal(sparse2[:n_before], sparse[:n_before])
    eng.close()


def test_arguments_and_state(kt, oracle):
    snap = synth.generate("C2", m=200, n=2000, p=700)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    L, h = eng._L, eng._h
    P = snap.pending.n
    out = abi.CheckSummary()
    call = lambda first, count: L.kt_get_check_summary(h, first, count, None, out)
    assert call(0, 0) == abi.ERR_STATE  # nothing uploaded, no pass
    eng.upload_snapshot(snap)
    assert call(0, P) == abi.ERR_STATE  # uploaded, no pass
    eng.evaluate(snap.now, abi.EVAL_FRESH_STATUS | abi.EVAL_SKIP_CHECK)
    assert call(0, P) == abi.ERR_STATE  # a reconcile-only pass writes no codes
    eng.evaluate(snap.now)
    assert call(0, P) == abi.OK and call(0, 0) == abi.OK and call(P, 0) == abi.OK and call(3, P - 3) == abi.OK
    for first, count in ((-1, 1), (0, -1), (0, P + 1), (P, 1), (P - 2, 3), (P + 1, 0)):
        assert call(first, count) == abi.ERR_INVALID, (first, count)
    assert L.kt_get_check_summary(h, 0, 1, None, None) == abi.ERR_INVALID
    eng.upload_pods(abi.PODS_PENDING, snap.pending)  # new pending rows: the codes belong to the old ones
    assert call(0, P) == abi.ERR_STATE
    eng.evaluate(snap.now, abi.EVAL_FRESH_STATUS | abi.EVAL_SKIP_CHECK)
    assert call(0, P) == abi.ERR_STATE
    eng.evaluate(snap.now)
    assert call(0, P) == abi.OK
    eng.upload_throttles(snap)  # new throttle columns: the same
    assert call(0, P) == abi.ERR_STATE
    eng.evaluate(snap.now)
    assert call(0, P) == abi.OK
    # count = 0 yields zeros; every output alone
    got = eng.check_summary(0, P)
    assert all(not a.any() for a in eng.check_summary(5, 0))
    for i, name in enumerate(("status_cnt", "sole_cnt", "held", "held_present")):
        one = abi.CheckSummary()
        a = np.zeros_like(got[i])
        setattr(one, name, abi.ptr(a))
        assert L.kt_get_check_summary(h, 0, P, None, one) == abi.OK
        np.testing.assert_array_equal(a, got[i], err_msg=name)
    eng.close()


def test_empty_pending_table(kt, oracle):
    snap = synth.generate("C2", m=100, n=1000, p=0)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    eng.evaluate(snap.now)
    got = eng.check_summary(0, 0)
    assert got[0].shape == (3, snap.m) and all(not a.any() for a in got)
    with pytest.raises(KtError):
        eng.check_summary(0, 1)
    eng.close()
