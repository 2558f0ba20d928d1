"""kt_update_status_rows / kt_update_reserved_rows: the observed status and the reservations of listed throttle columns, replaced in
place on the device.

Two engines hold the same pods and throttles.  One gets every change of the status and reservation columns as a whole-table
kt_upload_status / kt_set_reserved; the other gets the same final columns through the column deltas, in random batches of 1 .. M
columns (some of them unchanged), including deltas before any kt_set_reserved and after kt_set_reserved(NULL).  After every step
both must answer bit for bit alike: GIVEN_STATUS | SKIP_RECONCILE passes with and without ON_EQUAL, FRESH_STATUS passes and their
status diff (kt_get_changed), kt_check_pending_rows, kt_get_check_summary, kt_admit_queue and a kt_step_submit / kt_step_wait step
-- with the fused pass's builds and decide modes forced in turn, and with two passes queued back to back right after a delta.
Worlds: BASELINE C1-C4 slices, the wide-value golden world, negative and wide status and reservation values."""
import ctypes as C

import numpy as np
import pytest

from kube_throttler_b200 import KtError, abi, synth
from test_golden import INDEX
from test_partial_passes import observed_status, random_reserved

pytestmark = pytest.mark.gpu

FRESH = abi.EVAL_FRESH_STATUS
GIVEN = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE
PLANS = [(0, 0), (512, abi.PLAN_DECIDE_QUAD), (512, abi.PLAN_DECIDE_PER_POD), (768, abi.PLAN_DECIDE_QUAD), (768, abi.PLAN_DECIDE_PER_POD)]
STATUS = ("calculated", "calc_thr", "calc_present", "calc_cnt", "used", "used_present", "used_cnt", "throttled")

WORLDS = {
    "C1": dict(config="C1"),
    "C2": dict(config="C2", m=150, n=2500, p=600),
    "C3": dict(config="C3", m=200, n=2500, p=500),
    "C4": dict(config="C4", m=300, n=3000, p=500),
    "c2_value_edges": dict(config=INDEX["c2_value_edges"]["config"], **INDEX["c2_value_edges"]["kwargs"]),
    "ragged": dict(config="C2", m=40, n=70, p=33, R=1),
}


def cols_of(st, idx):
    return {f: (st[f][:, idx] if st[f].ndim == 2 else st[f][idx]) for f in STATUS}


def new_status(fresh, snap, rng, wild):
    st = observed_status(fresh, snap, rng)
    if wild:  # negative and wide values within the value domain
        m = snap.m
        for f in ("used", "calc_thr"):
            flip = rng.random(st[f].shape) < 0.2
            st[f][flip] = -st[f][flip]
            st[f][rng.random(st[f].shape) < 0.05] = rng.choice([-(1 << 52), 1 << 52, -1, 0])
        st["used_cnt"][rng.random(m) < 0.1] = -3
    return st


def new_reserved(snap, rng, wild):
    res, present, cnt = random_reserved(snap, rng)
    if wild:
        res[rng.random(res.shape) < 0.2] *= -1
        res[rng.random(res.shape) < 0.03] = 1 << 50
    return res, present, cnt


def batches(rng, cols):
    """The columns in random order, cut into random batches of 1 .. len(cols)."""
    cols = rng.permutation(cols)
    out, i = [], 0
    while i < len(cols):
        k = int(rng.integers(1, len(cols) - i + 1))
        out.append(cols[i:i + k])
        i += k
    return out


def observe(eng, snap, plan, rows):
    """Everything the throttle-side columns feed, in one list of arrays."""
    eng.set_pass_plan(*plan)
    out = []
    P = snap.pending.n
    # two passes queued back to back right behind the delta: the second one starts its first phase while the first decides
    eng.evaluate(snap.now, FRESH)
    eng.evaluate(0, GIVEN)
    r = eng.download()
    out += [r.pend_bitmap, r.codes, r.admit]
    out += list(eng.check_summary(0, P))
    eng.evaluate(0, GIVEN | abi.EVAL_ON_EQUAL)
    r = eng.download()
    out += [r.codes, r.admit]
    eng.evaluate(snap.now, FRESH)
    r = eng.download()
    out += [r.used, r.used_present, r.used_cnt, r.throttled, r.calc_thr, r.calc_present, r.calc_cnt, r.codes, r.admit]
    out += list(eng.get_changed())
    out += list(eng.check_summary(0, P))
    eng.set_pass_plan()
    for on_equal in (False, True):
        out += list(eng.check_pending_rows(rows, on_equal))
    out += list(eng.admit_queue(0, P))
    codes, admit = eng.get_check_rows(np.arange(P))
    out += [codes, admit]
    eng.step_submit(None, None, snap.now, GIVEN)
    res = eng.step_wait()
    out.append(np.ctypeslib.as_array(C.cast(res.admit, C.POINTER(C.c_uint8)), (max(P, 1),))[:P].copy())
    return out


def assert_same(a, b, where):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        np.testing.assert_array_equal(np.asarray(x), np.asarray(y), err_msg=f"{where}: output {i}")


def engines(kt, snap):
    out = []
    for _ in range(2):
        e = kt.Engine(snap.R, snap.L, snap.LN)
        e.upload_namespaces(snap.ns_labels)
        e.upload_throttles(snap)
        e.upload_pods(abi.PODS_RUNNING, snap.running)
        e.upload_pods(abi.PODS_PENDING, snap.pending)
        e.set_sparse_check(1 << 16)
        out.append(e)
    return out


@pytest.mark.parametrize("wild", [False, True])
@pytest.mark.parametrize("world", list(WORLDS))
def test_deltas_equal_full_uploads(kt, oracle, world, wild):
    kw = dict(WORLDS[world])
    snap = synth.generate(kw.pop("config"), **kw).normalize()
    rng = np.random.default_rng(sum(map(ord, world)) + wild)
    m, R = snap.m, snap.R
    full, delta = engines(kt, snap)
    fresh = oracle.columnar_evaluate(snap, FRESH, words_per_row=full.words_per_row)
    st = new_status(fresh, snap, rng, wild)
    snap.status = st
    full.upload_status(snap)
    delta.upload_status(snap)
    # reservations: the delta engine starts from "nothing reserved" (no kt_set_reserved yet)
    res = [np.zeros((R, m), np.int64), np.zeros(m, np.uint32), np.zeros(m, np.int64)]
    rows = rng.integers(0, snap.pending.n, size=min(snap.pending.n, 17))
    for step in range(8):
        plan = PLANS[step % len(PLANS)]
        what = step % 4
        if what in (0, 1):  # new reservations on some columns (step 0: before any kt_set_reserved of the delta engine)
            nres = new_reserved(snap, rng, wild)
            cols = np.nonzero(rng.random(m) < rng.choice([0.02, 0.3, 1.0]))[0]
            if len(cols) == 0:
                cols = np.array([int(rng.integers(0, m))])
            for a, b in zip(res, nres):
                if a.ndim == 2:
                    a[:, cols] = b[:, cols]
                else:
                    a[cols] = b[cols]
            snap.reserved, snap.reserved_present, snap.reserved_cnt = res
            full.set_reserved(snap)
            for b in batches(rng, cols):
                delta.update_reserved_rows(b, res[0][:, b], res[1][b], res[2][b])
        elif what == 2:  # a new observed status on some columns, a few unchanged ones listed as well
            nst = new_status(fresh, snap, rng, wild)
            cols = np.nonzero(rng.random(m) < rng.choice([0.02, 0.3, 1.0]))[0]
            for f in STATUS:
                if st[f].ndim == 2:
                    st[f][:, cols] = nst[f][:, cols]
                else:
                    st[f][cols] = nst[f][cols]
            listed = np.union1d(cols, rng.integers(0, m, size=3))
            full.upload_status(snap)
            for b in batches(rng, listed):
                delta.update_status_rows(b, cols_of(st, b))
        else:  # everything cleared, then a delta on a few columns: the others are "nothing reserved"
            for e in (full, delta):
                e._ck(e._L.kt_set_reserved(e._h, None, None, None))
            cols = rng.choice(m, size=min(m, 3), replace=False)
            for a in res:
                a[...] = 0
            nres = new_reserved(snap, rng, wild)
            for a, b in zip(res, nres):
                if a.ndim == 2:
                    a[:, cols] = b[:, cols]
                else:
                    a[cols] = b[cols]
            full.set_reserved(snap)
            delta.update_reserved_rows(cols, res[0][:, cols], res[1][cols], res[2][cols])
        where = f"{world} wild={wild} step {step} plan {plan}"
        assert_same(observe(full, snap, plan, rows), observe(delta, snap, plan, rows), where)
    # and the pass agrees with the oracle on the final columns
    full.evaluate(0, GIVEN)
    got = full.download()
    want = oracle.columnar_evaluate(snap, GIVEN, words_per_row=full.words_per_row)
    np.testing.assert_array_equal(got.codes, want.codes)
    np.testing.assert_array_equal(got.admit, want.admit)
    full.close()
    delta.close()


def test_argument_and_state_errors(kt):
    snap = synth.generate("C2", m=40, n=200, p=50).normalize()
    e = kt.Engine(snap.R, snap.L, snap.LN)
    L, h = e._L, e._h
    idx = np.array([1, 2], np.int32)
    st = {f: np.zeros((snap.R, 2) if f in ("calc_thr", "used") else 2, np.int64 if f in ("calc_thr", "used", "calc_cnt", "used_cnt") else
                      (np.uint8 if f == "calculated" else np.uint32)) for f in STATUS}
    res, present, cnt = np.zeros((snap.R, 2), np.int64), np.zeros(2, np.uint32), np.zeros(2, np.int64)

    def code(fn):
        with pytest.raises(KtError) as ex:
            fn()
        return ex.value.code

    # before kt_upload_throttles
    assert code(lambda: e.update_status_rows(idx, st)) == abi.ERR_STATE
    assert code(lambda: e.update_reserved_rows(idx, res, present, cnt)) == abi.ERR_STATE
    e.upload_namespaces(snap.ns_labels)
    e.upload_throttles(snap)
    # a partial status over no status
    assert code(lambda: e.update_status_rows(idx, st)) == abi.ERR_STATE
    e.update_reserved_rows(idx, res, present, cnt)  # reservations need no kt_set_reserved first
    snap.status = {f: np.zeros((snap.R, snap.m) if f in ("calc_thr", "used") else snap.m) for f in STATUS}
    snap.normalize()
    e.upload_status(snap)
    e.update_status_rows(idx, st)
    for bad in ([snap.m, 0], [-1, 0], [3, 3]):  # out of range, negative, duplicate
        b = np.array(bad, np.int32)
        assert code(lambda: e.update_status_rows(b, st)) == abi.ERR_INVALID
        assert code(lambda: e.update_reserved_rows(b, res, present, cnt)) == abi.ERR_INVALID
    sc = abi.StatusCols(*(abi.ptr(np.ascontiguousarray(st[f])) for f in STATUS))
    assert L.kt_update_status_rows(h, -1, abi.ptr(idx), C.byref(sc)) == abi.ERR_INVALID
    assert L.kt_update_reserved_rows(h, -1, abi.ptr(idx), abi.ptr(res), abi.ptr(present), abi.ptr(cnt)) == abi.ERR_INVALID
    assert L.kt_update_status_rows(h, 2, abi.ptr(idx), None) == abi.ERR_INVALID
    sc.used = None
    assert L.kt_update_status_rows(h, 2, abi.ptr(idx), C.byref(sc)) == abi.ERR_INVALID
    assert L.kt_update_reserved_rows(h, 2, abi.ptr(idx), abi.ptr(res), None, abi.ptr(cnt)) == abi.ERR_INVALID
    assert L.kt_update_reserved_rows(h, 2, None, abi.ptr(res), abi.ptr(present), abi.ptr(cnt)) == abi.ERR_INVALID
    # k = 0: a no-op, null columns allowed
    assert L.kt_update_status_rows(h, 0, None, None) == abi.OK
    assert L.kt_update_reserved_rows(h, 0, None, None, None, None) == abi.OK
    # kt_upload_throttles forgets the status again
    e.upload_throttles(snap)
    assert code(lambda: e.update_status_rows(idx, st)) == abi.ERR_STATE
    e.close()
