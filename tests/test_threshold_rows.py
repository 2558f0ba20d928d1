"""kt_update_threshold_rows: spec.threshold and spec.temporaryThresholdOverrides of listed throttle columns, replaced on the device
without recompiling the selector tables.

Two engines hold the same pods, throttles, status and reservations.  One gets every spec change as a kt_upload_throttles followed by
the same status and reservation uploads; the other gets the same final columns through kt_update_threshold_rows, in random batches
of 1 .. M columns, some of them unchanged.  Edits: threshold values (negative and wide ones within the value domain), presence
bits and resourceCounts nil / set, overrides added, removed, edited and reordered, counts 0 -> 3 and 3 -> 0, the total falling to
0 and growing from 0, parse-error flags and open ends.  Status, reservation, namespace-row and pod-row deltas and a later whole
kt_upload_throttles are mixed in.  After every step both must answer bit for bit alike through test_throttle_rows.observe (pass
modes with and without ON_EQUAL, forced pass plans, queued passes, kt_get_changed, the keyed calls, the summary, admission and a
step); at the end the pass also agrees with the columnar oracle."""
import ctypes as C

import numpy as np
import pytest

from kube_throttler_b200 import KtError, abi, synth
from test_partial_passes import observed_status, random_reserved
from test_throttle_rows import GIVEN, PLANS, assert_same, batches, engines, observe

pytestmark = pytest.mark.gpu

HOUR = 3600 * 10**9
WORLDS = {
    "C1": dict(config="C1"),
    "C2": dict(config="C2", m=150, n=2500, p=600),
    "C4": dict(config="C4", m=300, n=3000, p=500),
    "ragged": dict(config="C2", m=40, n=70, p=33, R=1),
}


def split(snap):
    """The threshold columns of every throttle: (thr[R], present, cnt, [(begin, end, flags, thr[R], present, cnt), ...])."""
    cols = []
    for t in range(snap.m):
        ovs = [(int(snap.ovr_begin[e]), int(snap.ovr_end[e]), int(snap.ovr_flags[e]), snap.ovr_thr[:, e].copy(), int(snap.ovr_present[e]),
                int(snap.ovr_cnt[e])) for e in range(snap.ovr_off[t], snap.ovr_off[t + 1])]
        cols.append((snap.thr[:, t].copy(), int(snap.thr_present[t]), int(snap.thr_cnt[t]), ovs))
    return cols


def pack(cols, R):
    """The columns of `cols` in the shape of kt_throttle_cols' threshold fields (Snapshot names)."""
    k = len(cols)
    ovs = [o for c in cols for o in c[3]]
    n = len(ovs)
    return dict(thr=np.array([c[0] for c in cols], np.int64).reshape(k, R).T.copy(), thr_present=np.array([c[1] for c in cols], np.uint32),
                thr_cnt=np.array([c[2] for c in cols], np.int64), ovr_off=np.cumsum([0] + [len(c[3]) for c in cols]).astype(np.int32),
                ovr_begin=np.array([o[0] for o in ovs], np.int64), ovr_end=np.array([o[1] for o in ovs], np.int64),
                ovr_flags=np.array([o[2] for o in ovs], np.uint8), ovr_thr=np.array([o[3] for o in ovs], np.int64).reshape(n, R).T.copy(),
                ovr_present=np.array([o[4] for o in ovs], np.uint32), ovr_cnt=np.array([o[5] for o in ovs], np.int64))


def set_columns(snap, cols):
    for f, v in pack(cols, snap.R).items():
        setattr(snap, f, v)
    snap.normalize()


def rand_amount(rng, R, wild):
    vals = rng.integers(0, 4000, size=R).astype(np.int64)
    if wild:
        vals[rng.random(R) < 0.3] *= -1
        vals[rng.random(R) < 0.15] = rng.choice([1 << 52, -(1 << 52), 0, -1])
    present = int(((rng.random(R) < 0.7).astype(np.uint32) << np.arange(R, dtype=np.uint32)).sum())
    vals[[r for r in range(R) if not present >> r & 1]] = 0
    cnt = 0
    if rng.random() < 0.6:  # resourceCounts set (else nil)
        present |= abi.COUNT_BIT
        cnt = int(rng.choice([0, 1, 3, 50, -2] if wild else [0, 1, 3, 50]))
    return vals, present, cnt


def rand_override(rng, R, now, wild):
    vals, present, cnt = rand_amount(rng, R, wild)
    begin = abi.TIME_OPEN_BEGIN if rng.random() < 0.25 else now + int(rng.integers(-3, 3)) * HOUR
    end = abi.TIME_OPEN_END if rng.random() < 0.25 else now + int(rng.integers(-2, 4)) * HOUR
    return (int(begin), int(end), abi.OVR_PARSE_ERROR if rng.random() < 0.1 else 0, vals, present, cnt)


def edit(rng, col, R, now, wild):
    thr, present, cnt, ovs = col
    ovs = list(ovs)
    how = rng.choice(["threshold", "presence", "add", "remove", "edit", "reorder", "zero_to_three", "three_to_zero", "same"])
    if how == "threshold":
        thr, present, cnt = rand_amount(rng, R, wild)
    elif how == "presence":
        thr = thr.copy()
        present ^= int(rng.choice([abi.COUNT_BIT, 1]))
        thr[0] = 0 if not present & 1 else thr[0]
        cnt = cnt if present & abi.COUNT_BIT else 0
    elif how == "add" or (how in ("edit", "reorder") and not ovs):
        ovs.insert(int(rng.integers(0, len(ovs) + 1)), rand_override(rng, R, now, wild))
    elif how == "remove" and ovs:
        ovs.pop(int(rng.integers(0, len(ovs))))
    elif how == "edit":
        ovs[int(rng.integers(0, len(ovs)))] = rand_override(rng, R, now, wild)
    elif how == "reorder":
        ovs.append(rand_override(rng, R, now, wild))
        ovs = [ovs[i] for i in rng.permutation(len(ovs))]
    elif how == "zero_to_three":
        ovs = [rand_override(rng, R, now, wild) for _ in range(3)]
    elif how == "three_to_zero":
        ovs = []
    return (thr, present, cnt, ovs)


def send(delta, rng, cols, listed):
    for b in batches(rng, np.array(sorted(listed))):
        delta.update_threshold_rows(b, pack([cols[t] for t in b], delta.R))


@pytest.mark.parametrize("wild", [False, True])
@pytest.mark.parametrize("world", list(WORLDS))
def test_threshold_deltas_equal_full_uploads(kt, oracle, world, wild):
    kw = dict(WORLDS[world])
    snap = synth.generate(kw.pop("config"), **kw).normalize()
    rng = np.random.default_rng(sum(map(ord, world)) + 7 * wild)
    m, R, now = snap.m, snap.R, snap.now
    full, delta = engines(kt, snap)
    fresh = oracle.columnar_evaluate(snap, abi.EVAL_FRESH_STATUS, words_per_row=full.words_per_row)
    snap.status = observed_status(fresh, snap, rng)
    snap.reserved, snap.reserved_present, snap.reserved_cnt = random_reserved(snap, rng)
    snap.normalize()
    for e in (full, delta):
        e.upload_status(snap)
        e.set_reserved(snap)
    cols = split(snap)
    rows = rng.integers(0, snap.pending.n, size=min(snap.pending.n, 17))
    n_ovr_seen = {int(snap.ovr_off[-1])}
    for step in range(10):
        plan = PLANS[step % len(PLANS)]
        what = ["edit", "edit", "clear", "edit", "mixed", "edit", "grow", "edit", "reupload", "edit"][step]
        listed = set()
        if what in ("edit", "mixed"):
            changed = np.nonzero(rng.random(m) < rng.choice([0.02, 0.3, 1.0]))[0]
            if len(changed) == 0:
                changed = np.array([int(rng.integers(0, m))])
            for t in changed:
                cols[t] = edit(rng, cols[t], R, now, wild)
            listed = set(changed.tolist()) | set(rng.integers(0, m, size=3).tolist())  # a few unchanged columns listed as well
        elif what == "clear":  # n_ovr falls to 0
            listed = {t for t in range(m) if cols[t][3]} or {0}
            for t in listed:
                cols[t] = (cols[t][0], cols[t][1], cols[t][2], [])
        elif what == "grow":  # and grows from 0 again
            listed = set(rng.choice(m, size=min(m, 5), replace=False).tolist())
            for t in listed:
                cols[t] = (cols[t][0], cols[t][1], cols[t][2], [rand_override(rng, R, now, wild) for _ in range(3)])
        set_columns(snap, cols)
        n_ovr_seen.add(int(snap.ovr_off[-1]))
        if what == "reupload":  # a whole kt_upload_throttles on both, then status and reservations again
            for e in (full, delta):
                e.upload_throttles(snap)
                e.upload_status(snap)
                e.set_reserved(snap)
        else:
            full.upload_throttles(snap)
            full.upload_status(snap)
            full.set_reserved(snap)
            send(delta, rng, cols, listed)
        if what == "mixed":  # status, reservation, namespace-row and pod-row deltas on both engines
            sc = rng.choice(m, size=min(m, 4), replace=False)
            nst = observed_status(fresh, snap, rng)
            for f in nst:
                if nst[f].ndim == 2:
                    snap.status[f][:, sc] = nst[f][:, sc]
                else:
                    snap.status[f][sc] = nst[f][sc]
            res, pres, cnt = random_reserved(snap, rng)
            snap.reserved[:, sc], snap.reserved_present[sc], snap.reserved_cnt[sc] = res[:, sc], pres[sc], cnt[sc]
            nsr = np.array([0], np.int32)
            pr = rng.choice(snap.pending.n, size=min(snap.pending.n, 5), replace=False)
            snap.pending.req[:, pr] = rng.integers(0, 3000, size=(R, len(pr)))
            for e in (full, delta):
                e.update_status_rows(sc, {f: (v[:, sc] if v.ndim == 2 else v[sc]) for f, v in snap.status.items()})
                e.update_reserved_rows(sc, snap.reserved[:, sc], snap.reserved_present[sc], snap.reserved_cnt[sc])
                e.update_namespace_rows(snap.n_ns, nsr, snap.ns_labels[:, nsr])
                e.update_pod_rows(abi.PODS_PENDING, pr, snap.pending.rows(pr))
        where = f"{world} wild={wild} step {step} ({what}) plan {plan}"
        assert_same(observe(full, snap, plan, rows), observe(delta, snap, plan, rows), where)
    assert 0 in n_ovr_seen and max(n_ovr_seen) > 0, n_ovr_seen
    # and the pass agrees with the oracle on the final columns
    for flags in (GIVEN, abi.EVAL_FRESH_STATUS):
        delta.evaluate(now, flags)
        got = delta.download()
        want = oracle.columnar_evaluate(snap, flags, words_per_row=delta.words_per_row)
        np.testing.assert_array_equal(got.codes, want.codes)
        np.testing.assert_array_equal(got.admit, want.admit)
        if flags == abi.EVAL_FRESH_STATUS:
            live = (snap.thr_flags & abi.THR_RESPONSIBLE) != 0
            for f in ("calc_thr", "calc_present", "calc_cnt", "throttled", "used"):
                a, b = getattr(got, f), getattr(want, f)
                np.testing.assert_array_equal(a[..., live], b[..., live], err_msg=f)
    full.close()
    delta.close()


def test_argument_and_state_errors(kt):
    snap = synth.generate("C2", m=40, n=200, p=50).normalize()
    e = kt.Engine(snap.R, snap.L, snap.LN)
    L, h = e._L, e._h
    cols = split(snap)
    idx = np.array([1, 2], np.int32)
    two = pack([cols[1], cols[2]], snap.R)

    def code(fn):
        with pytest.raises(KtError) as ex:
            fn()
        return ex.value.code

    assert code(lambda: e.update_threshold_rows(idx, two)) == abi.ERR_STATE  # before kt_upload_throttles
    e.upload_namespaces(snap.ns_labels)
    e.upload_throttles(snap)
    e.update_threshold_rows(idx, two)
    for bad in ([snap.m, 0], [-1, 0], [3, 3]):  # out of range, negative, duplicate
        assert code(lambda: e.update_threshold_rows(np.array(bad, np.int32), two)) == abi.ERR_INVALID
    keep = {f: np.ascontiguousarray(v) for f, v in two.items()}

    def struct(**over):
        a = dict(keep, **over)
        n = int(a["ovr_off"][-1]) if a["ovr_off"] is not None else 0
        tc = abi.ThrottleCols(None, None, None, *(abi.ptr(a[f]) for f in ("thr", "thr_present", "thr_cnt", "ovr_off")), n,
                              *(abi.ptr(a[f]) for f in ("ovr_begin", "ovr_end", "ovr_flags", "ovr_thr", "ovr_present", "ovr_cnt")))
        return tc

    assert L.kt_update_threshold_rows(h, -1, abi.ptr(idx), C.byref(struct())) == abi.ERR_INVALID
    assert L.kt_update_threshold_rows(h, 2, abi.ptr(idx), None) == abi.ERR_INVALID
    assert L.kt_update_threshold_rows(h, 2, None, C.byref(struct())) == abi.ERR_INVALID
    for f in ("thr", "thr_present", "thr_cnt", "ovr_off"):
        assert L.kt_update_threshold_rows(h, 2, abi.ptr(idx), C.byref(struct(**{f: None}))) == abi.ERR_INVALID, f
    for f in ("kind", "ns_id", "flags"):  # the columns the tables are made of
        tc = struct()
        setattr(tc, f, abi.ptr(np.zeros(2, np.int32)))
        assert L.kt_update_threshold_rows(h, 2, abi.ptr(idx), C.byref(tc)) == abi.ERR_INVALID, f
        assert L.kt_update_threshold_rows(h, 0, None, C.byref(tc)) == abi.ERR_INVALID, f
    # a bad ovr_off: not from 0, not monotone, not ending at n_ovr
    ovr = pack([cols[1][:3] + ([(0, 1, 0, np.zeros(snap.R, np.int64), 0, 0)] * 2,), cols[2][:3] + ([],)], snap.R)
    for off in ([1, 2, 2], [0, 2, 1], [0, 1, 1]):
        tc = struct(**{k: v for k, v in ovr.items() if k != "ovr_off"}, ovr_off=np.array(off, np.int32))
        tc.n_ovr = 2
        assert L.kt_update_threshold_rows(h, 2, abi.ptr(idx), C.byref(tc)) == abi.ERR_INVALID, off
    tc = struct(**ovr)
    tc.ovr_thr = None
    assert L.kt_update_threshold_rows(h, 2, abi.ptr(idx), C.byref(tc)) == abi.ERR_INVALID
    # k = 0: a no-op, null columns allowed
    assert L.kt_update_threshold_rows(h, 0, None, None) == abi.OK
    # the status and reservations held before the call are kept; a pass is needed again before the getters that read one
    snap.status = {f: np.zeros((snap.R, snap.m) if f in ("calc_thr", "used") else snap.m) for f in
                   ("calculated", "calc_thr", "calc_present", "calc_cnt", "used", "used_present", "used_cnt", "throttled")}
    snap.normalize()
    e.upload_status(snap)
    e.evaluate(snap.now, abi.EVAL_FRESH_STATUS)
    e.get_changed()
    e.update_threshold_rows(idx, ovr)
    assert code(lambda: e.get_changed()) == abi.ERR_STATE
    e.update_status_rows(idx, {f: (v[:, idx] if v.ndim == 2 else v[idx]) for f, v in snap.status.items()})  # still held
    e.evaluate(0, GIVEN)
    e.close()
