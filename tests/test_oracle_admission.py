"""The columnar oracle's queue admission (oracle/ko_columnar.h columnar_admit_queue: one pod per cycle, O(queue x m)) against
the obvious restatement of the cycle on top of the plain pass: one full columnar_evaluate after every admitted pod, with the pod's
requests added to the reservations of the throttles it affects (O(queue^2)).  CPU only; the GPU tests compare kt_admit_queue
with columnar_admit_queue at shapes the slow loop could not afford."""
import numpy as np
import pytest

from kube_throttler_b200 import abi, synth

FLAGS = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE


def admission_world(oracle, config, throttled=False, zero_counts=False, orphans=False, **kw):
    """A synthetic world as PreFilter sees it between reconciles: the observed status is this pass's, and the thresholds leave
    room for a few pods on most throttles, so that admissions and rejections interleave along the queue.
    throttled: a fifth of the status's throttled masks set; zero_counts: some count thresholds 0 (no pod fits);
    orphans: the Throttles of namespace 0 moved to namespace 1, so the pending pods of namespace 0 affect no throttle (C2)."""
    snap = synth.generate(config, **kw)
    if orphans:
        assert not (snap.kind == abi.KIND_CLUSTERTHROTTLE).any()
        snap.thr_ns = np.where(snap.thr_ns == 0, 1, snap.thr_ns).astype(np.int32)
        assert (snap.pending.ns_id == 0).any()
    fresh = oracle.columnar_evaluate(snap)
    m = snap.m
    rng = np.random.default_rng(3)
    snap.thr = np.where(snap.thr > 0, fresh.used + (snap.thr * rng.uniform(0.0, 0.08, size=snap.thr.shape)).astype(np.int64) + 1, 0)
    snap.thr_cnt = np.where(snap.thr_cnt > 0, fresh.used_cnt + rng.integers(0, 6, size=m), snap.thr_cnt)
    if zero_counts:
        zero = rng.random(m) < 0.1
        snap.thr_cnt = np.where(zero, 0, snap.thr_cnt)
        snap.thr_present = np.where(zero, snap.thr_present | abi.COUNT_BIT, snap.thr_present).astype(np.uint32)
    st_throttled = np.zeros(m, np.uint32)
    if throttled:
        st_throttled = np.where(rng.random(m) < 0.2, rng.integers(0, 1 << snap.R, size=m) | np.where(rng.random(m) < 0.5, abi.COUNT_BIT, 0), 0)
    snap.status = dict(calculated=np.ones(m, np.uint8), calc_thr=snap.thr.copy(), calc_present=snap.thr_present.copy(), calc_cnt=snap.thr_cnt.copy(),
                       used=fresh.used.copy(), used_present=fresh.used_present.copy(), used_cnt=fresh.used_cnt.copy(),
                       throttled=st_throttled.astype(np.uint32))
    return snap.normalize()


def pass_per_pod(oracle, snap, first, count, flags, W):
    """The cycle, restated on the plain pass: (codes, admit, admitted, (reserved, reserved_present, reserved_cnt))."""
    m, R = snap.m, snap.R
    saved = snap.reserved.copy(), snap.reserved_present.copy(), snap.reserved_cnt.copy()
    cur = oracle.columnar_evaluate(snap, flags, words_per_row=W)
    codes, admit, bitmap = cur.codes.copy(), cur.admit.copy(), cur.pend_bitmap
    rmask = np.uint32((1 << R) - 1)
    n_adm = 0
    for i in range(first, first + count):
        codes[i], admit[i] = cur.codes[i], cur.admit[i]
        if not cur.admit[i]:
            continue
        n_adm += 1
        ts = np.nonzero(((bitmap[i][:, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(-1)[:m])[0]
        if ts.size == 0:
            continue
        pres = snap.pending.present[i] & rmask
        for r in range(R):
            if (pres >> np.uint32(r)) & 1:
                snap.reserved[r, ts] += snap.pending.req[r, i]
        snap.reserved_present[ts] |= pres | abi.COUNT_BIT
        snap.reserved_cnt[ts] += 1
        snap.normalize()
        cur = oracle.columnar_evaluate(snap, flags, words_per_row=W)
    final = snap.reserved, snap.reserved_present, snap.reserved_cnt
    snap.reserved, snap.reserved_present, snap.reserved_cnt = saved
    return codes, admit, n_adm, final


@pytest.mark.parametrize("world,first,count,flags", [
    (dict(config="C2", m=60, n=1000, p=200), 0, 200, 0),
    (dict(config="C2", m=60, n=1000, p=200), 37, 120, 0),                        # a sub-range: the rows around it keep the pass's codes
    (dict(config="C3", m=50, n=800, p=150, R=5, seed=9), 0, 150, abi.EVAL_ON_EQUAL),
    (dict(config="C2", m=60, n=1000, p=200, throttled=True, zero_counts=True), 0, 200, 0),
    (dict(config="C2", m=60, n=1000, p=200, orphans=True), 0, 200, 0),
    (dict(config="C2", m=60, n=1000, p=200, values="signed"), 0, 200, 0),
    (dict(config="C4", m=80, n=1000, p=200), 0, 200, abi.EVAL_ON_EQUAL),          # overrides active
])
def test_columnar_admit_queue_equals_a_pass_per_admitted_pod(oracle, world, first, count, flags):
    world = dict(world)
    snap = admission_world(oracle, world.pop("config"), **world)
    W = abi.default_words_per_row(snap.m)
    got, admitted, reserved = oracle.columnar_admit_queue(snap, first, count, flags, words_per_row=W)
    codes, admit, n_adm, want_reserved = pass_per_pod(oracle, snap, first, count, FLAGS | flags, W)
    np.testing.assert_array_equal(got.admit, admit)
    np.testing.assert_array_equal(got.codes, codes)
    assert admitted == n_adm and 0 < n_adm < count, (n_adm, count)
    for a, b in zip(reserved, want_reserved):
        np.testing.assert_array_equal(a, b)
    # the reservations the queue left behind, checked once more without either loop: admitted requests summed per throttle
    affected = np.stack([((got.pend_bitmap[:, t >> 5] >> np.uint32(t & 31)) & 1).astype(bool) for t in range(snap.m)], axis=1)
    adm = got.admit.astype(bool) & (np.arange(snap.pending.n) >= first) & (np.arange(snap.pending.n) < first + count)
    np.testing.assert_array_equal(reserved[2], snap.reserved_cnt + (affected & adm[:, None]).sum(axis=0))
