"""The request-value regimes of the synthetic generator (synth.generate(values=...)): each does what the GPU parity tests rely
on it for, and the columnar oracle's int64 sums are exact on them (compared with Python-int sums over the matched rows)."""
import numpy as np
import pytest

from kube_throttler_b200 import abi, synth

SHAPE = dict(m=300, n=6000, p=800)


def _bits(mask, R):
    return ((np.asarray(mask, np.uint32)[None, :] >> np.arange(R, dtype=np.uint32)[:, None]) & 1).astype(bool)


def _matched(bitmap, t):
    return ((bitmap[:, t >> 5] >> np.uint32(t & 31)) & 1).astype(bool)


def test_default_snapshots_are_unchanged():
    a, b = synth.generate("C3", **SHAPE), synth.generate("C3", **SHAPE, values=None)
    for f in ("thr", "thr_present", "thr_cnt", "reserved"):
        np.testing.assert_array_equal(getattr(a, f), getattr(b, f))
    np.testing.assert_array_equal(a.running.req, b.running.req)
    assert a.running.req.max() < 1 << 37


@pytest.mark.parametrize("config", ["C3", "C4"])
@pytest.mark.parametrize("values", synth.VALUE_REGIMES)
def test_value_regime(oracle, config, values):
    snap = synth.generate(config, **SHAPE, values=values)
    R, m = snap.R, snap.m
    res = oracle.columnar_evaluate(snap)
    present = [_bits(pods.present, R) for pods in (snap.running, snap.pending)]
    vals = np.concatenate([snap.running.req[present[0]], snap.pending.req[present[1]]])
    if values == "wide":
        assert (vals >= synth.HIGH_LIMB).all()
    elif values == "carry":
        assert (vals & 0xFFFFFFFF == 0xFFFFFFFF).all() and (vals >= 1 << 32).any()
    else:
        assert (vals < 0).any() and (vals > 0).any() and (vals == 0).any()
        assert (res.used[_bits(res.used_present, R)] < 0).any()  # some matched sums are negative

    # the domain the host layer guarantees: per column, sum |v| over running + pending + reservations + status below 2^62
    for r in range(R):
        total = sum(abs(int(v)) for v in snap.running.req[r].tolist()) + sum(abs(int(v)) for v in snap.pending.req[r].tolist())
        total += sum(abs(int(v)) for v in snap.reserved[r].tolist()) + sum(abs(int(v)) for v in res.used[r].tolist())
        assert total < 1 << 62, (r, total)

    # the oracle's used sums are the exact (Python int) sums over the matched, counted rows: the int64 reference does not wrap
    f = snap.running.flags
    alive = ((f & abi.POD_SCHEDULER_MATCH) != 0) & ((f & abi.POD_SCHEDULED) != 0) & ((f & abi.POD_NOT_FINISHED) != 0)
    live = ((snap.thr_flags & abi.THR_RESPONSIBLE) != 0) & ((snap.thr_flags & abi.THR_SELECTOR_ERROR) == 0)
    req = (snap.running.req * present[0]).astype(object)
    for t in np.nonzero(live)[0]:
        rows = _matched(res.run_bitmap, t) & alive
        for r in range(R):
            assert int(res.used[r, t]) == sum(req[r, rows].tolist()), (t, r)

    # exact-equality thresholds: S3 (alreadyUsed == threshold) and S4 (alreadyUsed + a matched pending pod's request ==
    # threshold) on a resource column and on the pod count
    s3 = s3c = s4 = s4c = 0
    for t in np.nonzero(live & (np.diff(snap.ovr_off) == 0))[0]:
        already = [int(res.used[r, t]) + int(snap.reserved[r, t]) for r in range(R)]
        cnt = int(res.used_cnt[t]) + int(snap.reserved_cnt[t])
        has = _bits(snap.thr_present[t:t + 1], R)[:, 0]
        s3 += any(has[r] and already[r] == int(snap.thr[r, t]) for r in range(R))
        has_cnt = (int(snap.thr_present[t]) & abi.COUNT_BIT) != 0
        s3c += has_cnt and cnt == int(snap.thr_cnt[t])
        s4c += has_cnt and cnt + 1 == int(snap.thr_cnt[t])
        for i in np.nonzero(_matched(res.pend_bitmap, t))[0]:
            if any(has[r] and present[1][r, i] and snap.pending.req[r, i] != 0 and already[r] + int(snap.pending.req[r, i]) == int(snap.thr[r, t])
                   for r in range(R)):
                s4 += 1
                break
    assert min(s3, s3c, s4, s4c) >= 3, (s3, s3c, s4, s4c)


def test_value_regimes_refuse_what_the_domain_cannot_hold():
    with pytest.raises(ValueError):
        synth.generate("C2", values="wide")  # 110k pods: no room above 2^44 under the 2^62 column bound
    with pytest.raises(ValueError):
        synth.generate("C2", m=40, n=70, p=33, values="huge")
