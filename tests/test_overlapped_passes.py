"""Fused passes queued back to back whose first phase runs while the pass ahead of them still decides (early passes).

A fused pass (k_pass) queued right behind another one of this library, of another context or of the same one when neither
zero-fills, waits for it only once a CTA leaves its first phase: its match tiles, pre-records and reconcile tiles run beside
the previous pass's status and decide work.  Everything that first phase writes is therefore either its own (counters and
pre-records by pass parity, the partial-sum half of its parity) or rewritten with the value the previous pass reads.

Every case parks the stream behind one bounded spin kernel (torch.cuda._sleep, as in test_queued_passes.py), queues fused
passes whose `now` and flags make their codes differ in many rows, and compares what the getters read with the columnar oracle
of the last pass, and with the same queue synchronised after every pass.  A predecessor's grid is capped
(kt_debug_set_pass_plan) so that it still decides, on a few CTAs, long after its successor has been placed; the in-kernel
trace of both shows that the successor's tiles did begin before the predecessor's last CTA exited.  Every case runs once.
"""
import numpy as np
import pytest

from kube_throttler_b200 import abi
from test_partial_passes import check_diff, check_sparse
from test_queued_passes import DAY, SEQ_WORLD, WORLDS, World, assert_identical, assert_parked, check_result, park, torch_mod

pytestmark = pytest.mark.gpu

FRESH, GIVEN, ON_EQUAL = abi.EVAL_FRESH_STATUS, abi.EVAL_GIVEN_STATUS, abi.EVAL_ON_EQUAL
RUN, PEND = abi.PODS_RUNNING, abi.PODS_PENDING
# whole passes of every view: FRESH decides against this pass's sums, GIVEN against the observed status (the two views' codes
# differ in many rows: World.views_differ), ON_EQUAL moves the boundary of both
FUSED_FLAGS = (FRESH, GIVEN | ON_EQUAL, FRESH | ON_EQUAL, GIVEN, FRESH)
CAP = 2  # CTAs of a capped predecessor: its status and decide pieces take many rounds after it has let its successor start


def queue_sequence(w, nows, synced):
    eng = w.eng
    for i, flags in enumerate(FUSED_FLAGS):
        eng.evaluate(nows[i % len(nows)], flags)
        if synced:
            eng.sync()


def check_last(w, got, flags, now, cap=None):
    want = w.want(flags, now)
    check_result(w, got, want, True)
    check_diff(w.eng, w.snap, got, w.snap.status)
    if cap:
        check_sparse(w.eng, want.codes, want.admit, cap)


# worlds with overrides, so that the two `now` values switch some on and off (other thresholds, other codes)
ONE_CONTEXT_WORLDS = {"seq": SEQ_WORLD, "c2": dict(config="C2", override_frac=0.3)}


@pytest.mark.parametrize("world", list(ONE_CONTEXT_WORLDS))
def test_fused_queue_one_context(kt, oracle, world):
    """Five fused passes of alternating views and `now` on ONE context behind one park, with the sparse check list on: the
    last pass's bitmaps, codes, admit bits, status columns, changed list, sums and sparse list against the oracle, and the same
    bits as the queue synchronised after every pass."""
    w = World(kt, oracle, ONE_CONTEXT_WORLDS[world], 11)
    try:
        eng, snap = w.eng, w.snap
        w.views_differ()
        nows = (snap.now, snap.now - 40 * DAY)
        assert (w.want(FRESH, nows[0]).override_active != w.want(FRESH, nows[1]).override_active).any(), "these `now` values switch no override"
        cap = 2 * w.W * snap.pending.n + 64
        eng.set_sparse_check(cap)
        w.warm()
        for flags in FUSED_FLAGS:
            eng.evaluate(snap.now, flags)
            eng.sync()
        park(w.stream)
        queue_sequence(w, nows, synced=False)
        assert_parked(w.stream)
        got = eng.download()
        last = (FUSED_FLAGS[-1], nows[(len(FUSED_FLAGS) - 1) % len(nows)])
        check_last(w, got, *last, cap=cap)
        queue_sequence(w, nows, synced=True)
        synced = eng.download()
        assert_identical(snap, got, synced)
    finally:
        w.close()


def trace_of(eng):
    rows, roles = eng.trace()
    first = int(roles[0]) + int(roles[1])
    return rows[:first], rows


def test_fused_passes_overlap_across_contexts(kt, oracle):
    """Two contexts on one stream, A's grid capped to two CTAs: A, B, A, B queued behind one park.  B's first phase overlaps
    A's decide work (the trace: a tile of B began before A's last CTA exited) and every context's last pass equals the oracle
    and the same queue synchronised after every pass."""
    torch = torch_mod()
    stream = torch.cuda.Stream()
    ws = [World(kt, oracle, dict(WORLDS["small_fast"], seed=71 + i), 21 + i, stream) for i in range(2)]
    try:
        a, b = ws
        for w in ws:
            w.views_differ()
            w.warm()
        a.eng.set_pass_plan(max_ctas=CAP)
        for w in ws:
            w.eng.enable_trace(True)
        seq = [(a, FRESH), (b, GIVEN | ON_EQUAL), (a, GIVEN), (b, FRESH | ON_EQUAL)]

        def run(synced):
            for w, flags in seq:
                w.eng.evaluate(w.snap.now, flags)
                if synced:
                    w.eng.sync()

        for w, _ in seq:  # every kernel and buffer of the queue exists before the park
            w.eng.evaluate(w.snap.now, FRESH)
        torch.cuda.synchronize()
        park(stream)
        run(synced=False)
        assert_parked(stream)
        torch.cuda.synchronize()
        a_first, a_rows = trace_of(a.eng)
        b_first, _ = trace_of(b.eng)
        assert a.eng.pass_plan().grid == CAP
        exits = a_rows[:, 29][a_rows[:, 29] > 0]
        starts = b_first[:, 2]
        assert exits.shape[0] == CAP and (starts > 0).all()
        assert starts.min() < exits.max(), "B's first tile began only after A's last CTA exited: the passes did not overlap"
        got = [w.eng.download() for w in ws]
        for w, (_, flags) in zip(ws, seq[2:]):
            check_last(w, got[ws.index(w)], flags, w.snap.now)
        run(synced=True)
        for w, g in zip(ws, got):
            assert_identical(w.snap, g, w.eng.download())
    finally:
        for w in ws:
            w.eng.set_pass_plan()
            w.eng.enable_trace(False)
            w.close()


def test_zero_filling_pass_after_upload(kt, oracle):
    """New pending rows uploaded asynchronously behind the park, then two fused passes of different views on that context,
    right behind a capped pass of another context: the first of the two zero-fills (its successor is not let start early) and
    the second one's outputs equal the oracle on the new rows."""
    import copy

    from test_queued_passes import make, pinned_wide, rows_of

    torch = torch_mod()
    stream = torch.cuda.Stream()
    kw = WORLDS["small_fast"]
    a = World(kt, oracle, dict(kw, seed=81), 31, stream)
    b = World(kt, oracle, dict(kw, seed=82), 32, stream)
    keep = []
    try:
        for w in (a, b):
            w.warm()
        new = copy.copy(b.snap)
        new.pending = rows_of(b.snap, make(dict(kw, seed=83))).pending
        new.normalize()
        cols = pinned_wide(new.pending, keep)
        a.eng.set_pass_plan(max_ctas=CAP)
        b.eng.set_async_uploads(True)
        b.eng.upload_pods(PEND, cols)  # staging buffers reach their sizes before the park
        b.eng.evaluate(b.snap.now, FRESH)
        torch.cuda.synchronize()
        park(stream)
        a.eng.evaluate(a.snap.now, FRESH)
        b.eng.upload_pods(PEND, cols)
        b.eng.evaluate(b.snap.now, GIVEN | ON_EQUAL)  # zero-fills: new rows
        b.eng.evaluate(b.snap.now, FRESH)
        assert_parked(stream)
        got = b.eng.download()
        want = oracle.columnar_evaluate(new, FRESH, words_per_row=got.words_per_row)
        given = oracle.columnar_evaluate(new, GIVEN | ON_EQUAL, words_per_row=got.words_per_row)
        assert (want.codes != given.codes).any(axis=1).sum() >= 1
        from test_gpu_parity import assert_same

        assert_same(new, got, want)
        assert_same(a.snap, a.eng.download(), a.want(FRESH))
    finally:
        a.eng.set_pass_plan()
        b.eng.set_async_uploads(False)
        torch.cuda.synchronize()
        for w in (a, b):
            w.close()
        del keep
