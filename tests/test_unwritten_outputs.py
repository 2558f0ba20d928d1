"""Outputs a pass does not write read as zeros, never as what the allocator handed back.

A check-only pass (every PreFilter pass, the first step of kt_admit_queue) leaves the running match bitmap alone, and a
reconcile-only pass the pending bitmap, codes and admit bytes.  When such a pass is the first one after the buffers were
allocated, the getters used to deliver whatever device memory a freed context had left there -- so two engines holding the same
rows could answer differently.  Each test first frees an engine whose outputs were all written (non-zero), then asks a fresh
engine of the same shape."""
import numpy as np
import pytest

from kube_throttler_b200 import abi, synth
from test_check_rows import with_status

pytestmark = pytest.mark.gpu

CHK_ONLY = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE
REC_ONLY = abi.EVAL_FRESH_STATUS | abi.EVAL_SKIP_CHECK


def dirty_the_allocator(kt, snap):
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    eng.evaluate(snap.now)
    d = eng.download()
    assert d.run_bitmap.any() and d.pend_bitmap.any() and d.codes.any() and d.admit.any()
    eng.close()


@pytest.mark.parametrize("mode", [abi.ROW_ORDER_BY_NAMESPACE, abi.ROW_ORDER_AS_GIVEN])
def test_running_bitmap_after_a_first_check_only_pass(kt, oracle, mode):
    snap = synth.generate("C2", m=200, n=4000, p=2600, sort_by_namespace=False)
    dirty_the_allocator(kt, snap)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.set_row_order(abi.PODS_RUNNING, mode)
    with_status(eng, snap, oracle, np.random.default_rng(3))
    eng.admit_queue(0, snap.pending.n)
    words = np.zeros((snap.running.n, eng.words_per_row), np.uint32)
    eng._ck(eng._L.kt_get_match_bitmap(eng._h, abi.PODS_RUNNING, abi.ptr(words)))
    assert not words.any()
    eng.close()


def test_pending_outputs_after_a_first_reconcile_only_pass(kt):
    snap = synth.generate("C2", m=200, n=4000, p=2600)
    dirty_the_allocator(kt, snap)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    eng.evaluate(snap.now, REC_ONLY)
    d = eng.download()
    assert not d.pend_bitmap.any() and not d.codes.any() and not d.admit.any()
    assert d.run_bitmap.any()
    eng.close()
