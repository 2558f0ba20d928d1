"""The selector-table compiler (csrc/kt_tables.cc) checked WITHOUT a GPU.

kt_debug_compile_tables hands back the bit-sliced tables kt_upload_throttles would put into HBM; this test walks them with
numpy exactly as the kernels do (label -> row through keydir/valrow or the hash, AND of `sat`, bit-sliced count of `pos`
against `need`, namespace mask, OR over term planes) and requires the resulting pod x throttle relation to equal the
oracle's, for both pod kinds.  It is a test-side emulation of the device algorithm: the product has no such code path."""
import ctypes as C

import numpy as np
import pytest

from kube_throttler_b200 import abi, synth

KOTHER = 0xFFFFFFFE


def compile_tables(kt, snap):
    L = kt.lib()
    lim = abi.Limits(abi.ABI_VERSION, snap.R, snap.L, snap.LN)
    cols, sel = snap.throttle_cols(), snap.selector_table()
    dims = np.zeros(12, np.int32)
    args = [C.byref(lim), snap.m, C.byref(cols), C.byref(sel), snap.n_ns, abi.ptr(snap.ns_labels), dims.ctypes.data]
    assert L.kt_debug_compile_tables(*args, *([None] * 8)) == 0
    M, W, Wp, TPpad, B, rows, NS, nkd, nvr, nnsw, _, hslots = (int(x) for x in dims)
    t = dict(table=np.zeros((W, rows, TPpad, 2), np.uint32), need=np.zeros((W, TPpad, B), np.uint32), nsmask=np.zeros((NS, W, TPpad), np.uint32),
             nsw_off=np.zeros(NS + 1, np.int32), nsw_idx=np.zeros(max(nnsw, 1), np.int32), keydir=np.zeros((nkd + 1, 4), np.uint32),
             valrow=np.zeros(nvr, np.uint32), hash=np.zeros((hslots, 4), np.uint32))
    assert L.kt_debug_compile_tables(*args, *(t[k].ctypes.data for k in ("table", "need", "nsmask", "nsw_off", "nsw_idx", "keydir", "valrow", "hash"))) == 0
    t.update(M=M, W=W, Wp=Wp, TPpad=TPpad, B=B, rows=rows, NS=NS, n_keydir=nkd, hash_mask=hslots - 1)
    return t


def label_hash(key, val):
    h = (key * 0x9E3779B1 + val * 0x85EBCA77) & 0xFFFFFFFF
    h ^= h >> 16
    h = (h * 0x7FEB352D) & 0xFFFFFFFF
    return h ^ (h >> 15)


def hash_row(t, key, val):
    for v in (val, 0xFFFFFFFF):
        slot = label_hash(key, v) & t["hash_mask"]
        while True:
            e = t["hash"][slot]
            if e[0] == key and e[1] == v:
                return int(e[2])
            if (e[0] & e[1]) == 0xFFFFFFFF:
                break
            slot = (slot + 1) & t["hash_mask"]
    return t["rows"] - 1


def rows_of_labels(t, labels):
    """[L][n] int64 labels -> [L][n] row indices (the kernels' translate8)."""
    row_bytes = t["TPpad"] * 8
    neutral = t["rows"] - 1
    out = np.full(labels.shape, neutral, np.int64)
    key, val = (labels >> 32) & 0xFFFFFFFF, labels & 0xFFFFFFFF
    for idx in np.ndindex(labels.shape):
        if labels[idx] == abi.LABEL_EMPTY:
            continue
        k, v = int(key[idx]), int(val[idx])
        ke = t["keydir"][min(k, t["n_keydir"])]
        if t["n_keydir"] == 0 or ke[3] == 0xFFFFFFFF:
            out[idx] = hash_row(t, k, v)
            continue
        d = (v - int(ke[1])) & 0xFFFFFFFF
        vr = int(t["valrow"][int(ke[3]) + d]) if d < int(ke[2]) else KOTHER
        out[idx] = (vr if vr != KOTHER else int(ke[0])) // row_bytes
    return out


def match_bitmap(t, pods, counted_only):
    n = pods.n
    rows = rows_of_labels(t, pods.labels)
    bm = np.zeros((n, t["Wp"]), np.uint32)
    ok = np.ones(n, bool)
    if counted_only:
        need_flags = abi.POD_SCHEDULER_MATCH | abi.POD_SCHEDULED
        ok = (pods.flags & need_flags) == need_flags
    ok &= (pods.ns_id >= 0) & (pods.ns_id < t["NS"])
    for p in np.nonzero(ok)[0]:
        ns = int(pods.ns_id[p])
        for w in t["nsw_idx"][t["nsw_off"][ns]:t["nsw_off"][ns + 1]]:
            word = 0
            for s in range(t["TPpad"]):
                sat = int(t["nsmask"][ns, w, s])
                cnt = [0] * t["B"]
                for r in rows[:, p]:
                    e = t["table"][w, r, s]
                    sat &= int(e[0])
                    carry = int(e[1])
                    for b in range(t["B"]):
                        cnt[b], carry = cnt[b] ^ carry, cnt[b] & carry
                m = sat
                for b in range(t["B"]):
                    m &= ~(cnt[b] ^ int(t["need"][w, s, b])) & 0xFFFFFFFF
                word |= m
            bm[p, w] = word
    return bm


@pytest.mark.parametrize("kw", [
    dict(config="C1"),
    dict(config="C2", m=96, n=700, p=200),
    dict(config="C3", m=150, n=900, p=250),                       # ClusterThrottles with namespace selectors
    dict(config="C2", m=80, n=600, p=150, L=12, q_max=6),         # 6-bit counters, more label slots
    dict(config="C3", m=100, n=500, p=120, sort_by_namespace=False),
    dict(config="C3", m=150, n=900, p=250, column_layout=True),   # ClusterThrottles in the order the host layer lays its columns out in
])
def test_compiled_tables_reproduce_the_oracle_relation(kt, oracle, kw):
    kw = dict(kw)
    snap = synth.generate(kw.pop("config"), **kw)
    t = compile_tables(kt, snap)
    want = oracle.columnar_evaluate(snap, words_per_row=t["Wp"])
    np.testing.assert_array_equal(match_bitmap(t, snap.running, True), want.run_bitmap)
    np.testing.assert_array_equal(match_bitmap(t, snap.pending, False), want.pend_bitmap)


@pytest.mark.parametrize("config,terms,tppad", [
    ("C2", 1, 1), ("C3", 1, 1),   # one term per throttle: one plane per table entry
    ("C2", 3, 4), ("C3", 3, 4),   # up to three: two plane pairs, the fourth plane padding
    ("C2", 4, 4), ("C3", 4, 4),   # up to four: two full plane pairs
])
def test_term_planes(kt, oracle, config, terms, tppad):
    """synth terms=1 / 3 / 4 give the table compiler one plane per entry or two plane pairs; the relation still equals the
    oracle's, and a plane beyond a throttle's own terms (the padded plane when TP = 3) can match no pod: its namespace mask and
    its needed counts are zero."""
    snap = synth.generate(config, m=150, n=900, p=250, terms=terms)
    nterms = np.diff(snap.term_off)
    assert nterms.max() == terms and nterms.min() == 1
    t = compile_tables(kt, snap)
    assert t["TPpad"] == tppad
    want = oracle.columnar_evaluate(snap, words_per_row=t["Wp"])
    np.testing.assert_array_equal(match_bitmap(t, snap.running, True), want.run_bitmap)
    np.testing.assert_array_equal(match_bitmap(t, snap.pending, False), want.pend_bitmap)
    w = np.arange(snap.m) >> 5
    bit = np.uint32(1) << (np.arange(snap.m) & 31).astype(np.uint32)
    for s in range(tppad):
        unused = nterms <= s
        assert not (t["nsmask"][:, w[unused], s] & bit[unused]).any(), f"plane {s}"
        assert not (t["need"][w[unused], s, :] & bit[unused][:, None]).any(), f"plane {s}"
        if s < terms:
            assert t["nsmask"][:, :, s].any(), f"plane {s} is never used"
    if terms == 3:
        assert not t["nsmask"][:, :, 3].any() and not t["need"][:, 3, :].any()


def test_sparse_ids_take_the_hash(kt, oracle):
    from test_gpu_parity import _remap_label_ids

    snap = _remap_label_ids(synth.generate("C3", m=100, n=500, p=120), lambda k: k * 7919 + 70000, lambda v: v * 1009 + 5)
    t = compile_tables(kt, snap)
    assert t["n_keydir"] == 0  # key ids beyond the direct table
    want = oracle.columnar_evaluate(snap, words_per_row=t["Wp"])
    np.testing.assert_array_equal(match_bitmap(t, snap.pending, False), want.pend_bitmap)
    snap = _remap_label_ids(synth.generate("C3", m=100, n=500, p=120), lambda k: k, lambda v: v * 1000003 % (1 << 31))
    t = compile_tables(kt, snap)
    assert t["n_keydir"] > 0 and (t["keydir"][:, 3] == 0xFFFFFFFF).any()  # direct keys, hashed values
    want = oracle.columnar_evaluate(snap, words_per_row=t["Wp"])
    np.testing.assert_array_equal(match_bitmap(t, snap.pending, False), want.pend_bitmap)


def test_column_layout_shortens_the_namespaces_word_lists(kt):
    """What a pass costs per pod is the length of its namespace's word list.  With the ClusterThrottles ordered by the set of
    namespaces their namespaceSelectors admit (what kt_host.cc does with its device columns; synth column_layout=True) a C3-shaped
    table has markedly shorter lists than in the generator's random order."""
    words = {}
    for layout in (False, True):
        snap = synth.generate("C3", m=1000, n=2000, p=200, calibrate=False, column_layout=layout)
        t = compile_tables(kt, snap)
        ln = np.diff(t["nsw_off"])
        cnt = np.bincount(snap.running.ns_id, minlength=snap.n_ns)
        words[layout] = float((ln * cnt).sum() / cnt.sum())
    assert words[True] < 0.7 * words[False], words
