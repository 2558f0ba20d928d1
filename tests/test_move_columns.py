"""kt_move_throttle_columns: the throttle columns laid out again on the device -- column j taking previous column src[j], or an
empty column for -1 -- without compiling the selector tables.

Two engines hold the same pods, namespaces, throttles, observed status and reservations.  One gets every change as a whole
kt_upload_throttles of the gathered spec followed by the gathered status and reservations; the other gets kt_move_throttle_columns.
Moves: the identity, a reversal, random shuffles across 32-column words and 128-column (Wp) boundaries, compactions of 10% and
60% holes, growth with -1 columns, shrinking to a size that is not a multiple of 32, and m = 0.  Moves are followed by hole fills
through the selector and threshold deltas, appends, and status, reservation and namespace-row deltas; a fill or an append that
fits the resident tables must stay in place (recompiled = 0), which needs the engine's host copy of the tables to follow the
move.  After every step both engines must answer bit for bit alike (FRESH, GIVEN and ON_EQUAL passes under every forced pass
plan, the status diff, the check summary, the keyed calls, kt_admit_queue, the check rows), equal the columnar oracle, and hold
the namespace word lists kt_debug_compile_tables builds for the gathered spec (and its masks where the term-plane counts
agree)."""
import copy
import ctypes as C

import numpy as np
import pytest

from kube_throttler_b200 import abi, synth
from test_append_rows import code, engines, fits, pack_thr, thr_columns, vocab_of
from test_namespace_rows import PLANS, WORLDS, GIVEN, assert_oracle, assert_same, observe, synth_words
from test_partial_passes import observed_status
from test_selector_rows import columns, pack
from test_tables_cpu import compile_tables
from test_threshold_rows import rand_override

pytestmark = pytest.mark.gpu


def empty_col():
    return [abi.KIND_CLUSTERTHROTTLE, -1, 0, []]


class World:
    """The current throttle side (selector columns, threshold columns, status, reservations) over a fixed pod and namespace side."""

    def __init__(self, base, cols, tcols, status, reserved):
        self.base, self.cols, self.tcols, self.status, self.reserved = base, cols, tcols, status, reserved

    def snap(self):
        s = copy.copy(self.base)
        for f, v in dict(pack(self.cols), **pack_thr(self.tcols, s.R)).items():
            setattr(s, f, v)
        s.status = self.status
        s.reserved, s.reserved_present, s.reserved_cnt = self.reserved
        return s.normalize()

    def move(self, src):
        """Column j takes column src[j], or an empty one for -1."""
        R = self.base.R
        take = np.array([max(int(s), 0) for s in src], np.int64)
        hole = np.array([s < 0 for s in src], bool)
        self.cols = [list(self.cols[s]) if s >= 0 else empty_col() for s in src]
        self.tcols = [self.tcols[s] if s >= 0 else (np.zeros(R, np.int64), 0, 0, []) for s in src]

        def gather(v):
            if v.shape[-1] == 0:
                return np.zeros(v.shape[:-1] + (len(src),), v.dtype)
            g = v[..., take].copy()
            g[..., hole] = 0
            return g

        self.status = {f: gather(v) for f, v in self.status.items()}
        self.reserved = tuple(gather(v) for v in self.reserved)


def ns_lists_match(kt, eng, snap, where):
    """The resident word lists equal the table compiler's for the gathered spec (the resident namespace count is kept: namespaces
    beyond the compiler's have empty lists); the masks too when the term planes and namespace counts agree."""
    got, want = eng.ns_tables(), compile_tables(kt, snap)
    ns = min(len(got["nsw_off"]), len(want["nsw_off"])) - 1
    n = int(want["nsw_off"][ns])
    np.testing.assert_array_equal(got["nsw_off"][:ns + 1], want["nsw_off"][:ns + 1], err_msg=where)
    assert (got["nsw_off"][ns:] == n).all() and (want["nsw_off"][ns:] == n).all(), where
    np.testing.assert_array_equal(got["nsw_idx"][:n], want["nsw_idx"][:n], err_msg=where)
    if got["nsmask"].shape == want["nsmask"].shape:
        np.testing.assert_array_equal(got["nsmask"], want["nsmask"], err_msg=where)


def full_upload(e, snap):
    e.upload_throttles(snap)
    e.upload_status(snap)
    e.set_reserved(snap)


def moves(rng, m):
    """The moves in order, each a function of the current column count."""
    def shuffle_across(m):  # swaps inside a word, across words and across 128-column boundaries
        src = np.arange(m)
        for _ in range(max(1, m // 4)):
            a, b = rng.integers(0, m, size=2)
            src[[a, b]] = src[[b, a]]
        return src

    def compact(frac):
        def f(m):
            keep = np.sort(rng.choice(m, size=m - int(round(m * frac)), replace=False))
            return keep
        return f

    def grow(m):  # -1 columns between and after the existing ones: crosses word and Wp boundaries
        src = list(range(m))
        for _ in range(40):
            src.insert(int(rng.integers(0, len(src) + 1)), -1)
        return np.array(src + [-1] * (160 - (len(src) % 32)))

    return [("identity", lambda m: np.arange(m)), ("reverse", lambda m: np.arange(m)[::-1]), ("permute", lambda m: rng.permutation(m)),
            ("shuffle", shuffle_across), ("compact10", compact(0.1)), ("grow", grow), ("compact60", compact(0.6)),
            ("shrink", lambda m: np.sort(rng.choice(m, size=min(m, 45), replace=False))), ("zero", lambda m: np.zeros(0, np.int64)),
            ("grow_from_zero", lambda m: np.full(70, -1)), ("permute", lambda m: rng.permutation(m))]


@pytest.mark.parametrize("world", list(WORLDS))
def test_moves_equal_full_uploads(kt, oracle, world):
    full_snap = WORLDS[world]()
    rng = np.random.default_rng(sum(map(ord, world)) + 31)
    pool_cols, pool_thr = columns(full_snap), thr_columns(full_snap)
    pool_status = observed_status(oracle.columnar_evaluate(full_snap, abi.EVAL_FRESH_STATUS, words_per_row=synth_words(full_snap)), full_snap, rng)
    R, L, n_pool = full_snap.R, full_snap.L, full_snap.m
    for t in range(0, n_pool, 3):  # temporaryThresholdOverrides on every third column
        pool_thr[t] = pool_thr[t][:3] + ([rand_override(rng, R, full_snap.now, False) for _ in range(1 + (t // 3) % 3)],)
    reserved = (full_snap.reserved.copy(), full_snap.reserved_present.copy(), full_snap.reserved_cnt.copy()) if full_snap.reserved is not None \
        else (np.zeros((R, n_pool), np.int64), np.zeros(n_pool, np.uint32), np.zeros(n_pool, np.int64))
    w = World(full_snap, [list(c) for c in pool_cols], list(pool_thr), {f: v.copy() for f, v in pool_status.items()}, reserved)
    full, delta = engines(kt, w.snap())
    res, vocab = compile_tables(kt, w.snap()), vocab_of(w.cols)  # the resident tables: moves keep them
    ok = [t for t in range(n_pool) if fits(pool_cols[t], vocab, res, L)]
    nxt = 0
    for step, (name, make) in enumerate(moves(rng, n_pool)):
        src = np.asarray(make(len(w.cols)), np.int64)
        w.move(src)
        snap = w.snap()
        full_upload(full, snap)
        delta.move_throttle_columns(src)
        assert delta.m == snap.m == len(src)
        m = snap.m
        where = f"{world} step {step} {name} m={m}"
        check(kt, oracle, full, delta, snap, rng, step, where)
        if m == 0:
            continue
        # the empty columns (or, without any, a few deleted ones) filled through the selector and threshold deltas, with a status
        # and a reservation: in place, since the fills fit the resident tables
        holes = np.flatnonzero(src < 0).astype(np.int32)
        if holes.size == 0:
            holes = np.sort(rng.choice(m, size=min(m, 5), replace=False)).astype(np.int32)
            for t in holes:
                w.cols[t] = [w.cols[t][0], w.cols[t][1], 0, []]
            full_upload(full, w.snap())
            assert delta.update_selector_rows(holes, pack([w.cols[t] for t in holes])) is False, where
        holes = holes[rng.random(holes.size) < 0.7] if holes.size > 3 else holes
        for t in holes:
            s = ok[nxt % len(ok)]
            nxt += 1
            w.cols[t], w.tcols[t] = list(pool_cols[s]), pool_thr[s]
            for f, v in w.status.items():
                v[..., t] = pool_status[f][..., s]
            w.reserved[0][0, t] = int(rng.integers(0, 3000))
            w.reserved[1][t] |= 1
            w.reserved[2][t] = int(rng.integers(0, 4))
        snap = w.snap()
        full_upload(full, snap)
        if holes.size:
            assert delta.update_selector_rows(holes, pack([w.cols[t] for t in holes])) is False, where
            delta.update_threshold_rows(holes, pack_thr([w.tcols[t] for t in holes], R))
            delta.update_status_rows(holes, {f: (v[:, holes] if v.ndim == 2 else v[holes]) for f, v in w.status.items()})
            delta.update_reserved_rows(holes, w.reserved[0][:, holes], w.reserved[1][holes], w.reserved[2][holes])
        if step % 2 == 0:  # an append that fits: in place after the move
            k = int(rng.integers(1, 40))
            new = [ok[(nxt + i) % len(ok)] for i in range(k)]
            nxt += k
            new_cols, new_thr = [list(pool_cols[t]) for t in new], [pool_thr[t] for t in new]
            w.cols += new_cols
            w.tcols += new_thr
            w.status = {f: np.concatenate([v, np.zeros((R, k) if v.ndim == 2 else k, v.dtype)], axis=v.ndim - 1) for f, v in w.status.items()}
            w.reserved = tuple(np.concatenate([v, np.zeros(v.shape[:-1] + (k,), v.dtype)], axis=v.ndim - 1) for v in w.reserved)
            full_upload(full, w.snap())
            assert delta.append_throttle_rows(dict(pack(new_cols), **pack_thr(new_thr, R))) is False, where
        else:  # a namespace relabel on both engines
            nsr = np.array([int(rng.integers(0, w.base.n_ns))], np.int32)
            w.base = copy.copy(w.base)
            w.base.ns_labels = w.base.ns_labels.copy()
            w.base.ns_labels[:, nsr[0]] = w.base.ns_labels[:, int(rng.integers(0, w.base.n_ns))]
            snap = w.snap()
            for e in (full, delta):
                e.update_namespace_rows(snap.n_ns, nsr, snap.ns_labels[:, nsr])
        check(kt, oracle, full, delta, w.snap(), rng, step, where + " then fills")
    full.close()
    delta.close()


def check(kt, oracle, full, delta, snap, rng, step, where):
    assert full.words_per_row == delta.words_per_row, where
    ns_lists_match(kt, delta, snap, where)
    ns_lists_match(kt, full, snap, where)
    m = snap.m
    if m == 0:  # no throttle: a pass writes no running bitmap row and no status diff, so only the checks are compared
        got = []
        for e in (full, delta):
            e.evaluate(snap.now, abi.EVAL_FRESH_STATUS)
            r = e.download()
            got.append([r.pend_bitmap, r.codes, r.admit, *e.check_summary(0, snap.pending.n), *e.admit_queue(0, snap.pending.n)])
        assert_same(*got, where)
        return
    assert_oracle(delta, snap, oracle, where)
    rows = rng.integers(0, snap.pending.n, size=min(snap.pending.n, 19))
    idx = rng.choice(m, size=min(m, 9), replace=False).astype(np.int32)
    probe = (rows, idx, snap.pending.labels[:, rows], snap.pending.ns_id[rows].astype(np.int32))
    plan = PLANS[step % len(PLANS)]
    assert_same(observe(full, snap, plan, probe), observe(delta, snap, plan, probe), where + f" plan {plan}")


def test_argument_and_state_errors(kt):
    snap = synth.generate("C3", m=40, n=200, p=50, n_ns=6).normalize()
    e = kt.Engine(snap.R, snap.L, snap.LN)
    L, h = e._L, e._h

    def call(m, src):
        a = None if src is None else np.ascontiguousarray(src, np.int32)
        return L.kt_move_throttle_columns(h, m, abi.ptr(a))

    assert call(1, [0]) == abi.ERR_STATE  # before kt_upload_throttles
    assert call(-1, None) == abi.ERR_INVALID
    e.upload_namespaces(snap.ns_labels)
    e.upload_throttles(snap)
    M = snap.m
    assert call(-1, None) == abi.ERR_INVALID
    assert call(3, None) == abi.ERR_INVALID
    assert call(2, [0, M]) == abi.ERR_INVALID
    assert call(2, [-2, 0]) == abi.ERR_INVALID
    assert call(3, [5, 1, 5]) == abi.ERR_INVALID
    # nothing was moved by the rejected calls
    assert e.m == M and e.words_per_row == 4
    dims = np.zeros(5, np.int32)
    assert L.kt_debug_get_ns_tables(h, abi.ptr(dims), None, None, None) == 0
    assert int(dims[3]) == (M + 31) // 32
    # -1 may repeat; no status before the call: still none after it
    e.move_throttle_columns([-1, 3, -1, 0])
    assert e.m == 4
    assert code(lambda: e.evaluate(0, GIVEN)) == abi.ERR_STATE
    # a status held before the call is kept, and a pass is needed again before the getters that read one
    s2 = copy.copy(snap)
    cols, tcols = columns(snap), thr_columns(snap)
    for f, v in dict(pack([cols[3], cols[0]]), **pack_thr([tcols[3], tcols[0]], snap.R)).items():
        setattr(s2, f, v)
    s2.status = {f: np.zeros((snap.R, 2) if f in ("calc_thr", "used") else 2, np.uint8 if f == "calculated" else np.int64)
                 for f in ("calculated", "calc_thr", "calc_present", "calc_cnt", "used", "used_present", "used_cnt", "throttled")}
    s2.reserved, s2.reserved_present, s2.reserved_cnt = np.zeros((snap.R, 2), np.int64), np.zeros(2, np.uint32), np.zeros(2, np.int64)
    s2.normalize()
    e.move_throttle_columns([1, 3])
    e.upload_status(s2)
    e.evaluate(s2.now, abi.EVAL_FRESH_STATUS)
    e.get_changed()
    e.move_throttle_columns([1, 0, -1])
    assert e.m == 3 and e.words_per_row == 4
    assert code(lambda: e.get_changed()) == abi.ERR_STATE
    e.evaluate(0, GIVEN)  # (GIVEN needs the status: still held)
    # m = 0, with a null src
    assert call(0, None) == abi.OK
    assert e.m == 3  # (the binding's count: the raw call does not update it)
    assert L.kt_debug_get_ns_tables(h, abi.ptr(dims), None, None, None) == 0
    assert int(dims[3]) == 1 and L.kt_match_words(h) == 4
    e.close()
