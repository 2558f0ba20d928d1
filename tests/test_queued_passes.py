"""Passes queued back to back, engines on a caller's stream, async uploads and stream switches, against the columnar oracle.

kt_evaluate is asynchronous on the context stream: a caller may queue pass after pass, run several engines on one stream of
its own (kt_set_stream) and let uploads return as soon as their copies are queued (kt_set_async_uploads) -- bench.py does all
three.  The other GPU tests synchronise after every pass, so a pass that starts before the one ahead of it has finished, or a
stream switch that lets copies queued on the old stream land after the next pass, cannot fail there.

Here the engine's stream is first parked behind one bounded spin kernel (torch.cuda._sleep), so that everything a case queues
is in the stream before the first of it runs; `stream.query()` still False after queuing shows that no call synchronised in
between.  The results are then read with the getters and compared bit for bit with the columnar oracle under each pass's own
flags and `now`, and the same queue with eng.sync() after each pass must give the same bits.

A check-only pass (GIVEN_STATUS | SKIP_RECONCILE: PreFilter, and the first step of kt_admit_queue) decides against pre-records
that differ from a whole pass's (FRESH view): the observed status.used as base, the observed threshold, its own on_equal.  The
worlds lag the observed status behind the pods, hold reservations and meet thresholds exactly, and each test asserts that the
two views' codes differ in many rows, so a pass that decided against the other pass's records cannot go unnoticed.

Every case runs once: nothing is repeated to catch a race.  Uploads queued behind a park keep the row count (nothing is
reallocated) and the rows as given (no row map), so a pass that overtakes them reads stale rows, never freed memory.
"""
import copy

import numpy as np
import pytest

from kube_throttler_b200 import abi
from test_gpu_parity import _live, assert_same
from test_partial_passes import check_diff, check_sparse, observed_status, random_reserved, with_pending_of
from test_pass_plans import SHAPES, make

pytestmark = pytest.mark.gpu

FRESH, ON_EQUAL = abi.EVAL_FRESH_STATUS, abi.EVAL_ON_EQUAL
REC_ONLY = abi.EVAL_FRESH_STATUS | abi.EVAL_SKIP_CHECK
CHK_ONLY = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE
RUN, PEND = abi.PODS_RUNNING, abi.PODS_PENDING
DAY = 86400 * 10**9
PARK_CYCLES = 300_000_000  # one spin kernel of 0.15-0.2 s at H100 clocks: far longer than queuing any case here takes

# what a caller queues: kind -> (flags, timing, fused-pass grid cap)
KINDS = {
    "fused": (FRESH, False, 0),        # one k_pass
    # k_pass on a grid of 1 or 4 CTAs, with at least as many match tiles as status tiles: its match tiles write the pre-records
    # one tile after another, long after the next launch could have started
    "fused_cap1": (FRESH, False, 1),
    "fused_cap4": (FRESH, False, 4),
    "chained": (FRESH, True, 0),       # k_reconcile, k_finalize, k_check (timing on: plain launches)
    "reconcile_only": (REC_ONLY, False, 0),
    "check_only": (CHK_ONLY, False, 0),
    "check_only_on_equal": (CHK_ONLY | ON_EQUAL, False, 0),
}
SECONDS = ("check_only", "check_only_on_equal", "admit", "reconcile_only", "fused")
NOW_OFFSETS = (0, -40 * DAY, 10 * DAY)  # from snap.now: the overrides synth made active, almost none, another set

WORLDS = {
    # the grid of a pass is smaller than the device: the next launch's CTAs are placed at once.  P is raised so that the capped
    # fused passes have at least as many match tiles as status tiles (n_chk >= n_fin)
    "small_fast": dict(SHAPES["fast128_t2_r4"][0], p=2000),
    "small_general": dict(SHAPES["general_t2_b6"][0], p=3400),
    "c2": dict(config="C2"),  # BASELINE C2 at full size: 1k throttles x 100k running x 10k pending
}


def torch_mod():
    import torch

    return torch


def park(stream):
    torch = torch_mod()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(PARK_CYCLES)


def assert_parked(stream):
    assert not stream.query(), "an engine call synchronised while the passes were being queued"


class World:
    """A snapshot with a lagging observed status and reservations, its engine on a caller stream, and the oracle's results
    per (flags, now), computed once."""

    def __init__(self, kt, oracle, kw, seed, stream=None):
        torch = torch_mod()
        self.oracle = oracle
        self.snap = snap = make(kw)
        rng = np.random.default_rng(seed)
        snap.status = observed_status(oracle.columnar_evaluate(snap), snap, rng)
        snap.reserved, snap.reserved_present, snap.reserved_cnt = random_reserved(snap, rng)
        snap.normalize()
        self.stream = stream or torch.cuda.Stream()
        self.eng = kt.Engine(snap.R, snap.L, snap.LN)
        self.eng.set_stream(self.stream.cuda_stream)
        self.eng.upload_snapshot(snap)
        self.W = self.eng.words_per_row
        self._want = {}

    def want(self, flags, now=None):
        now = self.snap.now if now is None else now
        if (flags, now) not in self._want:
            s = copy.copy(self.snap)
            s.now = now
            self._want[flags, now] = self.oracle.columnar_evaluate(s, flags, words_per_row=self.W)
        return self._want[flags, now]

    def admit_range(self):
        P = self.snap.pending.n
        return P // 5, P // 2

    def want_admit(self):
        if "admit" not in self._want:
            first, count = self.admit_range()
            self._want["admit"] = self.oracle.columnar_admit_queue(self.snap, first, count, 0, words_per_row=self.W)
        return self._want["admit"]

    def views_differ(self):
        """The FRESH and the GIVEN view decide many rows differently, and ON_EQUAL changes some: a pass that decided against
        the other view's pre-records gives other codes."""
        P = self.snap.pending.n
        fresh, given, given_eq = self.want(FRESH), self.want(CHK_ONLY), self.want(CHK_ONLY | ON_EQUAL)
        for a, b, least in ((fresh, given, max(20, P // 50)), (fresh, given_eq, max(20, P // 50)), (given, given_eq, 1)):
            rows = int((a.codes != b.codes).any(axis=1).sum())
            assert rows >= least, (rows, least)

    def reset(self):
        """Automatic plan, timing off, and a whole pass at snap.now, synchronised: the state `expected` starts from."""
        self.eng.set_pass_plan()
        self.eng.enable_timing(False)
        self.eng.evaluate(self.snap.now, FRESH)
        self.eng.sync()

    def warm(self):
        """Every kind of pass once, synchronised: every kernel the cases launch is loaded before a stream is parked."""
        for kind in KINDS:
            queue(self.eng, kind, self.snap.now)
            self.eng.sync()
        self.reset()

    def close(self):
        torch_mod().cuda.synchronize()
        self.eng.close()


def queue(eng, kind, now):
    flags, timing, cap = KINDS[kind]
    eng.set_pass_plan(max_ctas=cap)
    eng.enable_timing(timing)
    eng.evaluate(now, flags)


def expected(w, seq):
    """(oracle result, whether the reconcile half is the last pass's) for what the getters read after the passes `seq` --
    (kind, now) pairs -- ran on a context that `reset` left: a reconcile-only pass leaves the pending outputs of the last
    checking pass, a check-only pass the reconcile outputs of the last reconciling one."""
    chk = w.want(FRESH)
    for kind, now in seq:
        flags = KINDS[kind][0]
        if not flags & abi.EVAL_SKIP_CHECK:
            chk = w.want(flags, now)
    kind, now = seq[-1]
    flags = KINDS[kind][0]
    want = w.want(flags, now)
    if flags & abi.EVAL_SKIP_CHECK:
        return with_pending_of(want, chk), True
    return want, not flags & abi.EVAL_SKIP_RECONCILE


def check_result(w, got, want, rec):
    assert_same(w.snap, got, want, check_reconcile=rec)
    if not rec:  # the running match rows are the same in every reconciling pass over these rows and tables
        np.testing.assert_array_equal(got.run_bitmap, w.want(FRESH).run_bitmap, err_msg="a check-only pass wrote the running match rows")


def assert_identical(snap, a, b):
    live = _live(snap)
    for f in ("pend_bitmap", "codes", "admit", "run_bitmap", "calc_thr", "calc_present", "calc_cnt", "override_active"):
        np.testing.assert_array_equal(getattr(a, f), getattr(b, f), err_msg=f)
    for f in ("used_present", "used_cnt", "throttled"):
        np.testing.assert_array_equal(getattr(a, f)[live], getattr(b, f)[live], err_msg=f)
    np.testing.assert_array_equal(a.used[:, live], b.used[:, live], err_msg="used")


# ---- 1. pass pairs with no host synchronisation between them ---------------------------------------------------------------
@pytest.fixture(scope="module")
def worlds(kt, oracle):
    made = {}

    def get(name):
        if name not in made:
            w = World(kt, oracle, WORLDS[name], 5)
            w.views_differ()
            w.warm()
            made[name] = w
        return made[name]

    yield get
    for w in made.values():
        w.close()


def run_pair(w, first, second, parked):
    eng, now = w.eng, w.snap.now
    w.reset()
    if parked:
        park(w.stream)
    queue(eng, first, now)
    if not parked:
        eng.sync()
    admitted = None
    if second == "admit":
        if parked:
            assert_parked(w.stream)  # kt_admit_queue waits for its own rounds: the check-only pass it starts with is queued first
        eng.set_pass_plan()
        eng.enable_timing(False)
        _, admitted = eng.admit_queue(*w.admit_range())
    else:
        queue(eng, second, now)
        if parked:
            assert_parked(w.stream)
    got = eng.download()
    eng.set_pass_plan()
    eng.enable_timing(False)
    return got, admitted


@pytest.mark.parametrize("first", list(KINDS))
@pytest.mark.parametrize("world", list(WORLDS))
def test_pass_pair_queued(worlds, world, first):
    """A pass of each kind, then at once -- behind one park -- a check-only pass with and without ON_EQUAL, a queue admission
    on a sub-range, a reconcile-only pass and a whole pass: every output the second pass defines, and what it must leave alone,
    against the oracle; the same pair with eng.sync() between gives the same bits."""
    w = worlds(world)
    if KINDS[first][2]:
        w.reset()
        queue(w.eng, first, w.snap.now)
        w.eng.sync()
        plan = w.eng.pass_plan()
        assert plan.grid == KINDS[first][2] and plan.n_chk >= plan.n_fin, (plan.grid, plan.n_chk, plan.n_fin)
    for second in SECONDS:
        try:
            got, admitted = run_pair(w, first, second, parked=True)
            synced, admitted_synced = run_pair(w, first, second, parked=False)
            if second == "admit":
                want, n_adm, _ = w.want_admit()
                for g in (got, synced):
                    np.testing.assert_array_equal(g.pend_bitmap, want.pend_bitmap, err_msg="pending match bitmap")
                    np.testing.assert_array_equal(g.codes, want.codes, err_msg="check codes")
                    np.testing.assert_array_equal(g.admit, want.admit, err_msg="admit")
                assert admitted == admitted_synced == n_adm
            else:
                want, rec = expected(w, [(first, w.snap.now), (second, w.snap.now)])
                check_result(w, got, want, rec)
                check_result(w, synced, want, rec)
                assert_identical(w.snap, got, synced)
        except Exception as e:
            raise AssertionError(f"{first} then {second}") from e


# ---- 2. seeded queued sequences ---------------------------------------------------------------------------------------------
SEQ_WORLD = dict(config="C2", m=300, n=4000, p=1500, override_frac=0.3)


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_queued_sequence(kt, oracle, seed):
    """8-16 passes of mixed kinds, flags and `now` (overrides switching on and off) queued on one engine behind one park, with
    the sparse check list on (even seeds) and off: the last pass's outputs, kt_get_changed when it reconciled, kt_get_check_sparse
    when it checked."""
    w = World(kt, oracle, SEQ_WORLD, seed)
    try:
        eng, snap = w.eng, w.snap
        nows = [snap.now + d for d in NOW_OFFSETS]
        active = [w.want(FRESH, now).override_active for now in nows]
        for i in range(len(nows)):
            for j in range(i):
                assert (active[i] != active[j]).any(), "these `now` values switch no override"
        cap = 2 * w.W * snap.pending.n + 64
        if seed % 2 == 0:
            eng.set_sparse_check(cap)  # (it synchronises: before the park)
        w.views_differ()
        w.warm()
        rng = np.random.default_rng(seed)
        kinds = list(KINDS)
        seq = [(kinds[int(rng.integers(len(kinds)))], nows[int(rng.integers(len(nows)))]) for _ in range(int(rng.integers(8, 17)))]
        assert len({now for _, now in seq}) >= 2
        park(w.stream)
        for kind, now in seq:
            queue(eng, kind, now)
        assert_parked(w.stream)
        got = eng.download()
        want, rec = expected(w, seq)
        flags = KINDS[seq[-1][0]][0]
        try:
            check_result(w, got, want, rec)
            if rec:
                check_diff(eng, snap, got, snap.status)
            if seed % 2 == 0 and not flags & abi.EVAL_SKIP_CHECK:
                check_sparse(eng, want.codes, want.admit, cap)
        except Exception as e:
            raise AssertionError(f"seed {seed}: {seq}") from e
    finally:
        w.close()


# ---- 3. several engines on one caller stream --------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [31, 32])
def test_engines_share_a_stream(kt, oracle, seed):
    """2-3 engines on ONE caller stream, whole and partial passes interleaved behind one park (bench.py's rotate mode queues
    whole passes of several contexts so): each engine's last pass against its own oracle."""
    torch = torch_mod()
    stream = torch.cuda.Stream()
    rng = np.random.default_rng(seed)
    E = 2 + seed % 2
    ws = [World(kt, oracle, dict(WORLDS["small_fast"], seed=seed * 10 + i), seed + i, stream) for i in range(E)]
    try:
        for w in ws:
            w.warm()
        kinds = list(KINDS)
        seqs = [[] for _ in ws]
        order = [i % E for i in range(4 * E)]
        rng.shuffle(order)
        park(stream)
        for i in order:
            kind = "fused" if not seqs[i] else kinds[int(rng.integers(len(kinds)))]
            queue(ws[i].eng, kind, ws[i].snap.now)
            seqs[i].append((kind, ws[i].snap.now))
        assert_parked(stream)
        for i, w in enumerate(ws):
            got = w.eng.download()
            want, rec = expected(w, seqs[i])
            try:
                check_result(w, got, want, rec)
            except Exception as e:
                raise AssertionError(f"engine {i} of {order}: {seqs[i]}") from e
    finally:
        for w in ws:
            w.close()


# ---- 4. async uploads and the stream hand-off -------------------------------------------------------------------------------
def pin(arr, keep, wc=False):
    import kube_throttler_b200 as kt

    b = kt.Pinned(arr.shape, arr.dtype, upload_only=wc)
    b.array[...] = arr
    keep.append(b)
    return b.array


def pin_block(arrays, keep, wc=False):
    """The arrays carved out of ONE pinned block (16-byte aligned pieces), as a packer with one arena per snapshot does."""
    import kube_throttler_b200 as kt

    offs, at = [], 0
    for a in arrays:
        offs.append(at)
        at += (a.nbytes + 15) & ~15
    blk = kt.Pinned((max(at, 16),), np.uint8, upload_only=wc)
    keep.append(blk)
    views = []
    for a, o in zip(arrays, offs):
        v = blk.array[o:o + a.nbytes].view(a.dtype).reshape(a.shape)
        v[...] = a
        views.append(v)
    return views


def pinned_wide(pods, keep):
    return abi.PodCols(*(pin(getattr(pods, f), keep) for f in ("labels", "req", "present", "flags", "ns_id")))


def pinned_compact(pods, keep):
    c = abi.compact_pods(pods)
    return abi.CompactPodCols(c.val_bits, pin(c.labels32, keep), pin(c.req32, keep), c.req_shift, pin(c.present, keep), pin(c.meta, keep))


def pinned_packed(pods, keep, block, wc=False):
    c = abi.packed_pods(pods, code_requests=True)
    arrays = [c.labels16, c.pairs, c.meta, c.req_codes, c.req_dict]
    labels16, pairs, meta, req_codes, req_dict = pin_block(arrays, keep, wc) if block else [pin(a, keep, wc) for a in arrays]
    return abi.PackedPodCols(c.ns_bits, pairs, labels16, None, None, meta, req_dict, c.req_dict_off, c.req_code_bytes, req_codes)


def rows_of(snap, donor):
    """The snapshot with the donor's running and pending rows (same counts, same tables)."""
    s = copy.copy(snap)
    s.running, s.pending = donor.running, donor.pending
    return s.normalize()


def async_engine(kt, snap, stream):
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.set_stream(stream.cuda_stream)
    eng.set_row_order(RUN, abi.ROW_ORDER_AS_GIVEN)
    eng.set_row_order(PEND, abi.ROW_ORDER_AS_GIVEN)
    eng.upload_snapshot(snap)
    return eng


def test_async_uploads_between_queued_passes(kt, oracle):
    """Async uploads in every format -- wide, compact, packed from one pinned write-combined block and from scattered pinned
    arrays -- interleaved with passes of several kinds behind one park: the last pass sees the rows the last uploads carried."""
    torch = torch_mod()
    kw = WORLDS["small_fast"]
    a = make(kw)
    a.status = observed_status(oracle.columnar_evaluate(a), a, np.random.default_rng(3))
    a.normalize()
    b, c = rows_of(a, make(dict(kw, seed=77))), rows_of(a, make(dict(kw, seed=78)))
    stream = torch.cuda.Stream()
    keep = []
    eng = async_engine(kt, a, stream)
    try:
        passes = ("fused", "check_only", "reconcile_only", "fused")
        args = []  # (upload call, kind, host columns pinned before the park)
        for fmt, (kind, pods) in zip(("wide", "packed", "packed_block_wc", "compact"), ((RUN, b.running), (PEND, b.pending), (RUN, c.running), (PEND, c.pending))):
            if fmt == "wide":
                args.append((eng.upload_pods, kind, pinned_wide(pods, keep)))
            elif fmt == "packed":
                args.append((eng.upload_pods_packed, kind, pinned_packed(pods, keep, block=False)))
            elif fmt == "packed_block_wc":
                args.append((eng.upload_pods_packed, kind, pinned_packed(pods, keep, block=True, wc=True)))
            else:
                args.append((eng.upload_pods_compact, kind, pinned_compact(pods, keep)))

        def run(parked):
            eng.set_async_uploads(False)
            eng.upload_pods(RUN, a.running)
            eng.upload_pods(PEND, a.pending)
            eng.set_async_uploads(True)
            eng.evaluate(a.now)
            eng.sync()
            if parked:
                park(stream)
            for (fn, kind, cols_), kind_ in zip(args, passes):
                fn(kind, cols_)
                queue(eng, kind_, a.now)
            if parked:
                assert_parked(stream)
            got = eng.download()
            eng.set_async_uploads(False)
            return got

        run(parked=False)  # the staging buffers reach their sizes: nothing is allocated behind the park
        got = run(parked=True)
        want = oracle.columnar_evaluate(c, FRESH, words_per_row=got.words_per_row)
        assert_same(c, got, want)
    finally:
        torch.cuda.synchronize()
        eng.close()
        del keep


@pytest.mark.parametrize("switch", ["caller_to_caller", "caller_to_null", "null_to_caller"])
def test_stream_switch_keeps_queued_work_ordered(kt, oracle, switch):
    """Async uploads of new pending rows queued on a parked caller stream A, then kt_set_stream: the pass and the download on
    the new stream see the new rows, and kt_sync on the new stream leaves A idle.  null_to_caller: the uploads are queued on
    the context's own stream after a switch away from parked A, then the context moves to caller stream B."""
    torch = torch_mod()
    kw = WORLDS["small_fast"]
    a = make(kw)
    b = rows_of(a, make(dict(kw, seed=77)))
    new = copy.copy(a)
    new.pending = b.pending
    new.normalize()
    want = oracle.columnar_evaluate(new, FRESH, words_per_row=None)
    old = oracle.columnar_evaluate(a, FRESH, words_per_row=None)
    assert (want.codes != old.codes).any(axis=1).sum() >= a.pending.n // 50
    s_a, s_b = torch.cuda.Stream(), torch.cuda.Stream()
    keep = []
    eng = async_engine(kt, a, s_a)
    try:
        eng.evaluate(a.now)
        got = eng.download()
        assert got.words_per_row == want.words_per_row
        assert_same(a, got, old)
        cols = pinned_wide(b.pending, keep)
        eng.set_async_uploads(True)
        park(s_a)
        if switch == "null_to_caller":
            eng.set_stream(None)
        eng.upload_pods(PEND, cols)
        eng.set_stream(None if switch == "caller_to_null" else s_b.cuda_stream)
        eng.evaluate(a.now)
        got = eng.download()
        eng.sync()
        idle = s_a.query()
        assert_same(new, got, want)
        assert idle, "kt_sync after the switch returned while work queued before it was still pending"
    finally:
        torch.cuda.synchronize()
        eng.close()
        del keep


# ---- 5. a ring of step contexts on caller streams ---------------------------------------------------------------------------
def test_step_ring_on_caller_streams(kt, oracle):
    """bench.py's pipelined end-to-end path: D = 4 contexts, each on its own caller stream, share the same pinned (and
    write-combined) packed blocks of two snapshots that alternate; step k+D-1 is submitted before step k is waited for, and
    every step's result is compared with the oracle."""
    import ctypes as C

    torch = torch_mod()

    def view(ptr, dtype, shape):
        n = int(np.prod(shape))
        if n == 0:
            return np.zeros(shape, dtype)
        buf = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(ptr)
        return np.frombuffer(buf, dtype=dtype, count=n).reshape(shape).copy()

    D, STEPS = 4, 14
    x = make(dict(config="C2", m=300, n=8000, p=1500))
    y = rows_of(x, make(dict(config="C2", m=300, n=8000, p=1500, seed=77)))
    keep = []
    packed = [tuple(pinned_packed(pods, keep, block=True, wc=wc) for pods in (s.running, s.pending)) for s, wc in ((x, False), (y, True))]
    args = [tuple((c.n, c.struct()) for c in cols) for cols in packed]
    ring = []
    try:
        for _ in range(D):
            st = torch.cuda.Stream()
            eng = kt.Engine(x.R, x.L, x.LN)
            eng._test_stream = st  # the stream lives as long as the engine
            eng.set_stream(st.cuda_stream)
            eng.upload_snapshot(x)
            eng.set_async_uploads(True)
            eng.set_sparse_check(4 * x.pending.n + 64)
            ring.append(eng)
        W = ring[0].words_per_row
        refs = [oracle.columnar_evaluate(s, words_per_row=W) for s in (x, y)]
        assert (refs[0].codes != refs[1].codes).any(axis=1).sum() >= x.pending.n // 50

        def snap_of(k):  # alternates between neighbouring steps and, for each context, from one of its steps to the next
            return (k + k // D) % 2

        def submit(k):
            r_, p_ = args[snap_of(k)]
            ring[k % D].step_submit(r_, p_, x.now)

        for k in range(D - 1):
            submit(k)
        for k in range(STEPS):
            if k + D - 1 < STEPS:
                submit(k + D - 1)
            res = ring[k % D].step_wait()
            snap, ref = (x, y)[snap_of(k)], refs[snap_of(k)]
            P, m, R = snap.pending.n, snap.m, snap.R
            try:
                assert res.n_pending == P
                np.testing.assert_array_equal(view(res.admit, np.uint8, (P,)), ref.admit)
                ent = view(res.entries, np.uint32, (int(res.n_sparse), 3))
                dense = np.zeros((P, 2 * W), np.uint32)
                dense[ent[:, 0], ent[:, 1]] = ent[:, 2]
                np.testing.assert_array_equal(dense, ref.codes)
                live = _live(snap)
                st = res.status
                np.testing.assert_array_equal(view(st.used, np.int64, (R, m))[:, live], ref.used[:, live])
                np.testing.assert_array_equal(view(st.used_cnt, np.int64, (m,))[live], ref.used_cnt[live])
                np.testing.assert_array_equal(view(st.used_present, np.uint32, (m,))[live], ref.used_present[live])
                np.testing.assert_array_equal(view(st.throttled, np.uint32, (m,))[live], ref.throttled[live])
                np.testing.assert_array_equal(view(st.calc_thr, np.int64, (R, m)), ref.calc_thr)
                np.testing.assert_array_equal(view(st.calc_present, np.uint32, (m,)), ref.calc_present)
            except Exception as e:
                raise AssertionError(f"step {k} on context {k % D}") from e
    finally:
        torch.cuda.synchronize()
        for eng in ring:
            eng.close()
        del keep
