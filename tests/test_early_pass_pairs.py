"""Early fused passes whose predecessor has another shape: every build, tile width, decide mode and kernel family as the early
successor, chains of contexts of different shapes, and work the library cannot see between two passes.

A k_pass queued right behind a k_pass of this library (of another context, or of the same one when neither zero-fills) runs
its whole first phase -- match tiles, pre-records, reconcile tiles -- before it waits for the pass ahead (test_overlapped_passes.py
has the argument and one shape pair).  Here the successor reaches its build (512 or 768 threads per SM), tile width (128 or
256 rows), decide mode (sub-tiles or lane-per-pod tiles) and kernel variant through the automatic choices of launch_pass and
dispatch_pass, because a forced plan poisons the pass's outputs with memsets queued before it, and those break adjacency: a
forced context is only ever a predecessor.  One successor world is sized from the capacity probe passes report, so that the
automatic plan takes the 768-thread build with lane-per-pod decide tiles and its CTAs can only be placed as the predecessor's
CTAs exit, as at every bench shape.

Every queue is built once behind one bounded park (torch.cuda._sleep) and checked once: each context's last pass against the
columnar oracle and against the same queue synchronised after every pass (which also loads every kernel and sizes every
buffer before the park).  Behind a predecessor capped to two CTAs the in-kernel trace shows that a tile of the successor
began before the predecessor's last CTA exited; the last test asserts that those witnessed early successors covered both
builds, both decide modes, both tile widths, the general family and R = 31.
"""
import ctypes as C

import numpy as np
import pytest

from kube_throttler_b200 import abi
from test_gpu_parity import _live
from test_overlapped_passes import CAP, FUSED_FLAGS, check_last, queue_sequence, trace_of
from test_partial_passes import EXTRA, observed_status, random_reserved
from test_pass_plans import SHAPES, make, with_rows
from test_queued_passes import DAY, WORLDS, World, assert_identical, assert_parked, park, torch_mod

pytestmark = pytest.mark.gpu

FRESH, GIVEN, ON_EQUAL = abi.EVAL_FRESH_STATUS, abi.EVAL_GIVEN_STATUS, abi.EVAL_ON_EQUAL
QUAD, PER_POD = abi.PLAN_DECIDE_QUAD, abi.PLAN_DECIDE_PER_POD
PEND = abi.PODS_PENDING

_EXTRA = {name: kw for name, kw, _, _ in EXTRA}
# world -> (synth keywords, World seed).  Pending counts are raised where the FRESH and GIVEN views would otherwise decide too
# few rows differently (World.views_differ); overrides where a one-context chain needs `now` values that switch them.
KW = {
    "pred_small": (dict(WORLDS["small_fast"], seed=71), 21),  # the capped predecessor of test_overlapped_passes
    "c2": (WORLDS["c2"], 5),                                  # BASELINE C2 at full size: 528 CTAs, the whole 512-thread grid
    "fast128_t2_r4": (dict(SHAPES["fast128_t2_r4"][0], p=2000, seed=41), 41),
    "fast256_t2_r8": (dict(SHAPES["fast256_t2_r8"][0], override_frac=0.3, seed=42), 42),
    "general_t2_b6": (dict(SHAPES["general_t2_b6"][0], p=3400, override_frac=0.3, seed=42), 42),
    "general_tp4": (dict(SHAPES["general_tp4"][0], p=3400, seed=41), 41),
    # R = 31: G = 32 finalize lanes per throttle, 30 status tiles against 16 match tiles, so each match tile writes the
    # pre-records of several status tiles
    "r31_l16": (dict(_EXTRA["limits_r31_l16"], p=2000, override_frac=0.3, seed=41), 41),
    # rows in no namespace order: the engine stores them clustered by namespace and maps them back at the boundary
    "c2_clustered": (dict(config="C2", m=300, n=8000, p=2000, sort_by_namespace=False, seed=41), 41),
    "sentinel": (dict(SHAPES["fast128_t1_r4"][0], p=2000, seed=41), 41),
    "big": (dict(config="C2", override_frac=0.3, seed=48), 48),  # rows: big_snapshot
}
# the automatic plan of every successor world: (threads per SM, decide mode, (tile, tpc, b, rt))
PLANS = {
    "fast128_t2_r4": (512, QUAD, (128, 2, 2, 4)),
    "fast256_t2_r8": (512, QUAD, (256, 2, 2, 8)),
    "general_t2_b6": (512, PER_POD, (128, 2, 6, 0)),  # 107 sub-tiles on a grid of 51
    "general_tp4": (512, PER_POD, (128, 2, 6, 0)),
    "r31_l16": (512, QUAD, (128, 2, 2, 0)),
    "c2_clustered": (512, QUAD, (128, 2, 2, 4)),
    "sentinel": (512, QUAD, (128, 1, 2, 4)),
    "big": (768, PER_POD, (128, 2, 2, 4)),
}


def big_snapshot(kt):
    """C2-like rows, cut from one pool so that the tables stay the same, sized from the capacity probe passes report: more
    first-phase tiles than 8 rounds of the 512-thread grid (the 768-thread build) and more decide sub-tiles than 2 rounds of
    the 768-thread grid (lane-per-pod tiles).  The pool holds 9 rounds of 512 / 768 resident threads per SM in 128-row CTAs."""
    torch = torch_mod()
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    T = 128
    pool = make(dict(KW["big"][0], n=9 * (512 // T) * sm * T, p=3 * (768 // T) * sm * (T // 4)))
    probe = with_rows(pool, 4000, 1000)
    eng = kt.Engine(probe.R, probe.L, probe.LN)
    try:
        eng.upload_snapshot(probe)
        caps = {}
        for threads in (0, 768):
            eng.set_pass_plan(threads=threads)
            eng.evaluate(probe.now)
            eng.sync()
            plan = eng.pass_plan()
            assert plan.tile == T and plan.threads_per_sm == (threads or 512), (plan.tile, plan.threads_per_sm)
            caps[plan.threads_per_sm] = plan.capacity
    finally:
        eng.close()
    p = 2 * caps[768] * (T // 4) + caps[768] * (T // 4) // 8   # 2.125 rounds of sub-tiles on the 768-thread grid
    n = 8 * caps[512] * T + caps[512] * T // 2 - p            # 8.5 rounds of first-phase tiles on the 512-thread grid
    assert n <= pool.running.n and p <= pool.pending.n, (caps, n, p)
    return with_rows(pool, n, p)


class CutWorld(World):
    """A World on a snapshot made here rather than from synth keywords (the big world is cut from a larger pool): the same
    lagging observed status and reservations, engine on the caller stream and oracle cache."""

    def __init__(self, kt, oracle, snap, seed, stream):
        self.oracle = oracle
        self.snap = snap
        rng = np.random.default_rng(seed)
        snap.status = observed_status(oracle.columnar_evaluate(snap), snap, rng)
        snap.reserved, snap.reserved_present, snap.reserved_cnt = random_reserved(snap, rng)
        snap.normalize()
        self.stream = stream
        self.eng = kt.Engine(snap.R, snap.L, snap.LN)
        self.eng.set_stream(stream.cuda_stream)
        self.eng.upload_snapshot(snap)
        self.W = self.eng.words_per_row
        self._want = {}


@pytest.fixture(scope="module")
def stream():
    torch = torch_mod()
    s = torch.cuda.Stream()
    yield s
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def worlds(kt, oracle, stream):
    """Every world once, its engine on the module's one caller stream, made when a case first asks for it."""
    made = {}

    def get(name):
        if name not in made:
            kw, seed = KW[name]
            w = CutWorld(kt, oracle, big_snapshot(kt), seed, stream) if name == "big" else World(kt, oracle, kw, seed, stream)
            w.views_differ()
            if name == "c2_clustered":
                assert w.eng.row_order(PEND)[0], "the pending rows are not stored clustered"
            w.reset()
            made[name] = w
        return made[name]

    yield get
    for w in made.values():
        w.close()


def prepare(w, sparse=False, trace=False):
    """The context's settings for a case (each call before the park; set_sparse_check synchronises): automatic plan, timing
    off, the sparse check list on or off, the trace on or off.  Returns the sparse list's capacity (0: off)."""
    w.eng.set_pass_plan()
    w.eng.enable_timing(False)
    cap = 2 * w.W * w.snap.pending.n + 64 if sparse else 0
    w.eng.set_sparse_check(cap)
    w.eng.enable_trace(trace)
    w.sparse_cap = cap
    return cap


def run_queue(seq, synced, between=None):
    """(world, flags) pairs queued in order at each world's snap.now; `between` is called between two passes."""
    for i, (w, flags) in enumerate(seq):
        if i and between:
            between()
        w.eng.evaluate(w.snap.now, flags)
        if synced:
            w.eng.sync()


def last_of(seq):
    """{world: flags of its last pass}, in order of first appearance."""
    last = {}
    for w, flags in seq:
        last[w] = flags
    return last


def run_and_check(stream, seq, between=None):
    """The queue synchronised after every pass, then behind one park: every world's last pass against the oracle (and its
    sparse list where it is on) and against the synchronised queue.  Returns the parked results."""
    run_queue(seq, synced=True, between=between)
    last = last_of(seq)
    synced = {w: w.eng.download() for w in last}
    torch_mod().cuda.synchronize()
    park(stream)
    run_queue(seq, synced=False, between=between)
    assert_parked(stream)
    got = {w: w.eng.download() for w in last}
    for i, (w, flags) in enumerate(last.items()):
        try:
            check_last(w, got[w], flags, w.snap.now, cap=w.sparse_cap or None)
            assert_identical(w.snap, got[w], synced[w])
        except Exception as e:
            raise AssertionError(f"context {i} of the queue (last flags {flags})") from e
    return got


def assert_plan(w, name):
    plan = w.eng.pass_plan()
    threads, decide, variant = PLANS[name]
    ran = (plan.threads_per_sm, plan.decide, (plan.tile, plan.tpc, plan.b, plan.rt))
    assert plan.max_ctas == 0 and ran == (threads, decide, variant), (name, ran)
    return plan


def overlapped(a, b):
    """The trace witness: a first-phase tile of b's last pass began before the last CTA of a's last pass (capped) exited."""
    _, a_rows = trace_of(a.eng)
    b_first, _ = trace_of(b.eng)
    assert a.eng.pass_plan().grid == CAP
    exits = a_rows[:, 29][a_rows[:, 29] > 0]
    starts = b_first[:, 2]
    assert exits.shape[0] == CAP and (starts > 0).all()
    return bool(starts.min() < exits.max())


# ---- 1. predecessor x successor, two contexts on one caller stream ----------------------------------------------------------
PREDECESSORS = {  # name -> (world, (threads, decide) forced on a grid capped to CAP CTAs, or None: automatic and uncapped)
    "512_quad_cap2": ("pred_small", (512, QUAD)),
    "512_per_pod_cap2": ("pred_small", (512, PER_POD)),
    "768_quad_cap2": ("pred_small", (768, QUAD)),
    "768_per_pod_cap2": ("pred_small", (768, PER_POD)),
    "c2_auto": ("c2", None),
}
SUCCESSORS = {  # name -> (world, sparse check list on)
    "fast128_t2_r4": ("fast128_t2_r4", False),
    "fast256_t2_r8": ("fast256_t2_r8", True),
    "general_t2_b6": ("general_t2_b6", False),
    "general_tp4": ("general_tp4", True),
    "r31_l16": ("r31_l16", True),
    "c2_clustered": ("c2_clustered", False),
    # k_order_sparse_rows follows the pass (device rows -> caller rows): the pass after it is not early
    "c2_clustered_sparse": ("c2_clustered", True),
    "big": ("big", False),
}
MATRIX_FLAGS = (FRESH, GIVEN | ON_EQUAL, GIVEN, FRESH | ON_EQUAL)  # A, B, A, B

_matrix = {}  # (predecessor, successor) -> (threads, decide, tile, variant, witnessed)


@pytest.mark.parametrize("succ", list(SUCCESSORS))
@pytest.mark.parametrize("pred", list(PREDECESSORS))
def test_predecessor_successor_matrix(worlds, stream, pred, succ):
    """A(FRESH), B(GIVEN|ON_EQUAL), A(GIVEN), B(FRESH|ON_EQUAL) behind one park, B automatic and of another shape than A: B's
    plan is the one its shape selects; both contexts' last passes equal the oracle (bitmaps, codes, admit bits, status
    columns, changed list, sparse list where it is on) and the queue synchronised after every pass; behind a capped A, a
    tile of B began before A's last CTA exited."""
    a_name, forced = PREDECESSORS[pred]
    b_name, sparse = SUCCESSORS[succ]
    a, b = worlds(a_name), worlds(b_name)
    try:
        prepare(a, trace=forced is not None)
        prepare(b, sparse=sparse, trace=forced is not None)
        if forced:
            a.eng.set_pass_plan(*forced, CAP)
        seq = [(w, flags) for w, flags in zip((a, b, a, b), MATRIX_FLAGS)]
        run_and_check(stream, seq)
        plan = assert_plan(b, b_name)
        witnessed = False
        if forced:
            ran = a.eng.pass_plan()
            assert (ran.threads_per_sm, ran.decide, ran.max_ctas, ran.tile) == (*forced, CAP, 128)
            witnessed = overlapped(a, b)
            assert witnessed, "B's first tile began only after A's last CTA exited: the passes did not overlap"
        _matrix[pred, succ] = (plan.threads_per_sm, plan.decide, plan.tile, (plan.tpc, plan.b, plan.rt), b.snap.R, witnessed)
    finally:
        for w in (a, b):
            w.eng.set_pass_plan()
            w.eng.enable_trace(False)


# ---- 2. chains of three contexts of different shapes ------------------------------------------------------------------------
CHAINS = {
    "fast256_general_r31": ("fast256_t2_r8", "general_t2_b6", "r31_l16"),
    "big_tp4_clustered": ("big", "general_tp4", "c2_clustered"),
}
CHAIN_FLAGS = (GIVEN, FRESH, GIVEN | ON_EQUAL, FRESH | ON_EQUAL, GIVEN | ON_EQUAL, FRESH, GIVEN)  # A B C A B C D


@pytest.mark.parametrize("chain", list(CHAINS))
def test_chain_of_three_contexts(worlds, stream, chain):
    """A, B, C, A, B, C, then a small sentinel D, all automatic, behind one park: every pass but the first is early behind a
    context of another shape, the pass parity of each context wraps while its neighbours differ, and the last pass of each of
    the four equals the oracle and the queue synchronised after every pass."""
    names = CHAINS[chain] + ("sentinel",)
    ws = [worlds(name) for name in names]
    for w in ws:
        prepare(w)
    order = [0, 1, 2, 0, 1, 2, 3]
    seq = [(ws[i], flags) for i, flags in zip(order, CHAIN_FLAGS)]
    run_and_check(stream, seq)
    for w, name in zip(ws, names):
        assert_plan(w, name)


# ---- 3. one-context chains per family ---------------------------------------------------------------------------------------
ONE_CONTEXT = ("fast256_t2_r8", "general_t2_b6", "r31_l16", "big")


@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
@pytest.mark.parametrize("world", ONE_CONTEXT)
def test_fused_queue_one_context_per_family(worlds, stream, world, sparse):
    """The five fused passes of test_fused_queue_one_context (alternating views, `now` values that switch overrides on and
    off) on ONE context of each shape behind one park: the last pass against the oracle, and the same bits as the queue
    synchronised after every pass."""
    w = worlds(world)
    snap = w.snap
    nows = (snap.now, snap.now - 40 * DAY)
    assert (w.want(FRESH, nows[0]).override_active != w.want(FRESH, nows[1]).override_active).any(), "these `now` values switch no override"
    cap = prepare(w, sparse=sparse)
    queue_sequence(w, nows, synced=True)
    synced = w.eng.download()
    torch_mod().cuda.synchronize()
    park(stream)
    queue_sequence(w, nows, synced=False)
    assert_parked(stream)
    got = w.eng.download()
    check_last(w, got, FUSED_FLAGS[-1], nows[(len(FUSED_FLAGS) - 1) % len(nows)], cap=cap or None)
    assert_identical(snap, got, synced)
    assert_plan(w, world)


# ---- 4. what the library cannot see between two passes ----------------------------------------------------------------------
@pytest.mark.parametrize("between", ["caller_kernel", "event_record"])
def test_caller_work_between_passes(worlds, stream, between):
    """A caller's kernel (a torch op on the stream) or a torch.cuda.Event record between every two passes of A (capped) and
    B: the library's record still names the last k_pass, so B is launched early behind it.  Both contexts' last passes are
    exact and the caller's tensor holds every one of its increments."""
    torch = torch_mod()
    a, b = worlds("pred_small"), worlds("general_t2_b6")
    x = torch.zeros(1 << 16, dtype=torch.int64, device="cuda")
    events = [torch.cuda.Event() for _ in range(6)]
    used = []

    def caller():
        with torch.cuda.stream(stream):
            if between == "caller_kernel":
                x.add_(1)
            else:
                events[len(used)].record(stream)
        used.append(1)

    try:
        prepare(a)
        prepare(b)
        a.eng.set_pass_plan(512, QUAD, CAP)
        torch.cuda.synchronize()
        seq = [(w, flags) for w, flags in zip((a, b, a, b), MATRIX_FLAGS)]
        run_and_check(stream, seq, between=caller)
        torch.cuda.synchronize()
        assert len(used) == 6
        if between == "caller_kernel":
            assert bool((x == 6).all()), x.unique()
        else:
            assert all(ev.query() for ev in events)
    finally:
        a.eng.set_pass_plan()


def host_view(ptr, dtype, shape):
    n = int(np.prod(shape))
    if n == 0:
        return np.zeros(shape, dtype)
    buf = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype, count=n).reshape(shape).copy()


def check_step(w, res, want):
    """A step block (admit bits, non-zero code words, status columns) against the oracle."""
    snap, W = w.snap, w.W
    P, m, R = snap.pending.n, snap.m, snap.R
    assert res.n_pending == P
    np.testing.assert_array_equal(host_view(res.admit, np.uint8, (P,)), want.admit, err_msg="admit")
    ent = host_view(res.entries, np.uint32, (int(res.n_sparse), 3))
    dense = np.zeros((P, 2 * W), np.uint32)
    dense[ent[:, 0], ent[:, 1]] = ent[:, 2]
    assert int(res.n_sparse) == int(np.count_nonzero(want.codes))
    np.testing.assert_array_equal(dense, want.codes, err_msg="codes")
    live = _live(snap)
    st = res.status
    np.testing.assert_array_equal(host_view(st.used, np.int64, (R, m))[:, live], want.used[:, live], err_msg="used")
    np.testing.assert_array_equal(host_view(st.used_cnt, np.int64, (m,))[live], want.used_cnt[live], err_msg="used_cnt")
    np.testing.assert_array_equal(host_view(st.used_present, np.uint32, (m,))[live], want.used_present[live], err_msg="used_present")
    np.testing.assert_array_equal(host_view(st.throttled, np.uint32, (m,))[live], want.throttled[live], err_msg="throttled")
    np.testing.assert_array_equal(host_view(st.calc_thr, np.int64, (R, m)), want.calc_thr, err_msg="calc_thr")
    np.testing.assert_array_equal(host_view(st.calc_present, np.uint32, (m,)), want.calc_present, err_msg="calc_present")


def test_step_right_behind_another_context(worlds, stream):
    """kt_step_submit with no new rows right behind another context's (capped) pass: the step's pass may start early, its
    result copies follow it (and, the pending rows being clustered, the sparse list's and admit bits' mapping back to caller
    rows), then A passes again.  The step block equals the oracle, and so does A's last pass."""
    a, b = worlds("pred_small"), worlds("c2_clustered")
    flags = GIVEN | ON_EQUAL
    try:
        prepare(a)
        prepare(b, sparse=True)
        a.eng.set_pass_plan(512, PER_POD, CAP)
        for parked in (False, True):  # the first round loads every kernel and sizes every buffer
            torch_mod().cuda.synchronize()
            if parked:
                park(stream)
            a.eng.evaluate(a.snap.now, FRESH)
            b.eng.step_submit(None, None, b.snap.now, flags)
            a.eng.evaluate(a.snap.now, GIVEN)
            if parked:
                assert_parked(stream)
            res = b.eng.step_wait()
            check_step(b, res, b.want(flags))
            check_last(a, a.eng.download(), GIVEN, a.snap.now)
    finally:
        a.eng.set_pass_plan()
        b.eng.set_sparse_check(0)


# ---- 5. what the matrix reached ---------------------------------------------------------------------------------------------
def test_every_shape_reached_as_early_successor():
    """Runs after the matrix: among the successors the trace showed overlapping a capped predecessor were both builds, both
    decide modes, both tile widths, the general family (rt = 0) and R = 31."""
    if set(_matrix) != {(p, s) for p in PREDECESSORS for s in SUCCESSORS}:
        pytest.skip("the matrix did not run in full")
    print("\npredecessor x successor: threads/SM, decide, tile, (tpc, b, rt), R, overlap witnessed")
    for (p, s), (threads, decide, tile, variant, R, seen) in _matrix.items():
        print(f"  {p:18s} {s:20s} {threads} {'quad' if decide == QUAD else 'per_pod'} {tile} {variant} R={R} {'yes' if seen else 'n/a'}")
    early = [v for v in _matrix.values() if v[5]]
    assert {v[0] for v in early} == {512, 768}
    assert {v[1] for v in early} == {QUAD, PER_POD}
    assert {v[2] for v in early} == {128, 256}
    assert any(v[3][2] == 0 for v in early), "no general-family successor"
    assert any(v[4] == 31 for v in early), "no R = 31 successor"
