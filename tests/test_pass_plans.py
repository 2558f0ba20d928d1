"""Every build and decide mode of the fused pass (k_pass) against the columnar oracle, bit-exact.

At launch, launch_pass picks from the shape a residency (the k_pass build for 512 or for 768 resident threads per SM) and a
decide mode (four-lane sub-tiles, check_decide_quad, or lane-per-pod tiles, check_decide_tile); dispatch_pass picks one of 12
kernel variants from the tables.  The shapes a test happens to use reach only a few of these 48 device code paths, so the
tests here force each of them through the test seam kt_debug_set_pass_plan (Engine.set_pass_plan): on the grid the device
holds, and on grids of 1 and 3 CTAs, where a CTA runs tile after tile and a wait on anything but a smaller ticket would stall.
Under a forced plan a timed-out wait is an error of sync(), and the pass's outputs are poisoned before it runs, so work it skipped
shows up even though the same engine ran the same snapshot just before.
"""
import copy

import numpy as np
import pytest

from kube_throttler_b200 import abi, synth
from test_gpu_parity import assert_same
from test_tables_cpu import compile_tables

pytestmark = pytest.mark.gpu

QUAD, PER_POD = abi.PLAN_DECIDE_QUAD, abi.PLAN_DECIDE_PER_POD
THREADS = (512, 768)
DECIDES = (QUAD, PER_POD)
CAPS = (0, 1, 3)

# One small shape per branch of dispatch_pass, with the (tile, tpc, b, rt) it must reach (rt 0: the general family) and its
# term planes per table entry.  A shape that drifts off its variant fails here instead of silently losing the coverage.
VARIANTS = [
    # fast family (L <= 8, 2-bit counters, R <= 8) with 128-row tiles
    ("fast128_t1_r4", dict(config="C2", m=200, n=3000, p=500, terms=1), (128, 1, 2, 4), 1),
    ("fast128_t1_r8", dict(config="C2", m=200, n=3000, p=500, R=8, terms=1), (128, 1, 2, 8), 1),
    ("fast128_t2_r4", dict(config="C2", m=200, n=3000, p=500, terms=2), (128, 2, 2, 4), 2),
    ("fast128_t2_r8", dict(config="C2", m=200, n=3000, p=500, R=8, terms=2), (128, 2, 2, 8), 2),
    # ClusterThrottle-heavy tables (a namespace's word list is long): 256-row tiles
    ("fast256_t1_r4", dict(config="C3", m=600, n=4000, p=700, R=4, terms=1), (256, 1, 2, 4), 1),
    ("fast256_t1_r8", dict(config="C3", m=600, n=4000, p=700, terms=1), (256, 1, 2, 8), 1),
    ("fast256_t2_r4", dict(config="C3", m=600, n=4000, p=700, R=4, terms=2), (256, 2, 2, 4), 2),
    ("fast256_t2_r8", dict(config="C3", m=600, n=4000, p=700, terms=2), (256, 2, 2, 8), 2),
    # general family: more than 8 label slots, more than 8 resources, or 6-bit counters (terms needing more than 3 keys)
    ("general_t1_b2", dict(config="C2", m=200, n=3000, p=500, L=12, terms=1), (128, 1, 2, 0), 1),
    ("general_t1_b6", dict(config="C2", m=200, n=3000, p=500, q_max=6, terms=1), (128, 1, 6, 0), 1),
    ("general_t2_b2", dict(config="C2", m=200, n=3000, p=500, R=12, terms=2), (128, 2, 2, 0), 2),
    ("general_t2_b6", dict(config="C3", m=200, n=3000, p=500, L=12, q_max=6, terms=2), (128, 2, 6, 0), 2),
    # two plane pairs per table entry (up to 3 terms: the fourth plane is padding; up to 4: both pairs full)
    ("fast128_tp4", dict(config="C2", m=200, n=3000, p=500, terms=3), (128, 2, 2, 4), 4),
    ("fast256_tp4", dict(config="C3", m=600, n=4000, p=700, terms=4), (256, 2, 2, 8), 4),
    ("general_tp4", dict(config="C2", m=200, n=3000, p=500, L=12, q_max=6, terms=3), (128, 2, 6, 0), 4),
]
SHAPES = {name: (kw, variant, tppad) for name, kw, variant, tppad in VARIANTS}

_reached = set()      # (tile, tpc, b, rt, threads, decide) the plan matrix ran
_matrix_shapes = set()


def make(kw):
    kw = dict(kw)
    return synth.generate(kw.pop("config"), **kw)


def with_rows(snap, n, p):
    """The snapshot with its first n running and first p pending rows."""
    assert n <= snap.running.n and p <= snap.pending.n
    s = copy.copy(snap)
    s.running = snap.running.rows(slice(0, n))
    s.pending = snap.pending.rows(slice(0, p))
    return s.normalize()


def engine(kt, snap):
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    return eng


def variant(plan):
    return (plan.tile, plan.tpc, plan.b, plan.rt)


def forced(eng, snap, threads, decide, cap, flags=abi.EVAL_FRESH_STATUS):
    """One pass under a forced plan; its waits must all have completed.  Returns (result, plan)."""
    eng.set_pass_plan(threads, decide, cap)
    eng.evaluate(snap.now, flags)
    eng.sync()  # KtError (KT_ERR_STATE) if an in-kernel wait timed out
    got = eng.download()
    plan = eng.pass_plan()
    assert (plan.threads_per_sm, plan.decide, plan.max_ctas) == (threads, decide, cap)
    tiles = plan.n_chk + plan.n_rec
    assert plan.grid == min(tiles, min(cap, plan.capacity) if cap else plan.capacity) >= 1
    assert (plan.n_chk, plan.n_rec) == (-(-snap.pending.n // plan.tile), -(-snap.running.n // plan.tile))
    return got, plan


def automatic(eng, snap, flags=abi.EVAL_FRESH_STATUS):
    """A pass with the automatic choices; checks them against the rules of launch_pass.  Returns (result, plan)."""
    eng.set_pass_plan()
    eng.evaluate(snap.now, flags)
    eng.sync()
    got = eng.download()
    plan = eng.pass_plan()
    tiles = plan.n_chk + plan.n_rec
    assert plan.max_ctas == 0 and plan.grid == min(tiles, plan.capacity)
    if plan.threads_per_sm == 512:  # (the 512-thread capacity is only known when that build ran)
        assert tiles <= 8 * plan.capacity
    n_quad = -(-snap.pending.n // (plan.tile // 4))
    assert plan.decide == (QUAD if n_quad <= 2 * plan.grid else PER_POD)
    assert plan.n_sub == (n_quad if plan.decide == QUAD else plan.n_chk)
    return got, plan


def check_trace(eng, plan):
    """The ticket queue as the trace shows it: every first-phase tile ran once, by a CTA of the grid, then every status tile."""
    rows, roles = eng.trace()
    assert list(roles) == [plan.n_chk, plan.n_rec, plan.n_fin, plan.grid]
    tiles = plan.n_chk + plan.n_rec
    assert rows.shape[0] == tiles + plan.n_fin
    first, status = rows[:tiles], rows[tiles:]
    np.testing.assert_array_equal(first[:, 0], np.arange(tiles))  # row i: ticket i
    assert (first[:, 3] > 0).all(), "a first-phase tile never closed its row"
    assert (rows[:, 28] < plan.grid).all()
    if plan.grid == 1:
        assert (rows[:, 28] == 0).all()
    assert (status[:, 3] > 0).all(), "a status tile never closed its row"
    tickets = status[:, 0].astype(np.int64)
    assert ((tickets >= tiles) & (tickets < tiles + plan.n_fin + plan.n_sub)).all()
    assert np.unique(tickets).shape[0] == plan.n_fin


@pytest.mark.parametrize("name", list(SHAPES))
def test_plan_matrix(kt, oracle, name):
    """Variant map + plan matrix: the shape reaches its dispatch_pass variant, then every build x decide mode x grid cap gives
    the oracle's bits, pass after pass on one engine (the counters re-arm across changes of the grid), and an automatic pass
    at the end still does."""
    kw, want_variant, tppad = SHAPES[name]
    snap = make(kw)
    assert compile_tables(kt, snap)["TPpad"] == tppad
    eng = engine(kt, snap)
    eng.enable_trace(True)
    got, plan = automatic(eng, snap)
    want = oracle.columnar_evaluate(snap, words_per_row=got.words_per_row)
    assert_same(snap, got, want)
    assert variant(plan) == want_variant, (variant(plan), want_variant)
    assert got.match_matrix("pending", snap.m).sum() > 0
    for threads in THREADS:
        for decide in DECIDES:
            for cap in CAPS:
                got, plan = forced(eng, snap, threads, decide, cap)
                assert variant(plan) == want_variant
                assert_same(snap, got, want)
                if cap:
                    check_trace(eng, plan)
                _reached.add(variant(plan) + (threads, decide))
    got, plan = automatic(eng, snap)
    assert_same(snap, got, want)
    eng.close()
    _matrix_shapes.add(name)


@pytest.mark.parametrize("base", ["fast128_t2_r4", "fast256_t2_r8"])
def test_pending_count_edges(kt, oracle, base):
    """Pending counts around the sub-tile (TILE/4) and tile sizes, against one running pod, under both decide modes and
    both builds: partial sub-tiles, partial tiles, a single pod."""
    kw, _, _ = SHAPES[base]
    full = make(kw)
    eng = engine(kt, full)
    _, plan = automatic(eng, full)
    T = plan.tile
    for p in (1, T // 4 - 1, T // 4, T // 4 + 1, T, T + 1):
        snap = with_rows(full, 1, p)
        eng.upload_pods(abi.PODS_RUNNING, snap.running)
        eng.upload_pods(abi.PODS_PENDING, snap.pending)
        want = None
        for threads in THREADS:
            for decide in DECIDES:
                for cap in (0, 1):
                    got, plan = forced(eng, snap, threads, decide, cap)
                    assert plan.tile == T
                    want = want or oracle.columnar_evaluate(snap, words_per_row=got.words_per_row)
                    assert_same(snap, got, want)
    eng.close()


@pytest.mark.parametrize("kw", [
    dict(config="C2", m=2500, n=3000, p=33),                  # one match tile writes the pre-records of ~160 status tiles
    dict(config="C3", m=120, n=2000, p=300, R=31, L=16),      # R = 31: 32 finalize lanes per throttle
], ids=["many_status_tiles_one_match_tile", "R31"])
def test_role_count_edges(kt, oracle, kw):
    snap = make(kw)
    eng = engine(kt, snap)
    eng.enable_trace(True)
    got, plan = automatic(eng, snap)
    want = oracle.columnar_evaluate(snap, words_per_row=got.words_per_row)
    assert_same(snap, got, want)
    if snap.m == 2500:
        assert plan.n_chk == 1 and plan.n_fin > 100 * plan.n_chk
    for threads in THREADS:
        for decide in DECIDES:
            for cap in (0, 1, 3):
                got, plan = forced(eng, snap, threads, decide, cap)
                assert_same(snap, got, want)
                if cap:
                    check_trace(eng, plan)
    eng.close()


def test_automatic_rule_boundaries(kt, oracle):
    """The automatic choices at a grid capped to g CTAs: 8g first-phase tiles run the 512-thread build and 8g + 1 the
    768-thread one (kDeepRounds); 2g decide sub-tiles run as sub-tiles and 2g + 1 as lane-per-pod tiles (the factor 2)."""
    g = 3
    full = make(dict(config="C2", m=200, n=4000, p=400))
    eng = engine(kt, full)
    eng.set_pass_plan(max_ctas=g)
    eng.evaluate(full.now)
    eng.sync()
    T = eng.pass_plan().tile
    cases = [  # (running rows, pending rows, build, decide mode)
        ((8 * g - 1) * T, T, 512, None),          # tiles = 8g
        (8 * g * T, T, 768, None),                # tiles = 8g + 1
        (2 * T, 2 * g * (T // 4), None, QUAD),    # 2g sub-tiles
        (2 * T, 2 * g * (T // 4) + 1, None, PER_POD),
    ]
    for n, p, threads, decide in cases:
        snap = with_rows(full, n, p)
        eng.upload_pods(abi.PODS_RUNNING, snap.running)
        eng.upload_pods(abi.PODS_PENDING, snap.pending)
        eng.set_pass_plan(max_ctas=g)
        eng.evaluate(snap.now)
        eng.sync()
        got = eng.download()
        plan = eng.pass_plan()
        assert plan.grid == g and plan.tile == T
        if threads is not None:
            assert plan.threads_per_sm == threads, (n, p, plan.n_chk + plan.n_rec)
        if decide is not None:
            assert plan.decide == decide, (n, p, plan.n_sub)
        want = oracle.columnar_evaluate(snap, words_per_row=got.words_per_row)
        assert_same(snap, got, want)
    eng.close()


FLAG_PLANS = [(512, QUAD, 1), (768, PER_POD, 3), (768, QUAD, 0), (512, PER_POD, 0)]


def _stale_status(oracle, snap):
    fresh = oracle.columnar_evaluate(snap)
    rng = np.random.default_rng(7)
    m = snap.m
    st = dict(calculated=(rng.random(m) < 0.8).astype(np.uint8), calc_thr=fresh.calc_thr.copy(), calc_present=fresh.calc_present.copy(),
              calc_cnt=fresh.calc_cnt.copy(), used=fresh.used.copy(), used_present=fresh.used_present.copy(),
              used_cnt=fresh.used_cnt.copy(), throttled=fresh.throttled.copy())
    stale = rng.random(m) < 0.33
    st["used"][:, stale] = (st["used"][:, stale] * 0.5).astype(np.int64)
    st["throttled"][rng.random(m) < 0.2] = 0
    snap.status = st
    return snap.normalize()


@pytest.mark.parametrize("base", ["fast128_t2_r4", "fast256_t2_r8", "general_t2_b6"])
@pytest.mark.parametrize("case", list(synth.VALUE_REGIMES) + ["on_equal", "given_status", "sparse"])
def test_plans_under_other_flags(kt, oracle, base, case):
    """A subset of the matrix under each request-value regime, isThrottledOnEqual, an observed (stale) status, and with the
    sparse check list on (its appends from the lane-per-pod decide tiles inside k_pass included)."""
    kw, _, _ = SHAPES[base]
    kw = dict(kw, values=case) if case in synth.VALUE_REGIMES else dict(kw)
    snap = make(kw)
    flags = abi.EVAL_FRESH_STATUS
    if case == "on_equal":
        flags = abi.EVAL_ON_EQUAL
    elif case == "given_status":
        snap = _stale_status(oracle, snap)
        flags = abi.EVAL_GIVEN_STATUS
    eng = engine(kt, snap)
    cap_entries = 4 * snap.pending.n + 64
    if case == "sparse":
        eng.set_sparse_check(cap_entries)
    want = None
    for threads, decide, cap in FLAG_PLANS:
        got, plan = forced(eng, snap, threads, decide, cap, flags)
        want = want or oracle.columnar_evaluate(snap, flags, words_per_row=got.words_per_row)
        assert_same(snap, got, want)
        if case == "sparse":
            ent = np.zeros((cap_entries, 3), np.uint32)
            admit = np.zeros(snap.pending.n, np.uint8)
            cnt = eng.get_check_sparse(admit, ent)
            dense = want.codes.reshape(snap.pending.n, -1)
            rows, widx = np.nonzero(dense)
            assert cnt == rows.shape[0]
            assert sorted(map(tuple, ent[:cnt].tolist())) == sorted(zip(rows.tolist(), widx.tolist(), dense[rows, widx].tolist()))
            np.testing.assert_array_equal(admit, want.admit)
    eng.close()


def test_plan_seam_arguments(kt):
    """Out-of-range plans are refused; the getter has nothing to report before the first fused pass."""
    eng = kt.Engine(4, 8, 4)
    with pytest.raises(kt.KtError) as e:
        eng.pass_plan()
    assert e.value.code == abi.ERR_STATE
    for bad in (dict(threads=256), dict(threads=1024), dict(decide=3), dict(decide=-1)):
        with pytest.raises(kt.KtError) as e:
            eng.set_pass_plan(**bad)
        assert e.value.code == abi.ERR_INVALID
    eng.set_pass_plan()
    eng.close()


def test_matrix_reached_every_build_and_decide_mode():
    """Runs after the plan matrix: all 24 k_pass builds (12 variants x 2 residencies) ran under both decide modes."""
    if _matrix_shapes != set(SHAPES):
        pytest.skip("the plan matrix did not run in full")
    want = {v + (threads, decide) for _, _, v, _ in VARIANTS for threads in THREADS for decide in DECIDES}
    assert len(want) == 48
    assert want <= _reached, sorted(want - _reached)
