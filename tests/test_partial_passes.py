"""The passes the plugin runs most, against the columnar oracle, bit-exact: reconcile-only (KT_EVAL_SKIP_CHECK, reconcile_all)
and check-only (KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE, every PreFilter pass and the first step of kt_admit_queue).

evaluate_locked runs the one-launch k_pass only for a whole pass with timing off and rows of both kinds; every other pass runs
the chained kernels: k_reconcile (8 variants, dispatch_reconcile), k_finalize and k_check (6 variants, dispatch_check).  The
tests here pin which variant each shape takes, run the plugin's cadence of passes on one engine per shape, drive long-lived
engines through seeded sequences of row deltas, re-uploads and settings, and take the paths only the chained kernels take
(no running rows, no pending rows, pending counts around kTileCheck).  Everything an engine carries from one pass to the next
-- the partial-sum halves, the diff counters, the maintained bitmaps, the translated rows, the sparse list, the upload flags --
is only right if the right kind of pass follows the right kind of event, and a single pass on a fresh engine never shows it.
"""
import copy
import zlib

import numpy as np
import pytest

from kube_throttler_b200 import abi, synth
from test_gpu_parity import _live, assert_same
from test_match_columns import numpy_columns
from test_pass_plans import SHAPES, make, with_rows
from test_tables_cpu import compile_tables

pytestmark = pytest.mark.gpu

FRESH, GIVEN, ON_EQUAL = abi.EVAL_FRESH_STATUS, abi.EVAL_GIVEN_STATUS, abi.EVAL_ON_EQUAL
REC_ONLY = abi.EVAL_FRESH_STATUS | abi.EVAL_SKIP_CHECK        # reconcile_all
CHK_ONLY = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE    # PreFilter
RUN, PEND = abi.PODS_RUNNING, abi.PODS_PENDING

# Shapes beyond the pass-plan ones, for pairings no k_pass build has: (tile, tpc, b, rt) of the fused pass, term planes.
EXTRA = [
    # L > 8 with 2-bit counters and two planes: the general k_check<2, 2, false> (general_t2_b2 has L = 8: a register-row check)
    ("general_l12_t2_b2", dict(config="C2", m=200, n=3000, p=500, L=12, terms=2), (128, 2, 2, 0), 2),
    # R > 8 with L <= 8: a general k_reconcile, and a register-row k_check whose pre-records hold more than 8 resources
    ("general_r12_l8", dict(config="C2", m=200, n=3000, p=500, R=12, terms=1), (128, 1, 2, 0), 1),
    ("general_r31_l8", dict(config="C3", m=120, n=2000, p=300, R=31, terms=2), (128, 2, 2, 0), 2),
    ("limits_r31_l16", dict(config="C3", m=120, n=2000, p=300, R=31, L=16, terms=2), (128, 2, 2, 0), 2),
]
CADENCE = dict(SHAPES, **{name: (kw, v, tppad) for name, kw, v, tppad in EXTRA})

RECONCILE_VARIANTS = {(1, 2, 4), (1, 2, 8), (2, 2, 4), (2, 2, 8), (1, 2, 0), (1, 6, 0), (2, 2, 0), (2, 6, 0)}
CHECK_VARIANTS = {(1, 2, True), (2, 2, True), (1, 2, False), (1, 6, False), (2, 2, False), (2, 6, False)}
_ran = set()  # (kernel, mode, variant) the cadence ran
_cadence_shapes = set()


def reconcile_variant(plan):
    """dispatch_reconcile takes the (tpc, b, rt) dispatch_pass takes for the same tables (always with 128-row tiles)."""
    return (plan.tpc, plan.b, plan.rt)


def check_variant(plan, L):
    return (plan.tpc, plan.b, L <= 8 and plan.b == 2)  # dispatch_check (kt_engine.cu): register rows for L <= 8 and B == 2, any R


def run_pass(eng, snap, flags, launches, timing=False):
    """One kt_evaluate; the path it took (k_pass: 1 launch; chained: 2 for a partial pass, 3 for a whole one) is asserted."""
    eng.enable_timing(timing)
    eng.evaluate(snap.now, flags)
    eng.sync()
    got = eng.download()
    assert eng.timing().launches == launches, (flags, timing, eng.timing().launches)
    eng.enable_timing(False)
    return got


def with_pending_of(want, prev):
    """The oracle's result with the pending outputs (match rows, codes, admit bits) of `prev`: a reconcile-only pass writes none of them."""
    w = copy.copy(want)
    w.pend_bitmap, w.codes, w.admit = prev.pend_bitmap, prev.codes, prev.admit
    return w


def observed_status(fresh, snap, rng):
    """An informer copy of the status that lags behind `fresh` (the oracle's outputs), perturbed as test_device_side_status_diff
    and test_given_status do: other sums, halved sums, a flipped throttled bit, a stale threshold, a lost key, calculatedAt unset."""
    m, R = snap.m, snap.R
    st = dict(calculated=(rng.random(m) < 0.9).astype(np.uint8), calc_thr=fresh.calc_thr.copy(), calc_present=fresh.calc_present.copy(),
              calc_cnt=fresh.calc_cnt.copy(), used=fresh.used.copy(), used_present=fresh.used_present.copy(),
              used_cnt=fresh.used_cnt.copy(), throttled=fresh.throttled.copy())
    st["used"][0, rng.random(m) < 0.2] += 7
    stale = rng.random(m) < 0.2
    st["used"][:, stale] //= 2
    st["throttled"][rng.random(m) < 0.05] ^= 1
    st["calc_thr"][min(1, R - 1), rng.random(m) < 0.05] += 1
    st["used_present"][rng.random(m) < 0.05] &= ~np.uint32(1)
    return st


def random_reserved(snap, rng):
    """Reservations (what the plugin's cache has reserved but no reconcile has observed yet) within the value domain: a share of
    each threshold on some resources, present keys with zero amounts included, pod counts on some throttles."""
    m, R = snap.m, snap.R
    bits = rng.random((R, m)) < 0.3
    reserved = np.where(bits, (np.maximum(snap.thr, 1) * rng.uniform(0.0, 0.6, size=(R, m))).astype(np.int64), 0).astype(np.int64)
    has_cnt = rng.random(m) < 0.3
    present = (bits.astype(np.uint32) << np.arange(R, dtype=np.uint32)[:, None]).sum(axis=0, dtype=np.uint32)
    present |= np.where(has_cnt, abi.COUNT_BIT, 0).astype(np.uint32)
    return reserved, present, np.where(has_cnt, rng.integers(0, 4, size=m), 0).astype(np.int64)


def set_reserved(eng, snap, cols):
    snap.reserved, snap.reserved_present, snap.reserved_cnt = cols
    snap.normalize()
    eng.set_reserved(snap)  # all None: cleared


def check_diff(eng, snap, got, st):
    """kt_get_changed == a numpy diff of the pass's status columns against the observed status; kt_get_reconcile_rows of the
    listed throttles == their columns of the full download."""
    R, m = snap.R, snap.m
    idx, flags = eng.get_changed()
    differs = np.zeros(m, bool)
    bits = (np.uint32(1) << np.arange(R, dtype=np.uint32))[:, None]
    for name_v, name_p, cnt in (("used", "used_present", "used_cnt"), ("calc_thr", "calc_present", "calc_cnt")):
        gp, sp = getattr(got, name_p), st[name_p]
        differs |= gp != sp
        differs |= ((getattr(got, name_v) != st[name_v]) & ((gp[None, :] & bits) != 0)).any(axis=0)
        differs |= (getattr(got, cnt) != st[cnt]) & ((gp & abi.COUNT_BIT) != 0)
    differs |= got.throttled != st["throttled"]
    differs |= st["calculated"] == 0
    differs &= _live(snap)
    np.testing.assert_array_equal(flags.astype(bool), differs)
    np.testing.assert_array_equal(idx, np.nonzero(differs)[0])
    assert 0 < idx.shape[0] < m
    rows = eng.get_reconcile_rows(idx)
    for f in ("used", "calc_thr"):
        np.testing.assert_array_equal(getattr(rows, f), getattr(got, f)[:, idx], err_msg=f)
    for f in ("used_present", "used_cnt", "throttled", "calc_present", "calc_cnt", "override_active"):
        np.testing.assert_array_equal(getattr(rows, f), getattr(got, f)[idx], err_msg=f)


def check_sparse(eng, codes, admit, cap):
    """The sparse list: exactly the non-zero code words of the dense rows, each once, and the same admit bits."""
    ent = np.zeros((cap, 3), np.uint32)
    adm = np.zeros(admit.shape[0], np.uint8)
    cnt = eng.get_check_sparse(adm, ent)
    rows, widx = np.nonzero(codes)
    assert cnt == rows.shape[0] <= cap
    assert sorted(map(tuple, ent[:cnt].tolist())) == sorted(zip(rows.tolist(), widx.tolist(), codes[rows, widx].tolist()))
    np.testing.assert_array_equal(adm, admit)


def check_rows(eng, got, rng):
    pick = np.sort(rng.choice(got.admit.shape[0], size=min(got.admit.shape[0], 77), replace=False)).astype(np.int64)
    codes, admit = eng.get_check_rows(pick)
    np.testing.assert_array_equal(codes, got.codes[pick])
    np.testing.assert_array_equal(admit, got.admit[pick])


@pytest.mark.parametrize("name", list(CADENCE))
def test_plugin_cadence(kt, oracle, name):
    """One engine per shape through the plugin's cycle: reconcile-only, status upload, reservations, check-only, whole passes
    chained and fused, queue admission, check-only again.  Every pass against the oracle under the same flags."""
    kw, want_variant, tppad = CADENCE[name]
    snap = make(kw)
    assert compile_tables(kt, snap)["TPpad"] == tppad
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)  # with the snapshot's reservations
    P = snap.pending.n

    # 1. a whole pass, fused: its plan names the variants the chained kernels take for these tables
    prev = run_pass(eng, snap, FRESH, 1)
    plan = eng.pass_plan()
    assert (plan.tile, plan.tpc, plan.b, plan.rt) == want_variant
    W = prev.words_per_row
    ev = lambda flags: oracle.columnar_evaluate(snap, flags, words_per_row=W)
    assert_same(snap, prev, ev(FRESH))
    rec_v, chk_v = reconcile_variant(plan), check_variant(plan, snap.L)
    assert rec_v in RECONCILE_VARIANTS and chk_v in CHECK_VARIANTS

    # 2. reconcile only: the reconcile half, and the pending outputs exactly as the fused pass left them
    got = run_pass(eng, snap, REC_ONLY, 2)
    fresh = ev(REC_ONLY)
    assert_same(snap, got, with_pending_of(fresh, prev))
    _ran.add(("reconcile", "skip_check", rec_v))

    # 3. an observed status, then reconcile-only twice: the device diff alternates its counters pass by pass
    st = observed_status(fresh, snap, rng)
    snap.status = st
    snap.normalize()
    eng.upload_status(snap)
    for _ in range(2):
        got = run_pass(eng, snap, REC_ONLY, 2)
        assert_same(snap, got, with_pending_of(fresh, prev))
        check_diff(eng, snap, got, st)

    # 4. reservations, then check-only passes (sparse list on)
    cap = 2 * W * P + 64
    eng.set_sparse_check(cap)
    set_reserved(eng, snap, random_reserved(snap, rng))
    last = got
    for flags, reserve in ((CHK_ONLY, True), (CHK_ONLY | ON_EQUAL, True), (CHK_ONLY, False)):
        if not reserve:
            set_reserved(eng, snap, (None, None, None))
        got = run_pass(eng, snap, flags, 2)
        want = ev(flags)
        assert_same(snap, got, want, check_reconcile=False)  # `used` is not this pass's: the last reconcile's sums
        np.testing.assert_array_equal(got.run_bitmap, last.run_bitmap, err_msg="a check-only pass wrote the running match rows")
        check_sparse(eng, got.codes, got.admit, cap)
        check_rows(eng, got, rng)
        _ran.add(("check", "skip_reconcile", chk_v))
        last = got

    # 5. whole passes, chained (timing on) and fused: the third and later reconciling passes must not see a half left non-zero
    got = run_pass(eng, snap, FRESH, 3, timing=True)
    assert_same(snap, got, ev(FRESH))
    _ran.add(("reconcile", "chained", rec_v))
    _ran.add(("check", "chained", chk_v))
    got = run_pass(eng, snap, FRESH, 1)
    assert_same(snap, got, ev(FRESH))
    check_sparse(eng, got.codes, got.admit, cap)

    # 6. queue admission on a sub-range, then check-only: the admission leaves nothing behind for the next pass
    set_reserved(eng, snap, random_reserved(snap, rng))
    first, count = P // 5, P // 2
    _, admitted = eng.admit_queue(first, count)
    got = eng.download()
    want, n_adm, _ = oracle.columnar_admit_queue(snap, first, count, 0, words_per_row=W)
    np.testing.assert_array_equal(got.pend_bitmap, want.pend_bitmap)
    np.testing.assert_array_equal(got.codes, want.codes)
    np.testing.assert_array_equal(got.admit, want.admit)
    assert admitted == n_adm
    got = run_pass(eng, snap, CHK_ONLY, 2)
    assert_same(snap, got, ev(CHK_ONLY), check_reconcile=False)
    check_sparse(eng, got.codes, got.admit, cap)
    eng.close()
    _cadence_shapes.add(name)


# ---- seeded event sequences on one long-lived engine ----------------------------------------------------------------------
WORLDS = {
    # fast family (L = 8, R = 4) with some ClusterThrottles; q_max = 6 re-uploads move it into the general family for a while
    "fast": dict(config="C2", m=300, n=4000, p=1000, n_ns=24, cluster_frac=0.1),
    # general family (L = 12), ClusterThrottle-heavy
    "general": dict(config="C3", m=400, n=5000, p=1200, L=12, n_ns=50),
}
STREAMS = [("fast", 11), ("fast", 12), ("general", 13), ("general", 14)]
M_CHOICES = (200, 300, 450, 600)  # words per row 8, 12, 16, 20
N_RANGE, P_RANGE = (3000, 6000), (500, 1500)
THROTTLE_FIELDS = ("kind", "thr_ns", "thr_flags", "thr", "thr_present", "thr_cnt", "ovr_off", "ovr_begin", "ovr_end", "ovr_flags", "ovr_thr",
                   "ovr_present", "ovr_cnt", "term_off", "term_flags", "pod_req_off", "ns_req_off", "req_key", "req_op", "req_val_off", "req_vals")
STEPS = 30


class Stream:
    """An engine and its model (a Snapshot): every mutation goes to both.  `ref` holds, per kind, the oracle result of the last
    pass that wrote that kind's match rows (and, for pending rows, the codes and admit bits), until the rows or the tables change:
    a pass that does not write them must leave them as they are, and the getters must read them."""

    def __init__(self, kt, oracle, world, seed):
        base = dict(WORLDS[world])
        self.config = base.pop("config")
        self.base = base
        self.oracle = oracle
        self.rng = np.random.default_rng(seed)
        self.model = synth.generate(self.config, seed=seed, **base)
        self.donor = synth.generate(self.config, seed=seed + 1000, **dict(base, n=N_RANGE[1], p=P_RANGE[1]))  # rows to draw from
        self.n_ns = self.model.n_ns
        self.eng = kt.Engine(self.model.R, self.model.L, self.model.LN)
        self.eng.upload_snapshot(self.model)  # with the snapshot's reservations
        self.sparse_cap = 0
        self.ref = {RUN: None, PEND: None}
        self.log = []

    # -- mutations --------------------------------------------------------------------------------------------------------
    def pods(self, kind):
        return self.model.running if kind == RUN else self.model.pending

    def row_delta(self, kind):
        rng, pods = self.rng, self.pods(kind)
        src = self.donor.running if kind == RUN else self.donor.pending
        k = int(rng.integers(1, 200))
        rows = np.sort(rng.choice(pods.n, size=k, replace=False)).astype(np.int64)
        delta = src.rows(rng.integers(0, src.n, size=k))
        what = rng.integers(0, 3, size=k)  # 0: moves to another namespace (another word list), 1: deleted, 2: relabelled in place
        moved = what == 0
        delta.ns_id[moved] = (pods.ns_id[rows[moved]] + rng.integers(1, self.n_ns, size=int(moved.sum()))) % self.n_ns
        gone = what == 1
        delta.flags[gone] = 0
        delta.labels[:, gone] = abi.LABEL_EMPTY
        kept = what == 2
        delta.ns_id[kept] = pods.ns_id[rows[kept]]
        self.eng.update_pod_rows(kind, rows, delta)
        for name in ("labels", "req"):
            getattr(pods, name)[:, rows] = getattr(delta, name)
        for name in ("present", "flags", "ns_id"):
            getattr(pods, name)[rows] = getattr(delta, name)
        self.ref[kind] = None
        return f"delta kind={kind} k={k} moved={int(moved.sum())} deleted={int(gone.sum())}"

    def reupload(self, kind):
        rng = self.rng
        src = self.donor.running if kind == RUN else self.donor.pending
        lo, hi = N_RANGE if kind == RUN else P_RANGE
        n = int(rng.integers(lo, hi + 1))
        start = int(rng.integers(0, src.n - n + 1))
        pods = src.rows(slice(start, start + n))
        fmt = ("wide", "compact", "packed")[int(rng.integers(3))]
        if fmt == "wide":
            self.eng.upload_pods(kind, pods)
        elif fmt == "compact":
            self.eng.upload_pods_compact(kind, abi.compact_pods(pods))
        else:  # with tables in place: unpacked and translated in one kernel
            self.eng.upload_pods_packed(kind, abi.packed_pods(pods, code_requests=bool(rng.integers(2))))
        if kind == RUN:
            self.model.running = pods
        else:
            self.model.pending = pods
        self.model.normalize()
        self.ref[kind] = None
        return f"reupload kind={kind} n={n} {fmt}"

    def throttles(self):
        rng, model = self.rng, self.model
        m = int(rng.choice([x for x in M_CHOICES if x != model.m]))
        terms = (None, 1, 2)[int(rng.integers(3))]
        q_max = 6 if rng.random() < 0.3 else 0
        t = synth.generate(self.config, **dict(self.base, seed=int(rng.integers(1 << 30)), m=m, n=model.running.n, p=100, terms=terms, q_max=q_max))
        for f in THROTTLE_FIELDS:
            setattr(model, f, getattr(t, f))
        model.status = model.reserved = model.reserved_present = model.reserved_cnt = None  # the engine drops both
        model.normalize()
        self.eng.upload_throttles(model)
        self.ref = {RUN: None, PEND: None}
        return f"throttles m={m} terms={terms} q_max={q_max} Wp={self.eng.words_per_row}"

    def namespaces(self):
        rng, model = self.rng, self.model
        ns = model.ns_labels.copy()
        pick = rng.random(self.n_ns) < 0.4
        ns[1, pick] = (np.int64(synth.NS_KEY_TEAM) << 32) | rng.integers(0, synth.N_TEAMS, size=int(pick.sum()))
        ns[2, pick] = (np.int64(synth.NS_KEY_ENV) << 32) | rng.integers(0, synth.N_ENVS, size=int(pick.sum()))
        model.ns_labels = np.ascontiguousarray(ns)
        self.eng.upload_namespaces(model.ns_labels)
        self.ref = {RUN: None, PEND: None}
        return f"namespaces relabelled={int(pick.sum())}"

    def upload_status(self):
        fresh = self.oracle.columnar_evaluate(self.model, words_per_row=self.eng.words_per_row)
        self.model.status = observed_status(fresh, self.model, self.rng)
        self.model.normalize()
        self.eng.upload_status(self.model)
        return "status"

    def reserve(self):
        set_reserved(self.eng, self.model, random_reserved(self.model, self.rng))
        return "reserve"

    def unreserve(self):
        set_reserved(self.eng, self.model, (None, None, None))
        return "unreserve"

    def toggle_sparse(self):
        self.sparse_cap = 0 if self.sparse_cap else 1 << 16
        self.eng.set_sparse_check(self.sparse_cap)
        return f"sparse cap={self.sparse_cap}"

    # -- passes -----------------------------------------------------------------------------------------------------------
    def full_flags(self):
        return (FRESH, ON_EQUAL, GIVEN)[int(self.rng.integers(3 if self.model.status is not None else 2))]

    def evaluate(self, kind):
        rng, model = self.rng, self.model
        if kind in ("check_only", "admit") and model.status is None:
            self.log.append(self.upload_status())
        if kind == "admit":
            return self.admit()
        timing = kind == "chained"
        if kind == "reconcile_only":
            flags, launches = REC_ONLY, 2
        elif kind == "check_only":
            flags, launches = CHK_ONLY | (ON_EQUAL if rng.random() < 0.5 else 0), 2
        else:
            flags, launches = self.full_flags(), (3 if timing else 1)
        self.log.append(f"{kind} flags={flags}")
        got = run_pass(self.eng, model, flags, launches, timing)
        want = self.oracle.columnar_evaluate(model, flags, words_per_row=got.words_per_row)
        rec, chk = not flags & abi.EVAL_SKIP_RECONCILE, not flags & abi.EVAL_SKIP_CHECK
        w = copy.copy(want)
        if not chk:  # what the last checking pass left, when the rows and tables are still the same (else not compared)
            w = with_pending_of(want, self.ref[PEND] or got)
        assert_same(model, got, w, check_reconcile=rec)
        if not rec and self.ref[RUN] is not None:
            np.testing.assert_array_equal(got.run_bitmap, self.ref[RUN].run_bitmap, err_msg="a check-only pass changed the running match rows")
        if rec:
            self.ref[RUN] = want
        if chk:
            self.ref[PEND] = want
            if self.sparse_cap:
                check_sparse(self.eng, want.codes, want.admit, self.sparse_cap)
        return got

    def admit(self):
        rng, model = self.rng, self.model
        P = model.pending.n
        first = int(rng.integers(0, P // 2))
        count = int(rng.integers(1, P - first + 1))
        flags = ON_EQUAL if rng.random() < 0.5 else 0
        self.log.append(f"admit first={first} count={count} flags={flags}")
        _, admitted = self.eng.admit_queue(first, count, flags)
        got = self.eng.download()
        want, n_adm, _ = self.oracle.columnar_admit_queue(model, first, count, flags, words_per_row=got.words_per_row)
        np.testing.assert_array_equal(got.pend_bitmap, want.pend_bitmap)
        np.testing.assert_array_equal(got.codes, want.codes)
        np.testing.assert_array_equal(got.admit, want.admit)
        assert admitted == n_adm
        self.ref[PEND] = want
        return got

    def check_getters(self):
        """Match rows of random rows and match columns of a few throttles, read from the maintained bitmaps (and codes)."""
        rng, m = self.rng, self.model.m
        for kind in (RUN, PEND):
            ref = self.ref[kind]
            if ref is None:
                continue
            bitmap = ref.run_bitmap if kind == RUN else ref.pend_bitmap
            rows = rng.choice(bitmap.shape[0], size=min(bitmap.shape[0], 64), replace=False).astype(np.int64)
            np.testing.assert_array_equal(self.eng.match_rows(kind, rows), bitmap[rows], err_msg=f"match rows, kind {kind}")
            idx = rng.integers(0, m, size=5)
            off, got_rows, codes = self.eng.match_columns(kind, idx)
            w_off, w_rows, w_codes = numpy_columns(bitmap, m, idx, ref.codes if kind == PEND else None)
            np.testing.assert_array_equal(off, w_off)
            np.testing.assert_array_equal(got_rows, w_rows)
            if kind == PEND:
                np.testing.assert_array_equal(codes, w_codes)


MUTATIONS = (("delta_running", 3), ("delta_pending", 3), ("reupload_running", 1), ("reupload_pending", 1), ("throttles", 1.5), ("namespaces", 1),
             ("status", 1), ("reserve", 1), ("unreserve", 0.5), ("sparse", 0.5))
PASSES = (("reconcile_only", 3), ("check_only", 3), ("fused", 1.5), ("chained", 1.5), ("admit", 1))


def _pick(rng, table):
    names, w = zip(*table)
    return names[int(rng.choice(len(names), p=np.asarray(w) / sum(w)))]


@pytest.mark.parametrize("world,seed", STREAMS, ids=[f"{w}-{s}" for w, s in STREAMS])
def test_event_stream(kt, oracle, world, seed):
    """A long-lived engine through row deltas (namespace moves, deletions, relabels), re-uploads in every format with other row
    counts, throttle re-uploads that move Wp, TPpad and B, namespace relabels, status / reservation / sparse-list settings, and
    every kind of pass; after each pass its outputs and the getters against the oracle on the model."""
    s = Stream(kt, oracle, world, seed)
    acts = dict(delta_running=lambda: s.row_delta(RUN), delta_pending=lambda: s.row_delta(PEND), reupload_running=lambda: s.reupload(RUN),
                reupload_pending=lambda: s.reupload(PEND), throttles=s.throttles, namespaces=s.namespaces, status=s.upload_status,
                reserve=s.reserve, unreserve=s.unreserve, sparse=s.toggle_sparse)
    kinds = set()
    for step in range(STEPS):
        try:
            if step > 0 and s.rng.random() < 0.6:
                s.log.append(acts[_pick(s.rng, MUTATIONS)]())
            kind = "fused" if step == 0 else _pick(s.rng, PASSES)
            s.evaluate(kind)
            s.check_getters()
            kinds.add(kind)
        except Exception as e:
            raise AssertionError(f"seed {seed}, step {step}, last operations {s.log[-5:]}") from e
    s.eng.close()
    assert {"reconcile_only", "check_only"} <= kinds


# ---- edges only the chained path takes ------------------------------------------------------------------------------------
@pytest.mark.parametrize("base", ["fast128_t1_r4", "fast128_t2_r8", "general_t1_b2", "general_t2_b6"])
def test_empty_tables_and_check_tile_edges(kt, oracle, base):
    """On an engine that has run non-empty passes: no running rows (chained finalize + check: nothing counted, Counts nil, Q3),
    no pending rows (chained reconcile + finalize), back to both (nothing of the empty passes leaks into the sums), then a single
    pending row and pending counts around kTileCheck = 64 in whole chained, check-only and fused passes."""
    kw, _, _ = SHAPES[base]
    full = make(kw)
    N, P = full.running.n, full.pending.n
    eng = kt.Engine(full.R, full.L, full.LN)
    eng.upload_snapshot(full)
    got = run_pass(eng, full, FRESH, 1)
    W = got.words_per_row
    ev = lambda snap, flags=FRESH: oracle.columnar_evaluate(snap, flags, words_per_row=W)
    assert_same(full, got, ev(full))

    snap = with_rows(full, 0, P)
    eng.upload_pods(RUN, snap.running)
    got = run_pass(eng, snap, FRESH, 2)
    assert_same(snap, got, ev(snap))
    assert not got.used.any() and not got.used_cnt.any() and not (got.used_present & abi.COUNT_BIT).any()

    snap = with_rows(full, N, 0)
    eng.upload_pods(RUN, snap.running)
    eng.upload_pods(PEND, snap.pending)
    got = run_pass(eng, snap, FRESH, 2)
    assert_same(snap, got, ev(snap))

    eng.upload_pods(PEND, full.pending)
    for launches, timing in ((1, False), (3, True), (1, False)):
        got = run_pass(eng, full, FRESH, launches, timing)
        assert_same(full, got, ev(full))

    full.status = observed_status(got, full, np.random.default_rng(5))
    full.normalize()
    eng.upload_status(full)
    for p in (1, 63, 64, 65, 129):
        snap = with_rows(full, N, p)
        eng.upload_pods(PEND, snap.pending)
        for flags, launches, timing in ((FRESH, 3, True), (CHK_ONLY, 2, False), (CHK_ONLY | ON_EQUAL, 2, False), (FRESH, 1, False)):
            got = run_pass(eng, snap, flags, launches, timing)
            assert_same(snap, got, ev(snap, flags), check_reconcile=not flags & abi.EVAL_SKIP_RECONCILE)
    eng.close()


def test_cadence_reached_every_chained_variant():
    """Runs after the cadence: every k_reconcile variant (8) ran in reconcile-only and in whole chained passes, every k_check
    variant (6) in check-only and in whole chained passes."""
    if _cadence_shapes != set(CADENCE):
        pytest.skip("the cadence did not run in full")
    for kernel, modes, want in (("reconcile", ("skip_check", "chained"), RECONCILE_VARIANTS), ("check", ("skip_reconcile", "chained"), CHECK_VARIANTS)):
        for mode in modes:
            ran = {v for k, md, v in _ran if (k, md) == (kernel, mode)}
            assert ran == want, (kernel, mode, sorted(want - ran))
    assert len(RECONCILE_VARIANTS) == 8 and len(CHECK_VARIANTS) == 6
