"""Namespace word lists past their encodings: the fused pass, the keyed calls, kt_admit_queue and namespace row deltas where a
namespace's list of 32-throttle words outgrows the regimes the device handles it in.

  slots      more than kMaxSlots - 2 = 30 words in a namespace: the reconcile tile's accumulator slots fill up and later words go
             straight to the HBM partials; the decide tile's staging table fills up
  list       3..254 words: the row inlines its first two words, the rest comes from nsw_off / nsw_idx; the inlined count
             saturates at 254, so 254, 255 and 256 words take the same inlined count
  inline12   tables of up to 4096 words inline 12-bit word indices (indices of 2048 and up use the field's top bit); wider tables
             (W = 4097) inline nothing
  deltas     kt_update_namespace_rows past W = 32 (k_ns_count / k_ns_fill carry a count across 32-word rounds), past 1024
             namespaces (k_ns_scan gives each thread a run of namespaces) and past 65535 evaluated rows in one call (k_ns_rows'
             grid is chunked in y)

The worlds are synth's pods and podSelectors with rewritten namespace sides.  In the group worlds every namespace carries a
`group` label, and each word's ClusterThrottles select `group In {...}`, so a namespace of group g has exactly the words of g.
Thresholds are set from the oracle's FRESH sums so that the pending pods are partly admitted, partly rejected.  The CPU test
asserts that each world reaches its regime; the GPU tests compare the engine with the columnar oracle and, for the row deltas,
with kt_debug_compile_tables and an engine that gets every namespace change as a whole upload."""
import copy
import functools

import numpy as np
import pytest

from kube_throttler_b200 import abi, synth
from test_check_summary import expected as summary_of
from test_gpu_parity import _live
from test_match_columns import numpy_columns
from test_namespace_rows import FRESH, GIVEN, PLANS, assert_oracle, assert_same, assert_tables, batches, new_rows, observe, setup
from test_partial_passes import check_diff, check_sparse, observed_status, random_reserved
from test_reconcile_throttles import STATUS_FIELDS
from test_tables_cpu import compile_tables

GROUP = 103          # namespace label key of the group worlds, in namespace label slot 3
K_MAX_SLOTS = 32     # kt_kernels.cuh kMaxSlots
ON_EQ = abi.EVAL_ON_EQUAL


# ---- worlds -----------------------------------------------------------------------------------------------------------------
def reqs_of(snap, off):
    """Per term, the requirements [(key, op, [vals])] of the selector whose CSR offsets are `off` (pod_req_off or ns_req_off)."""
    vo = snap.req_val_off
    return [[(int(snap.req_key[q]), int(snap.req_op[q]), [int(v) for v in snap.req_vals[vo[q]:vo[q + 1]]]) for q in range(off[j], off[j + 1])]
            for j in range(len(off) - 1)]


def set_reqs(snap, ns_reqs, pod_reqs=None):
    """The snapshot's selector CSR with every term's namespaceSelector (and, given, podSelector) replaced."""
    pod_reqs = reqs_of(snap, snap.pod_req_off) if pod_reqs is None else pod_reqs
    for k, v in synth.build_selector_csr(snap.term_off, pod_reqs, ns_reqs, snap.term_flags).items():
        setattr(snap, k, v)
    return snap.normalize()


def spread_pods(snap, rng, weights, sort):
    """Pods' namespaces drawn from `weights` (the labels are drawn independently of the namespace)."""
    p = np.asarray(weights, float) / np.sum(weights)
    for pods in (snap.running, snap.pending):
        ns = rng.choice(len(p), size=pods.n, p=p).astype(np.int32)
        pods.ns_id = np.sort(ns) if sort else ns


def group_world(m, counts, ns_group, owners, *, n, p, seed, sort=True, q_max=0, throttle_frac=0.3, weights=None):
    """ClusterThrottle-heavy world over len(ns_group) namespaces; namespace i is in group ns_group[i], group g has counts[g]
    distinct words (group 0 every word).  Every word's first throttle selects `group In {the groups that have the word}`, the
    others a subset of those groups (some with synth's team / env requirements on top), or are Throttles of an `owners`
    namespace of such a group.  A namespace that owns no Throttle has exactly the words of its group."""
    W = (m + 31) // 32
    assert counts[0] == W
    snap = synth.generate("C3", seed=seed, m=m, n=n, p=p, n_ns=len(ns_group), cluster_frac=1.0, calibrate=False, sort_by_namespace=sort,
                          q_max=q_max)
    rng = np.random.default_rng(seed)
    ns_group = np.asarray(ns_group)
    snap.ns_labels[3] = synth._lab(GROUP, ns_group)
    has = np.zeros((len(counts), W), bool)
    for g, c in enumerate(counts):
        has[g, rng.choice(W, size=c, replace=False)] = True
    old = reqs_of(snap, snap.ns_req_off)
    reqs = [None] * len(old)
    kind = np.full(m, abi.KIND_CLUSTERTHROTTLE, np.uint8)
    thr_ns = np.full(m, -1, np.int32)
    owners = np.asarray(owners)
    for t in range(m):
        g_w = np.flatnonzero(has[:, t // 32])
        cand = owners[np.isin(ns_group[owners], g_w)]
        u = rng.random()
        if t % 32 and u < throttle_frac and cand.size:
            kind[t], thr_ns[t], sel = abi.KIND_THROTTLE, rng.choice(cand), None
        elif t % 32 == 0:
            snap.thr_flags[t] = abi.THR_RESPONSIBLE  # the word's anchor: it must apply
            sel = [(GROUP, abi.OP_IN, [int(g) for g in g_w])]
        else:
            sub = [int(g) for g in g_w if rng.random() < 0.5] or [int(rng.choice(g_w))]
            sel = [(GROUP, abi.OP_IN, sub)]
        for j in range(snap.term_off[t], snap.term_off[t + 1]):
            reqs[j] = [] if sel is None else sel + (old[j] if u > 0.8 else [])
    snap.kind, snap.thr_ns = kind, thr_ns
    spread_pods(snap, rng, np.ones(len(ns_group)) if weights is None else weights, sort)
    set_reqs(snap, reqs)
    snap.meta.update(counts=list(counts), ns_group=ns_group)
    return snap


def slots_world(sort=True, q_max=0):
    """synth C3 with 1260 ClusterThrottles: every word applies to every namespace (44 words, more than kMaxSlots)."""
    return synth.generate("C3", m=1400, n=3000, p=900, n_ns=40, cluster_frac=0.9, calibrate=False, sort_by_namespace=sort, q_max=q_max)


LIST_COUNTS = [282, 256, 255, 254, 253, 3, 2, 1, 31, 29, 0]  # M = 9000: W = 282


def list_world():
    """W = 282: namespaces 0..10 have exactly LIST_COUNTS words (every word; 256, 255, 254 and 253; 3, 2, 1; 31, 29; none) and
    own no Throttle; namespaces 11..39 are in random groups and own the Throttles."""
    groups = list(range(11)) + list(np.random.default_rng(254).choice([0, 5, 6, 7, 8, 9, 10], size=29))
    weights = [4] * 11 + [1] * 29
    return group_world(9000, LIST_COUNTS, groups, np.arange(11, 40), n=3000, p=1000, seed=254, weights=weights)


def wide_world(m):
    """4096 namespaces, namespace i owning the Throttles of word i; 64 ClusterThrottles select `metadata.name In {...}` over 1..40
    namespaces; with M = 131073 the last throttle is a Throttle of namespace 4000 (words 4000 and 4096 inline, if anything were
    inlined at W = 4097).  Pods in every namespace, more of them in 4000 and the upper half."""
    n_ns = 4096
    snap = synth.generate("C3", seed=4096, m=m, n=3000, p=1500, n_ns=n_ns, cluster_frac=0.0, calibrate=False)
    rng = np.random.default_rng(m)
    t = np.arange(m)
    snap.thr_ns = np.minimum(t // 32, n_ns - 1).astype(np.int32)
    if m > n_ns * 32:
        snap.thr_ns[n_ns * 32:] = 4000
        snap.thr_flags[n_ns * 32:] = abi.THR_RESPONSIBLE
    cluster = rng.choice(m - 1, size=64, replace=False)
    snap.kind[cluster] = abi.KIND_CLUSTERTHROTTLE
    snap.thr_ns[cluster] = -1
    reqs = [[] for _ in range(int(snap.term_off[-1]))]
    for c in cluster:
        names = rng.choice(n_ns, size=int(rng.integers(1, 41)), replace=False)
        names = names[names != 4000]
        for j in range(snap.term_off[c], snap.term_off[c + 1]):
            reqs[j] = [(synth.NS_KEY_NAME, abi.OP_IN, [1000 + int(x) for x in names])]
    pod_reqs = reqs_of(snap, snap.pod_req_off)
    if m > n_ns * 32:  # namespace 4000's pods match the last throttle: `key 0 NotIn {0}`
        for j in range(snap.term_off[m - 1], snap.term_off[m]):
            pod_reqs[j] = [(0, abi.OP_NOTIN, [0])]
    w = np.ones(n_ns)
    w[n_ns // 2:] = 3
    w[4000] = 300
    spread_pods(snap, rng, w, True)
    return set_reqs(snap, reqs, pod_reqs)


WORLDS = {
    "slots_sorted": lambda: slots_world(),
    "slots_arrival": lambda: slots_world(sort=False),
    "slots_q6": lambda: slots_world(q_max=6),
    "list_254": list_world,
    "wide_4096": lambda: wide_world(4096 * 32),
    "wide_4097": lambda: wide_world(4096 * 32 + 1),
}


@functools.lru_cache(maxsize=None)
def world(name):
    return WORLDS[name]()


# ---- the CPU check: every world reaches its regime ----------------------------------------------------------------------------
def word_lists(kt, snap):
    t = compile_tables(kt, snap)
    return t, np.diff(t["nsw_off"])


@pytest.mark.parametrize("name", list(WORLDS) + ["delta_slots", "delta_list", "delta_many", "delta_65k"])
def test_worlds_reach_their_regimes(kt, name):
    """kt_debug_compile_tables on every world: the word counts each regime needs are there (or synth has drifted)."""
    if name.startswith("delta_"):
        snap, n0, steps = delta_world(name)
        snap = copy.copy(snap)
        snap.ns_labels = np.ascontiguousarray(snap.ns_labels[:, :n0])
    else:
        snap = world(name)
    t, cnt = word_lists(kt, snap)
    W, NS, longest = t["W"], t["NS"], int(cnt.max())
    assert W == (snap.m + 31) // 32
    if name.startswith("slots"):  # slots: more words than accumulator slots in every namespace, at most 60
        assert K_MAX_SLOTS - 2 < longest <= 60 and (cnt > K_MAX_SLOTS).mean() > 0.8, (longest, cnt)
        if name == "slots_q6":
            assert t["B"] == 6  # 6-bit counters: the general kernel family
    elif name == "list_254":  # list: exactly 3, 253, 254, 255, 256 and 282 words, and 0..2-word namespaces next to them
        np.testing.assert_array_equal(cnt[:11], LIST_COUNTS)
        assert W == 282 and {0, 1, 2} <= set(cnt.tolist())
    elif name.startswith("wide"):  # inline12: W = 4096 and 4097; inlined word indices >= 2048
        assert W in (4096, 4097) and NS == 4096
        first = t["nsw_idx"][t["nsw_off"][:-1][cnt > 0]]
        assert (first >= 2048).sum() > 1000 and (cnt <= 2).mean() > 0.5 and (cnt > 2).any()
        pods_ns = np.concatenate([snap.running.ns_id, snap.pending.ns_id])
        assert (pods_ns >= 2048).mean() > 0.5
        if W == 4097:  # namespace 4000's second word is 4096: 0 in 12 bits
            assert list(t["nsw_idx"][t["nsw_off"][4000]:t["nsw_off"][4001]]) == [4000, 4096]
            rows = np.flatnonzero(snap.pending.ns_id == 4000)
            assert synth.match_matrix_numpy(snap, snap.pending, snap.m - 1, rows).any()
    elif name == "delta_slots":  # deltas past W = 32, across 30 words
        assert 32 < W <= 64 and 1024 < snap.m <= 2048
        assert any(c > 30 for c in steps_counts(steps)) and any(c <= 30 for c in steps_counts(steps))
    elif name == "delta_list":  # deltas across 254 / 255
        assert {254, 255, 256} <= set(steps_counts(steps))
    elif name == "delta_many":  # more than 1024 namespaces after the deltas, Throttles past the first count
        assert n0 <= 1024 < max(n for n, _ in steps) and (snap.thr_ns >= n0).any()
    else:  # delta_65k: one call evaluates more than 65535 rows
        assert max(n for n, _ in steps) - n0 > 65535 and snap.LN <= 2 and (snap.thr_ns >= n0).any()


def steps_counts(steps):
    """The word counts the relabel steps of a group world give the namespace they move."""
    return [c for _, moves in steps for (_, _, c) in moves]


# ---- thresholds and expected results ------------------------------------------------------------------------------------------
def calibrate(snap, oracle, rng, tight):
    """Thresholds from the oracle's FRESH sums, as synth scales them: a share `tight` of the throttles below the sum, as many
    within about one pod of it, as many at the sum exactly (isThrottledOnEqual decides), the rest with ample headroom."""
    R, m = snap.R, snap.m
    fresh = oracle.columnar_evaluate(snap, FRESH)
    used, ucnt = fresh.used, fresh.used_cnt
    one_pod = np.array([2000, 1 << 30, 2, 50 << 30] + [2] * max(0, R - 4), np.int64)[:R, None]
    u = rng.random(m)
    q = np.where(u < tight, rng.uniform(0.5, 1.0, (R, m)), rng.uniform(1.2, 2.0, (R, m)))
    thr = (np.where(used > 0, used, 4 * one_pod) * q).astype(np.int64)
    near = (u >= tight) & (u < 2 * tight)
    thr = np.where(near, used + (rng.uniform(0.0, 1.5, (R, m)) * one_pod).astype(np.int64), thr)
    exact = u > 1 - tight
    thr = np.maximum(1, np.where(exact, used, thr))
    cnt = np.maximum(1, (np.where(ucnt > 0, ucnt, 10) * q[0]).astype(np.int64))
    cnt = np.where(exact, np.maximum(ucnt, 1), np.where(near, ucnt + rng.integers(0, 3, m), cnt))
    has = (snap.thr_present[None, :] >> np.arange(R, dtype=np.uint32)[:, None]) & 1
    snap.thr = (thr * has).astype(np.int64)
    snap.thr_cnt = np.where(snap.thr_present & abi.COUNT_BIT, cnt, 0).astype(np.int64)
    return snap.normalize()


# (tight, lag): a pod of the slots worlds matches a hundred throttles or more, so few of them may stop it
TIGHT = {"slots_sorted": (0.002, 0.03), "slots_arrival": (0.002, 0.03), "slots_q6": (0.002, 0.03), "list_254": (0.002, 0.3),
         "wide_4096": (0.03, 1.0), "wide_4097": (0.03, 1.0)}


@functools.lru_cache(maxsize=None)
def prepared(name):
    """The world with thresholds, an observed status that lags behind and reservations on a share `lag` of the throttles, and
    the oracle's answers: (snap, {flags: PassResult}, columnar_admit_queue over the whole queue)."""
    from oracle import ko

    snap = copy.deepcopy(world(name))
    rng = np.random.default_rng(len(name))
    tight, lag = TIGHT[name]
    calibrate(snap, ko, rng, tight)
    Wp = abi.default_words_per_row(snap.m)
    fresh = ko.columnar_evaluate(snap, FRESH, words_per_row=Wp)
    snap.status = observed_status(fresh, snap, rng)
    res = random_reserved(snap, rng)
    keep = rng.random(snap.m) >= lag  # status current, nothing reserved
    snap.status["calculated"][keep] = 1
    for f in ("calc_thr", "calc_present", "calc_cnt", "used", "used_present", "used_cnt", "throttled"):
        snap.status[f][..., keep] = getattr(fresh, f)[..., keep]
    for col in res:
        col[..., keep] = 0
    snap.reserved, snap.reserved_present, snap.reserved_cnt = res
    snap.normalize()
    want = {f: ko.columnar_evaluate(snap, f, words_per_row=Wp) for f in (FRESH, GIVEN, GIVEN | ON_EQ)}
    return snap, want, ko.columnar_admit_queue(snap, 0, snap.pending.n, 0, words_per_row=Wp)


def assert_pass(got, want, where):
    for f in ("pend_bitmap", "codes", "admit"):
        np.testing.assert_array_equal(getattr(got, f), getattr(want, f), err_msg=f"{where}: {f}")


def assert_fresh(got, want, live, where):
    assert_pass(got, want, where)
    np.testing.assert_array_equal(got.run_bitmap, want.run_bitmap, err_msg=f"{where}: run_bitmap")
    for f in STATUS_FIELDS[:-1]:
        np.testing.assert_array_equal(getattr(got, f)[..., live], getattr(want, f)[..., live], err_msg=f"{where}: {f}")


def widest(kt, snap):
    """The namespaces with pending pods, longest word list first, and the compiled tables."""
    t, cnt = word_lists(kt, snap)
    cnt = np.where(np.isin(np.arange(cnt.size), snap.pending.ns_id), cnt, -1)
    return np.argsort(-cnt, kind="stable"), t


# ---- the GPU checks on the static worlds -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WORLDS))
def test_passes_equal_the_oracle(kt, oracle, name):
    """FRESH and GIVEN passes queued back to back under every forced plan and the automatic one: bitmaps, codes, admit bits, the
    status columns of live throttles, the changed list and the sparse check list, against the oracle."""
    snap, want, _ = prepared(name)
    live = _live(snap)
    P = snap.pending.n
    adm = want[GIVEN].admit.mean()
    assert 0.05 < adm < 0.95 and 0.05 < want[FRESH].admit.mean() < 0.95, (adm, want[FRESH].admit.mean())
    cap = 2 * max(int(np.count_nonzero(w.codes)) for w in want.values()) + 64
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    eng.set_sparse_check(cap)
    for plan in PLANS:
        where = f"{name} plan {plan}"
        eng.set_pass_plan(*plan)
        eng.evaluate(snap.now, FRESH)
        eng.evaluate(0, GIVEN)  # queued right behind the FRESH pass
        got = eng.download()
        assert_pass(got, want[GIVEN], where + " GIVEN")
        check_sparse(eng, got.codes, got.admit, cap)
        eng.evaluate(snap.now, FRESH)
        got = eng.download()
        assert_fresh(got, want[FRESH], live, where + " FRESH")
        check_diff(eng, snap, got, snap.status)
        check_sparse(eng, got.codes, got.admit, cap)
        eng.evaluate(0, GIVEN | ON_EQ)
        assert_pass(eng.download(), want[GIVEN | ON_EQ], where + " GIVEN on equal")
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WORLDS))
def test_keyed_calls_and_queue_admission_equal_the_oracle(kt, oracle, name):
    """kt_check_pending_rows, kt_check_pods, kt_match_pods over the rows of the widest namespaces; kt_reconcile_throttles and
    kt_get_match_columns over throttles of more than 32 words, the widest namespace's among them; kt_get_check_summary; and
    kt_admit_queue over the whole queue."""
    snap, want, (w_adm, n_adm, _) = prepared(name)
    rng = np.random.default_rng(7)
    m, P = snap.m, snap.pending.n
    wide, t = widest(kt, snap)
    rows = np.flatnonzero(np.isin(snap.pending.ns_id, wide[:3]))
    last = np.flatnonzero(np.isin(snap.pending.ns_id, np.flatnonzero(t["nsmask"][:, -1].any(axis=1))))  # the top word's namespaces
    rows = np.concatenate([rng.choice(rows, size=min(rows.size, 96), replace=False), rng.choice(last, size=min(last.size, 32), replace=False),
                           rng.integers(0, P, size=16)]).astype(np.int64)
    lo, hi = t["nsw_off"][wide[0]], t["nsw_off"][wide[0] + 1]
    words = np.union1d(t["nsw_idx"][lo:hi], rng.choice(t["W"], size=40, replace=False))
    assert words.size > 32
    idx = np.minimum(words * 32 + rng.integers(0, 32, size=words.size), m - 1)
    idx = np.concatenate([idx, np.arange(words[0] * 32, min(m, words[0] * 32 + 32))]).astype(np.int32)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    pods = snap.pending.rows(rows)
    for on_equal, w in ((False, want[GIVEN]), (True, want[GIVEN | ON_EQ])):
        for call, got in (("check_pending_rows", eng.check_pending_rows(rows, on_equal)),
                          ("check_pods", eng.check_pods(pods.labels, pods.req, pods.present, pods.ns_id, on_equal))):
            for f, g, x in zip(("words", "codes", "admit"), got, (w.pend_bitmap, w.codes, w.admit)):
                np.testing.assert_array_equal(g, x[rows], err_msg=f"{name} {call} {f} on_equal={on_equal}")
    np.testing.assert_array_equal(eng.match_pods(pods.labels, pods.ns_id), want[GIVEN].pend_bitmap[rows], err_msg=f"{name} match_pods")
    st, off, rrows = eng.reconcile_throttles(snap.now, idx)
    for f in STATUS_FIELDS:
        np.testing.assert_array_equal(getattr(st, f), getattr(want[FRESH], f)[..., idx], err_msg=f"{name} reconcile_throttles {f}")
    w_off, w_rows, _ = numpy_columns(want[FRESH].run_bitmap, m, idx)
    np.testing.assert_array_equal(off, w_off, err_msg=f"{name} reconcile_throttles off")
    np.testing.assert_array_equal(rrows, w_rows, err_msg=f"{name} reconcile_throttles rows")
    eng.evaluate(snap.now, FRESH)
    for kind, bm, codes in ((abi.PODS_RUNNING, want[FRESH].run_bitmap, None), (abi.PODS_PENDING, want[FRESH].pend_bitmap, want[FRESH].codes)):
        got = eng.match_columns(kind, idx)
        for f, g, x in zip(("off", "rows", "codes"), got, numpy_columns(bm, m, idx, codes)):
            if x is not None:
                np.testing.assert_array_equal(g, x, err_msg=f"{name} match_columns kind {kind} {f}")
    for first, count in ((0, P), (P // 3, P // 2), (P - 1, 1)):
        got = eng.check_summary(first, count)
        for f, g, x in zip(("status_cnt", "sole_cnt", "held", "held_present"), got, summary_of(snap, want[FRESH].codes, want[FRESH].admit, first, count)):
            np.testing.assert_array_equal(g, x, err_msg=f"{name} check_summary [{first}, +{count}) {f}")
    _, admitted = eng.admit_queue(0, P)
    got = eng.download()
    for f in ("pend_bitmap", "codes", "admit"):
        np.testing.assert_array_equal(getattr(got, f), getattr(w_adm, f), err_msg=f"{name} admit_queue {f}")
    assert admitted == n_adm and 0 < n_adm < P
    eng.close()


# ---- namespace row deltas ----------------------------------------------------------------------------------------------------
SLOT_COUNTS = [41, 31, 30, 29, 3, 2, 1, 0]  # M = 1300: W = 41


@functools.lru_cache(maxsize=None)
def delta_world(name):
    """(snap with every namespace row the test ends with, the first namespace count, steps).  A step is (namespace count, moves):
    moves (namespace, group, that group's word count) relabel one namespace of a group world; steps without moves relabel random
    rows (test_namespace_rows.new_rows) and list the new rows."""
    if name == "delta_slots":  # W = 41; namespace 3 (29 words) moves across 30 and back; Throttles of namespaces 24..29 exist first
        groups = list(range(8)) + list(np.random.default_rng(30).choice([0, 1, 4, 5, 6, 7], size=22))
        snap = group_world(1300, SLOT_COUNTS, groups, np.arange(8, 30), n=2500, p=800, seed=30)
        c = SLOT_COUNTS
        steps = [(24, [(3, 1, c[1])]), (24, [(3, 2, c[2]), (5, 0, c[0])]), (30, [(3, 0, c[0])]), (30, []), (30, [(3, 3, c[3]), (5, 5, c[5])])]
        return snap, 24, steps
    if name == "delta_list":  # W = 282; namespaces 3 (254) and 2 (255) move across 254 / 255 and back
        snap = list_world()
        c = LIST_COUNTS
        steps = [(40, [(3, 2, c[2])]), (40, [(3, 1, c[1]), (2, 3, c[3])]), (40, [(3, 3, c[3]), (2, 2, c[2])]), (40, [(6, 1, c[1])]),
                 (40, [(6, 6, c[6])]), (40, [])]
        return snap, 40, steps
    if name == "delta_many":  # 900 namespaces, grown past 1024 by deltas
        snap = synth.generate("C3", seed=1025, m=300, n=3000, p=900, n_ns=1500, cluster_frac=0.5)
        return snap, 900, [(1000, []), (1100, []), (1100, []), (1500, []), (1500, [])]
    # delta_65k: namespace labels {name, team} (LN = 2); 40 namespaces, then one call grows the count to 70040
    snap = synth.generate("C3", seed=65535, m=64, n=3000, p=900, n_ns=70040, cluster_frac=0.5)
    snap.ns_labels = np.ascontiguousarray(snap.ns_labels[:2])
    snap.LN = 2
    set_reqs(snap, [[r for r in reqs if r[0] != synth.NS_KEY_ENV] for reqs in reqs_of(snap, snap.ns_req_off)])
    rng = np.random.default_rng(65535)
    for pods in (snap.running, snap.pending):
        pods.ns_id = np.sort(rng.integers(0, 70040, size=pods.n)).astype(np.int32)
    return snap, 40, [(70040, []), (70040, [])]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["delta_slots", "delta_list", "delta_many", "delta_65k"])
def test_row_deltas_across_the_regimes(kt, oracle, name):
    """Row deltas that move namespaces across 30 and 254 / 255 words and back, grow the count past 1024 and by more than 65535 rows
    in one call, and over Throttles whose namespace has no row yet.  After every step: the resident namespace masks and word lists
    equal kt_debug_compile_tables', the delta engine answers bit for bit as the engine that got whole uploads, and (once every
    Throttle's namespace has a row) FRESH and GIVEN passes equal the oracle."""
    full_snap, n0, steps = delta_world(name)
    snap = copy.deepcopy(full_snap)
    pool = np.ascontiguousarray(full_snap.ns_labels)
    LN = pool.shape[0]
    rng = np.random.default_rng(len(name))
    calibrate(snap, oracle, rng, 0.01)
    cur = pool[:, :n0].copy()
    full, delta = setup(kt, oracle, snap, cur, rng)
    P = snap.pending.n
    probe_rows = rng.integers(0, P, size=min(P, 19))
    probe_idx = rng.choice(snap.m, size=min(snap.m, 40), replace=False).astype(np.int32)
    probe = (probe_rows, probe_idx, snap.pending.labels[:, probe_rows], snap.pending.ns_id[probe_rows])
    assert_tables(kt, delta, snap, f"{name} start")
    for step, (n_new, moves) in enumerate(steps):
        n = cur.shape[1]
        nxt = np.full((LN, n_new), abi.LABEL_EMPTY, np.int64)
        nxt[:, :n] = cur
        if moves:
            listed = np.array([ns for ns, _, _ in moves])
            for ns, g, _ in moves:
                nxt[3, ns] = synth._lab(GROUP, g)
        else:  # new namespaces take their own rows (some stay label-less), a few old ones random rows
            grown = np.arange(n, n_new)
            listed = np.union1d(grown[rng.random(grown.size) < 0.7], rng.choice(n, size=min(n, 3), replace=False))
            vals = np.where(listed < n, 0, 1)
            nxt[:, listed] = np.where(vals[None, :] == 1, pool[:, np.minimum(listed, pool.shape[1] - 1)], new_rows(rng, pool[:, :n], listed.size))
        cur = nxt
        snap.ns_labels = np.ascontiguousarray(cur)
        full.upload_namespaces(snap.ns_labels)
        if n_new - n > 65535:  # the whole growth in one call
            delta.update_namespace_rows(n_new, listed.astype(np.int32), cur[:, listed])
        else:
            for b in batches(rng, listed):
                delta.update_namespace_rows(n_new, b.astype(np.int32), cur[:, b])
            if not listed.size and n_new > n:
                delta.update_namespace_rows(n_new, np.zeros(0, np.int32), np.zeros((LN, 0), np.int64))
        where = f"{name} step {step} n_ns {n_new} moves {moves}"
        got_tables = delta.ns_tables()
        assert_tables(kt, delta, snap, where)
        for ns, _, c in moves:
            assert got_tables["nsw_off"][ns + 1] - got_tables["nsw_off"][ns] == c, where
        if ((snap.kind != abi.KIND_THROTTLE) | (snap.thr_ns < n_new)).all():
            assert_oracle(delta, snap, oracle, where)
        plan = PLANS[step % len(PLANS)]
        assert_same(observe(full, snap, plan, probe), observe(delta, snap, plan, probe), where + f" plan {plan}")
    full.close()
    delta.close()
