"""Row order: the engine may store a pod table's rows sorted by namespace (kt_debug_set_row_order / kt_debug_get_row_order,
include/kt_b200.h "row order of the pod tables").  Every row number that crosses the ABI stays the caller's and no result
changes, so an engine forced to lay its rows out by namespace must deliver exactly what an engine forced to keep them as given
delivers, getter by getter, and the layout itself must be the stable argsort of the namespace keys."""
import os
import subprocess
import sys

import numpy as np
import pytest

from kube_throttler_b200 import abi, synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUN, PEND = abi.PODS_RUNNING, abi.PODS_PENDING
GIVEN, BY_NS, AUTO = abi.ROW_ORDER_AS_GIVEN, abi.ROW_ORDER_BY_NAMESPACE, abi.ROW_ORDER_AUTO
REC_ONLY = abi.EVAL_FRESH_STATUS | abi.EVAL_SKIP_CHECK
CHK_ONLY = abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE


def layout_key(ns, n_ns):
    ns = np.asarray(ns, np.int64)
    return np.where((ns >= 0) & (ns < n_ns), ns, n_ns)


def expected_dev_row(ns, n_ns):
    """dev_row[caller row] of the stable sort by namespace key"""
    order = np.argsort(layout_key(ns, n_ns), kind="stable")
    dev = np.empty(order.shape[0], np.int64)
    dev[order] = np.arange(order.shape[0])
    return dev


def bare_rows(ns, flags=None):
    n = len(ns)
    return abi.PodCols(np.full((1, n), abi.LABEL_EMPTY, np.int64), np.zeros((1, n), np.int64), np.zeros(n, np.uint32),
                       np.full(n, 5, np.uint32) if flags is None else np.asarray(flags, np.uint32), np.asarray(ns, np.int32))


def view(ptr, dtype, shape):
    import ctypes as C

    n = int(np.prod(shape))
    if n == 0:
        return np.zeros(shape, dtype)
    buf = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype, count=n).reshape(shape).copy()


def upload(eng, kind, pods, fmt):
    if fmt == "wide":
        eng.upload_pods(kind, pods)
    elif fmt == "compact":
        eng.upload_pods_compact(kind, abi.compact_pods(pods))
    else:
        eng.upload_pods_packed(kind, abi.packed_pods(pods, code_requests=fmt == "packed-coded"))


def layout_engine(kt, n_ns):
    eng = kt.Engine(1, 1, 1)
    eng.upload_namespaces(np.full((1, n_ns), abi.LABEL_EMPTY, np.int64))
    return eng


# ---- 1. the layout --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,n_ns,negative", [(0, 10, False), (1, 10, False), (31, 5, True), (33, 5, True), (100_000, 50, True),
                                             (5000, 1, False), (20_000, 300, False), (20_000, 70_000, False), (3000, 200, True)])
@pytest.mark.parametrize("fmt", ["wide", "compact", "packed", "packed-coded"])
def test_layout_is_the_stable_argsort_of_the_namespace_keys(kt, n, n_ns, negative, fmt):
    """Forced by namespace, every upload format lays its rows out as np.argsort(key, kind="stable"), where rows outside
    [0, n_ns) form one group at the end; several radix digits when n_ns passes 256 and 65536."""
    if negative and fmt != "wide":
        pytest.skip("only the wide format carries negative namespace ids")
    rng = np.random.default_rng(n + n_ns)
    ns = rng.integers(-3 if negative else 0, n_ns + 4, size=n)  # some ids past n_ns (and below 0): the trailing group
    eng = layout_engine(kt, n_ns)
    for kind in (RUN, PEND):
        eng.set_row_order(kind, BY_NS)
        upload(eng, kind, bare_rows(ns), fmt)
        clustered, dev = eng.row_order(kind)
        assert clustered == (n > 0)
        np.testing.assert_array_equal(dev, expected_dev_row(ns, n_ns))
    eng.close()


def test_automatic_rule_flips_at_its_threshold(kt):
    """More than one sampled group in four mixed: by namespace.  4096 rows = 128 groups of 32; the sample takes every second
    group (64 of them).  16 mixed sampled groups stay as given, 17 are clustered; mixing unsampled groups changes nothing."""
    n = 4096
    eng = layout_engine(kt, 100)
    for fmt in ("wide", "compact", "packed"):
        for mixed, want in ((16, False), (17, True)):
            ns = np.repeat(np.arange(128) % 100, 32)   # one namespace per group
            for g in range(mixed):
                ns[(2 * g) * 32 + 7] = 99 - ns[(2 * g) * 32]  # a second namespace in sampled group 2g
            for g in range(40):
                ns[(2 * g + 1) * 32 + 3] = 98 - ns[(2 * g + 1) * 32]  # unsampled groups do not count
            upload(eng, RUN, bare_rows(ns), fmt)
            clustered, dev = eng.row_order(RUN)
            assert clustered == want, (fmt, mixed)
            np.testing.assert_array_equal(dev, expected_dev_row(ns, 100) if want else np.arange(n))
    eng.close()


def test_clustered_inputs_stay_as_given(kt):
    """Rows sorted by namespace (the synth generator's, bench.py's C2 headline) and arena-shaped rows (chunks of 32 rows per
    namespace, interleaved, with tombstones of any namespace inside the chunks) keep identity maps; arrival order is clustered."""
    for cfg in ("C2", "C3"):
        snap = synth.generate(cfg)
        eng = kt.Engine(snap.R, snap.L, snap.LN)
        eng.upload_namespaces(snap.ns_labels)
        upload(eng, RUN, snap.running, "packed")
        upload(eng, PEND, snap.pending, "wide")
        assert not eng.row_order(RUN)[0] and not eng.row_order(PEND)[0], cfg
        arr = synth.generate(cfg, sort_by_namespace=False)
        upload(eng, RUN, arr.running, "packed")
        upload(eng, PEND, arr.pending, "wide")
        assert eng.row_order(RUN)[0] and eng.row_order(PEND)[0], cfg
        eng.close()
    eng = layout_engine(kt, 64)
    rng = np.random.default_rng(5)
    chunks = rng.integers(0, 64, size=400)             # chunk c belongs to namespace chunks[c]
    ns = np.repeat(chunks, 32)
    flags = np.full(ns.shape[0], 5, np.uint32)
    dead = rng.random(ns.shape[0]) < 0.3                # tombstones: flags 0, any namespace
    flags[dead] = 0
    ns[dead] = rng.integers(0, 64, size=int(dead.sum()))
    for fmt in ("wide", "compact", "packed"):
        upload(eng, PEND, bare_rows(ns, flags), fmt)
        clustered, dev = eng.row_order(PEND)
        assert not clustered
        np.testing.assert_array_equal(dev, np.arange(ns.shape[0]))
    eng.close()


# ---- 2. parity: every getter, laid out by namespace or as given -------------------------------------------------------------
def engine(kt, snap, mode, sparse=True):
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    for kind in (RUN, PEND):
        eng.set_row_order(kind, mode)
    eng.upload_snapshot(snap)
    if sparse:
        eng.set_sparse_check(4 * snap.pending.n + 64)
    for kind in (RUN, PEND):
        assert eng.row_order(kind)[0] == (mode == BY_NS and eng.n[kind] > 0)
    return eng


FIELDS = ("run_bitmap", "pend_bitmap", "codes", "admit", "used", "used_present", "used_cnt", "throttled", "calc_thr", "calc_present",
          "calc_cnt", "override_active")


def assert_results_equal(a, b, what=""):
    for f in FIELDS:
        np.testing.assert_array_equal(getattr(a, f), getattr(b, f), err_msg=f"{what} {f}")


def getters(eng, snap, rng_seed):
    """Everything the engine answers after a pass, in caller rows."""
    rng = np.random.default_rng(rng_seed)
    out = {"pass": eng.download()}
    out["changed"] = eng.get_changed()
    ent = np.zeros((4 * snap.pending.n + 64, 3), np.uint32)
    admit = np.zeros(snap.pending.n, np.uint8)
    cnt = eng.get_check_sparse(admit, ent)
    out["sparse"] = (cnt, sorted(map(tuple, ent[:cnt].tolist())), admit)
    for kind, pods in ((RUN, snap.running), (PEND, snap.pending)):
        rows = rng.integers(0, pods.n, size=min(pods.n, 97))
        out[f"match_rows{kind}"] = eng.match_rows(kind, rows)
        idx = rng.integers(0, snap.m, size=min(snap.m, 40))
        out[f"match_columns{kind}"] = eng.match_columns(kind, idx)
    out["check_rows"] = eng.get_check_rows(rng.integers(0, snap.pending.n, size=min(snap.pending.n, 97)))
    idx = rng.integers(0, snap.m, size=min(snap.m, 40))
    rt, off, rows = eng.reconcile_throttles(snap.now, idx)
    out["reconcile_throttles"] = tuple(getattr(rt, f) for f in ("used", "used_present", "used_cnt", "throttled", "calc_thr")) + (off, rows)
    return out


def assert_getters_equal(a, b):
    assert_results_equal(a["pass"], b["pass"])
    for k in a:
        if k == "pass":
            continue
        for x, y in zip(a[k], b[k]):
            if x is None:
                assert y is None
            elif isinstance(x, list):
                assert x == y, k
            else:
                np.testing.assert_array_equal(x, y, err_msg=k)


PARITY = [dict(config="C1", n=700, p=300, R=1, L=3), dict(config="C2", m=333, n=7777, p=1111, R=4, L=8),
          dict(config="C3", m=400, n=9000, p=1500, R=8, L=12), dict(config="C4", m=900, n=8000, p=1200, R=12, L=3),
          dict(config="C2", m=200, n=5000, p=700, R=1, L=12), dict(config="C3", m=300, n=6000, p=900, R=12, L=8)]


@pytest.mark.parametrize("world", PARITY, ids=lambda w: "{config}-R{R}-L{L}".format(**w))
def test_every_getter_agrees_with_rows_as_given(kt, oracle, world):
    from test_oracle_admission import admission_world

    world = dict(world)
    snap = admission_world(oracle, world.pop("config"), sort_by_namespace=False, **world)
    engines = [engine(kt, snap, BY_NS), engine(kt, snap, GIVEN)]
    res = []
    for eng in engines:
        eng.evaluate(snap.now)
        res.append(getters(eng, snap, 1))
    assert_getters_equal(res[0], res[1])
    if world.get("R") == 4:  # one shape against the columnar oracle as well
        want = oracle.columnar_evaluate(snap, words_per_row=res[0]["pass"].words_per_row)
        for f in ("run_bitmap", "pend_bitmap", "codes", "admit", "calc_thr"):
            np.testing.assert_array_equal(getattr(res[0]["pass"], f), getattr(want, f), err_msg=f)
    # the step API on the same rows, packed: admit bits, the sparse entries (rows rewritten to caller rows) and the status
    packed = [abi.packed_pods(p_, code_requests=True) for p_ in (snap.running, snap.pending)]
    steps = []
    for eng in engines:
        eng.step_submit(packed[0], packed[1], snap.now)
        r = eng.step_wait()
        P, n_sp = r.n_pending, int(r.n_sparse)
        admit = view(r.admit, np.uint8, (P,))
        ent = view(r.entries, np.uint32, (n_sp, 3))
        used = view(r.status.used, np.int64, (snap.R, snap.m))
        steps.append((admit, sorted(map(tuple, ent.tolist())), used))
        assert eng.row_order(PEND)[0] == (eng is engines[0])
    np.testing.assert_array_equal(steps[0][0], steps[1][0])
    assert steps[0][1] == steps[1][1]
    np.testing.assert_array_equal(steps[0][2], steps[1][2])
    np.testing.assert_array_equal(steps[0][0], res[1]["pass"].admit)
    for eng in engines:
        eng.close()


# ---- 3. every fused-pass build and the chained passes ----------------------------------------------------------------------
def test_pass_plans_and_chained_passes_on_clustered_rows(kt, oracle):
    from test_oracle_admission import admission_world

    snap = admission_world(oracle, "C3", m=300, n=6000, p=1000, sort_by_namespace=False)
    clus, given = engine(kt, snap, BY_NS, sparse=False), engine(kt, snap, GIVEN, sparse=False)
    plans = [(t, d, c) for t in (512, 768) for d in (abi.PLAN_DECIDE_QUAD, abi.PLAN_DECIDE_PER_POD) for c in (0, 3)]
    for eng in (clus, given):
        eng.evaluate(snap.now)
    ref = given.download()
    for t, d, c in plans:
        clus.set_pass_plan(t, d, c)
        clus.evaluate(snap.now)
        assert_results_equal(clus.download(), ref, f"plan {t}/{d}/{c}")
    clus.set_pass_plan()
    clus.enable_timing(True)  # the three chained kernels instead of the fused launch
    clus.evaluate(snap.now)
    assert_results_equal(clus.download(), ref, "chained")
    clus.enable_timing(False)
    for flags in (REC_ONLY, CHK_ONLY, CHK_ONLY | abi.EVAL_ON_EQUAL):
        for eng in (clus, given):
            eng.evaluate(snap.now, flags)
        a, b = clus.download(), given.download()
        assert_results_equal(a, b, f"flags {flags}")
    clus.close()
    given.close()


# ---- 4. row deltas ---------------------------------------------------------------------------------------------------------
def test_row_deltas_on_clustered_rows(kt, oracle):
    """Deltas leave the layout alone (a row that moves to another namespace stays in its slot) and every getter still equals
    the engine that keeps the rows as given, pass after pass."""
    from test_oracle_admission import admission_world

    snap = admission_world(oracle, "C2", m=300, n=6000, p=1200, sort_by_namespace=False)
    donor = synth.generate("C2", m=300, n=6000, p=1200, seed=99, sort_by_namespace=False)
    clus, given = engine(kt, snap, BY_NS), engine(kt, snap, GIVEN)
    before = {kind: clus.row_order(kind)[1] for kind in (RUN, PEND)}
    rng = np.random.default_rng(17)
    for step in range(6):
        for kind, src in ((RUN, donor.running), (PEND, donor.pending)):
            n = snap.running.n if kind == RUN else snap.pending.n
            rows = rng.choice(n, size=int(rng.integers(1, 200)), replace=False).astype(np.int64)
            new = src.rows(rng.integers(0, src.n, size=rows.shape[0]))  # other pods: other namespaces, labels, requests
            gone = rng.random(rows.shape[0]) < 0.25                     # deleted pods: flags 0, no labels
            new.flags[gone] = 0
            new.labels[:, gone] = abi.LABEL_EMPTY
            for eng in (clus, given):
                eng.update_pod_rows(kind, rows, new)
        for eng in (clus, given):
            eng.evaluate(snap.now)
        assert_getters_equal(getters(clus, snap, step), getters(given, snap, step))
    for kind in (RUN, PEND):
        clustered, dev = clus.row_order(kind)
        assert clustered
        np.testing.assert_array_equal(dev, before[kind])
    clus.close()
    given.close()


# ---- 5. queue admission ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("first,count,flags", [(0, None, 0), (0, 1, 0), (41, 1025, 0), (300, 700, abi.EVAL_ON_EQUAL), (0, None, abi.EVAL_ON_EQUAL)])
def test_queue_admission_on_clustered_rows(kt, oracle, first, count, flags):
    """kt_admit_queue on pending rows laid out by namespace admits the queue in caller order, one pod per cycle: the same
    admit bits, codes, rounds and count as the engine with the rows as given and as the oracle's walk."""
    from test_oracle_admission import admission_world

    snap = admission_world(oracle, "C2", m=200, n=4000, p=2600, sort_by_namespace=False)
    count = snap.pending.n - first if count is None else count
    out = []
    for mode in (BY_NS, GIVEN):
        eng = engine(kt, snap, mode, sparse=False)
        rounds, admitted = eng.admit_queue(first, count, flags)
        out.append((rounds, admitted, eng.download()))
        eng.close()
    assert out[0][:2] == out[1][:2]
    assert_results_equal(out[0][2], out[1][2])
    want, n_adm, _ = oracle.columnar_admit_queue(snap, first, count, flags, words_per_row=out[0][2].words_per_row)
    np.testing.assert_array_equal(out[0][2].admit, want.admit)
    np.testing.assert_array_equal(out[0][2].codes, want.codes)
    assert out[0][1] == n_adm


# ---- 6. state and arguments ------------------------------------------------------------------------------------------------
def test_relayout_voids_results_and_bad_arguments_are_refused(kt):
    snap = synth.generate("C2", m=100, n=3000, p=500, sort_by_namespace=False)
    eng = engine(kt, snap, BY_NS)
    eng.evaluate(snap.now)
    eng.download()
    eng.upload_pods(PEND, snap.pending)  # a fresh layout: results wait for the next pass
    with pytest.raises(kt.KtError) as e:
        eng.get_check(np.zeros((snap.pending.n, 2 * eng.words_per_row), np.uint32), None)
    assert e.value.code == abi.ERR_STATE
    with pytest.raises(kt.KtError) as e:
        eng.match_rows(RUN, np.arange(3))
    assert e.value.code == abi.ERR_STATE
    for kind, mode in ((2, AUTO), (-1, GIVEN), (RUN, 3), (PEND, -1)):
        with pytest.raises(kt.KtError) as e:
            eng.set_row_order(kind, mode)
        assert e.value.code == abi.ERR_INVALID
    with pytest.raises(kt.KtError) as e:
        eng.row_order(2)
    assert e.value.code == abi.ERR_INVALID
    eng.evaluate(snap.now)
    eng.download()
    eng.close()


# ---- 7. two GPUs -----------------------------------------------------------------------------------------------------------
def test_two_gpu_sharded_clustered_world():
    """Each rank lays its own shard out by namespace; the stacked results equal the oracle's evaluation of the whole world."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29517", os.path.join("tools", "multi_gpu_parity.py"), "C3", "1000", "20011", "2003", "arrival"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "OK" in r.stdout
