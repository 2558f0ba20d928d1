"""Small passes through every device path for compute-sanitizer (memcheck / racecheck / synccheck), checked against nothing:
the tool is the check.
  compute-sanitizer --tool racecheck python tools/sanitize_target.py
Paths: fused pass (persistent grid; shared second phase) and chained kernels (per-kernel timing), fast family (L <= 8) with 128- and
256-row tiles (a ClusterThrottle-heavy table has long per-namespace word lists), general family (L = 12, 6-bit counters), ragged
R = 1; wide / compact / packed uploads (packed: the fused unpack + translate kernel), row deltas, the one-call step with the
sparse check result, observed status + the device-side status diff + row getters, GIVEN_STATUS passes, queue admission rounds.
KT_SANITIZE_BIG=1 adds two 120k-row snapshots with more tiles than the device holds CTAs at once, so that CTAs run several tiles
one after the other in the same shared memory: 4k pending pods (four-lane decide sub-tiles) and 40k (more sub-tiles than two
rounds of the grid: lane-per-pod decide tiles after reconcile tiles).
Forced plans (kt_debug_set_pass_plan) then run every k_pass build (512 and 768 threads per SM) under both decide modes on the
grid the device holds and on one of a single CTA, for small shapes of 128- and 256-row tiles, the general family and two plane
pairs per table entry.  KT_SANITIZE_PLANS=1 runs only those."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import kube_throttler_b200 as kt
from kube_throttler_b200 import abi, synth

plan_cases = [("C2", dict(m=40, n=70, p=33, R=1)), ("C3", dict(m=600, n=1500, p=300, terms=2)), ("C2", dict(m=200, n=600, p=300, q_max=6, terms=3))]
for cfg, kw in plan_cases:
    snap = synth.generate(cfg, **kw)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    eng.set_sparse_check(4 * snap.pending.n + 64)
    for threads in (512, 768):
        for decide in (abi.PLAN_DECIDE_QUAD, abi.PLAN_DECIDE_PER_POD):
            for cap in (0, 1):
                eng.set_pass_plan(threads, decide, cap)
                eng.evaluate(snap.now)
                eng.sync()
    plan = eng.pass_plan()
    eng.close()
    print(cfg, kw, "ok: forced plans, tile", plan.tile, "tpc", plan.tpc, "b", plan.b, "rt", plan.rt, flush=True)
if os.environ.get("KT_SANITIZE_PLANS"):
    print("sanitize target done")
    sys.exit(0)

cases = [("C3", dict(m=300, n=3000, p=500)), ("C3", dict(m=900, n=2500, p=400)), ("C2", dict(m=200, n=2000, p=300, L=12, q_max=6)),
         ("C2", dict(m=40, n=70, p=33, R=1))]
if os.environ.get("KT_SANITIZE_SMALL"):  # a quick look at the fused pass only (128- and 256-row tiles)
    cases = [cases[0], cases[3]]
if os.environ.get("KT_SANITIZE_BIG"):
    cases += [("C2", dict(m=500, n=120_000, p=4000)), ("C2", dict(m=500, n=120_000, p=40_000))]
for cfg, kw in cases:
    snap = synth.generate(cfg, **kw)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    eng.upload_pods_compact(abi.PODS_PENDING, abi.compact_pods(snap.pending))
    for timing in (False, True):
        eng.enable_timing(timing)
        eng.evaluate(snap.now)
        eng.sync()
    fresh = eng.download()
    eng.enable_timing(False)
    # packed uploads + the one-call step with the sparse check result
    try:
        packed = tuple(abi.packed_pods(p, code_requests=True) for p in (snap.running, snap.pending))
    except ValueError:
        try:
            packed = tuple(abi.packed_pods(p) for p in (snap.running, snap.pending))
        except ValueError:
            packed = None
    if packed:
        eng.set_sparse_check(4 * snap.pending.n + 64)
        for _ in range(2):
            eng.step_submit(packed[0], packed[1], snap.now)
            res = eng.step_wait()
        assert int(res.n_pending) == snap.pending.n
        eng.set_sparse_check(0)
    # row deltas: a few running rows rewritten in place (with their own values)
    k = min(17, snap.running.n)
    rows = np.sort(np.random.default_rng(1).choice(snap.running.n, size=k, replace=False)).astype(np.int64)
    eng.update_pod_rows(abi.PODS_RUNNING, rows, snap.running.rows(rows))
    eng.evaluate(snap.now)
    eng.sync()
    # observed status: device-side diff, changed rows, GIVEN_STATUS check, queue admission
    m = snap.m
    snap.status = dict(calculated=np.ones(m, np.uint8), calc_thr=fresh.calc_thr.copy(), calc_present=fresh.calc_present.copy(), calc_cnt=fresh.calc_cnt.copy(),
                       used=fresh.used.copy(), used_present=fresh.used_present.copy(), used_cnt=fresh.used_cnt.copy(), throttled=fresh.throttled.copy())
    snap.status["used_cnt"][: m // 3] += 1  # a third of the throttles differ from what the pass computes
    snap.normalize()
    eng.upload_status(snap)
    eng.evaluate(snap.now)
    idx, _ = eng.get_changed()
    if idx.size:
        eng.get_reconcile_rows(idx)
    eng.get_check_rows(np.arange(min(5, snap.pending.n), dtype=np.int64))
    eng.evaluate(snap.now, abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE)
    eng.sync()
    rounds, admitted = eng.admit_queue(0, min(snap.pending.n, 300))
    eng.download()
    eng.close()
    print(cfg, kw, "ok: changed", idx.size, "admission rounds", rounds, "admitted", admitted, flush=True)
print("sanitize target done")
