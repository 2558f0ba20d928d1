"""Randomised object-level parity: the PRODUCT plugin (kt_host.h above the CUDA engine) against the object-level
ORACLE on the same Kubernetes manifests -- quantities as strings (m, Mi, Gi, decimals), matchLabels and
matchExpressions, both throttle kinds, namespace selectors, overrides, reservations, pod updates.

Every status field and every PreFilter result must be identical (quantities compared by value)."""
import random
from fractions import Fraction

import pytest

from test_oracle_kat import q
from test_scenarios import NOW, SCHED, THROTTLER, namespace



@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def new_plugin(request):
    """NewPlugin on the product (GPU), or on the product's host layer over the engine test double that evaluates with the
    columnar oracle (CPU; conftest.host_on_oracle): the latter checks kt_host.cc against the OBJECT-level oracle -- packing,
    scales, status bookkeeping, reservations, reasons -- and says nothing about the kernels."""
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin

KEYS = ["app", "tier", "team", "env", "zone"]
VALS = ["a", "b", "c", "d"]
CPUS = ["50m", "100m", "250m", "0.5", "1", "1500m", "2", "0"]
MEMS = ["64Mi", "128Mi", "512Mi", "1Gi", "1.5Gi", "1000000", "0"]


def rand_labels(rng, lo=0, hi=4):
    return {k: rng.choice(VALS) for k in rng.sample(KEYS, rng.randint(lo, hi))}


def rand_selector(rng):
    sel = {}
    if rng.random() < 0.85:
        sel["matchLabels"] = rand_labels(rng, 0 if rng.random() < 0.1 else 1, 3)
    exprs = []
    for _ in range(rng.choice([0, 0, 1, 2])):
        op = rng.choice(["In", "NotIn", "Exists", "DoesNotExist"])
        e = {"key": rng.choice(KEYS), "operator": op}
        if op in ("In", "NotIn"):
            e["values"] = rng.sample(VALS, rng.randint(1, 3))
        exprs.append(e)
    if exprs:
        sel["matchExpressions"] = exprs
    return sel


def rand_amount(rng, scale=1):
    a = {}
    if rng.random() < 0.5:
        a["resourceCounts"] = {"pod": (0 if rng.random() < 0.05 else rng.choice([3, 20, 60, 200])) * scale}
    rr = {}
    if rng.random() < 0.8:
        rr["cpu"] = rng.choice(["200m", "2500m", "10", "30.5", "80", "400"] if rng.random() < 0.8 else ["0", "1n"])
    if rng.random() < 0.5:
        rr["memory"] = rng.choice(["256Mi", "4Gi", "30000000000", "64Gi", "1Ti"])
    if rng.random() < 0.2:
        rr["nvidia.com/gpu"] = str(rng.choice([0, 4, 40]))
    if rr or rng.random() < 0.5:
        a["resourceRequests"] = rr
    return a


def rand_pod(rng, ns, name, running):
    reqs = {}
    if rng.random() < 0.9:
        reqs["cpu"] = rng.choice(CPUS)
    if rng.random() < 0.6:
        reqs["memory"] = rng.choice(MEMS)
    if rng.random() < 0.15:
        reqs["nvidia.com/gpu"] = str(rng.randint(0, 2))
    spec = {"schedulerName": SCHED if rng.random() < 0.92 else "other", "nodeName": "", "containers": [{"name": "c", "resources": {"requests": reqs}}]}
    if rng.random() < 0.2:
        spec["containers"].append({"name": "c2", "resources": {"requests": {"cpu": rng.choice(CPUS)}}})
    if rng.random() < 0.15:
        spec["initContainers"] = [{"name": "i", "resources": {"requests": {"cpu": rng.choice(CPUS), "memory": rng.choice(MEMS)}}}]
    if rng.random() < 0.1:
        spec["overhead"] = {"cpu": "10m"}
    phase = "Pending"
    if running:
        spec["nodeName"] = "node-1" if rng.random() < 0.95 else ""
        phase = rng.choice(["Running", "Running", "Running", "Succeeded", "Failed", "Pending"])
    return {"kind": "Pod", "metadata": {"namespace": ns, "name": name, "labels": rand_labels(rng)}, "spec": spec, "status": {"phase": phase}}


def rand_throttle(rng, i, nss):
    kind = "ClusterThrottle" if rng.random() < 0.4 else "Throttle"
    terms = []
    for _ in range(rng.choice([0, 1, 1, 1, 2])):
        t = {"podSelector": rand_selector(rng)}
        if kind == "ClusterThrottle":
            t["namespaceSelector"] = rng.choice([{}, {"matchLabels": {"team": rng.choice(VALS)}}, {"matchExpressions": [{"key": "env", "operator": "NotIn", "values": ["a"]}]}])
        terms.append(t)
    spec = {"throttlerName": THROTTLER if rng.random() < 0.93 else "foreign", "threshold": rand_amount(rng), "selector": {"selectorTerms": terms}}
    if rng.random() < 0.3:
        spec["temporaryThresholdOverrides"] = [
            {"begin": rng.choice(["", "2025-12-01T00:00:00Z", "2026-06-01T00:00:00Z", "garbage"]),
             "end": rng.choice(["", "2026-02-01T00:00:00+09:00", "2025-12-15T00:00:00Z"]), "threshold": rand_amount(rng, 2)}
            for _ in range(rng.randint(1, 3))]
    md = {"name": f"t{i}"}
    if kind == "Throttle":
        md["namespace"] = rng.choice(nss)
    return {"kind": kind, "metadata": md, "spec": spec}


def norm_amount(a):
    return (a.get("resourceCounts"), {k: q(v) for k, v in a.get("resourceRequests", {}).items()} if "resourceRequests" in a else None)


def norm_status(s):
    ct = s["calculatedThreshold"]
    return dict(thr=norm_amount(ct["threshold"]), at=(ct["calculatedAtSet"], ct["calculatedAtUnix"] if ct["calculatedAtSet"] else None), msgs=ct.get("messages"),
                throttled=s["throttled"], used=norm_amount(s["used"]))


def norm_prefilter(r):
    # (an Error status carries its message and nothing else, plugin.go:154-156 / :166-168; the oracle's debug breakdown beside it is not compared)
    return {k: r.get(k) for k in (("code", "reasons") if r.get("code") == "Error" else ("code", "reasons", "event", "throttle", "clusterthrottle"))}


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_random_world(oracle, new_plugin, seed):

    rng = random.Random(seed)
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    nss = [f"ns{i}" for i in range(5)]
    for n in nss:
        both(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
    throttles = [rand_throttle(rng, i, nss) for i in range(40)]
    both(*throttles)
    pods = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(300)]
    both(*pods)

    def compare_status():
        for t in throttles:
            ns = t["metadata"].get("namespace", "")
            a, b = ref.status(t["metadata"]["name"], ns), dut.status(t["metadata"]["name"], ns)
            assert norm_status(a) == norm_status(b), (t, a, b)

    def compare_prefilter(pending):
        want = [norm_prefilter(ref.prefilter(p)) for p in pending]
        got = [norm_prefilter(r) for r in dut.prefilter_batch(pending)]  # the whole queue in ONE device pass
        assert got == want
        assert norm_prefilter(dut.prefilter(pending[0])) == want[0]    # and the per-pod entry point agrees
        return want

    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    compare_status()
    pending = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(120)]
    res = compare_prefilter(pending)
    assert len({x.split("=")[0] for r in res for x in r["reasons"]} | {r["code"] for r in res}) >= 3  # the scenario is not degenerate

    # admit a few: Reserve on both, bind half of them, leave the rest reserved-only; then update labels of some running pods
    admitted = [p for p, r in zip(pending, res) if r["code"] == "Success"][:20]
    for i, p in enumerate(admitted):
        assert ref.reserve(p)["code"] == dut.reserve(p)["code"] == "Success"
        if i % 2 == 0:
            both(dict(p, spec=dict(p["spec"], nodeName="node-2"), status={"phase": "Running"}))
    for p in rng.sample(pods, 25):
        p["metadata"]["labels"] = rand_labels(rng)
        both(p)
    compare_prefilter(pending[20:80])  # stale status + reservations in play
    for t in throttles:
        k, nn = t["kind"], t["metadata"].get("namespace", "") + "/" + t["metadata"]["name"]
        a, b = ref.reserved(k, nn), dut.reserved(k, nn)
        assert sorted(a["pods"]) == sorted(b["pods"]) and norm_amount(a["amount"]) == norm_amount(b["amount"]), (nn, a, b)
    later = "2026-03-01T12:00:00Z"  # the override windows have moved on
    ref.reconcile_all(later), dut.reconcile_all(later)
    compare_status()
    compare_prefilter(pending[60:])
    # a threshold edit is invisible to PreFilter until the next reconcile (Q6)
    throttles[0]["spec"]["threshold"] = {"resourceCounts": {"pod": 0}}
    both(throttles[0])
    compare_prefilter(pending[:40])
    ref.reconcile_all(later), dut.reconcile_all(later)
    compare_status()
    compare_prefilter(pending[:40])
    dut.close()


@pytest.mark.parametrize("seed", [5, 6, 7])
def test_resident_queue_by_key(oracle, new_plugin, seed):
    """Pods the informer delivered that are waiting to be scheduled live in the device's pending table; PreFilter / Reserve /
    Unreserve address them BY KEY (kth_pre_filter_key, ...) and must say exactly what the manifest calls -- and the oracle's
    per-pod PreFilter -- say, through every kind of event that can change a verdict: reservations, reconciles, relabelled pods,
    throttle edits, pods leaving the queue.  Verdicts are served from the cached queue pass whenever nothing a pod depends on
    changed (the stats say so)."""
    rng = random.Random(seed)
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    nss = [f"ns{i}" for i in range(4)]
    both(*[namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}) for n in nss])
    throttles = [rand_throttle(rng, i, nss) for i in range(30)]
    both(*throttles)
    both(*[rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(200)])
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(90)]
    both(*queue)  # the informer delivers the pending pods: they are resident from here on
    key = lambda p: (p["metadata"]["namespace"], p["metadata"]["name"])

    def compare(pods):
        for p in pods:
            want = norm_prefilter(ref.prefilter(p))
            assert norm_prefilter(dut.prefilter_key(*key(p))) == want, key(p)
            assert norm_prefilter(dut.prefilter(p)) == want  # the manifest entry point, same pod
        return [ref.prefilter(p)["code"] for p in pods]

    codes = compare(queue)
    verdicts = dut.prefilter_queue()
    names = {"Success": 1, "UnschedulableAndUnresolvable": 2, "Error": 3}
    queued = 0
    for p, c in zip(queue, codes):
        row = dut.queue_row(*key(p))
        if row < 0:  # another scheduler's pod: known to the informer, not in OUR queue (by-key calls check it like a manifest)
            assert p["spec"]["schedulerName"] != SCHED
            continue
        queued += 1
        assert verdicts[row] == names[c], key(p)
    assert queued > len(queue) // 2 and (verdicts != 0).sum() >= queued  # (+ the "running" pods of the world that have no node yet)
    before = dut.queue_stats()
    compare(queue[:30])  # nothing changed: no further device pass over the queue for the by-key calls
    after = dut.queue_stats()
    assert after["hits"] >= before["hits"] + 28 and after["passes"] <= before["passes"] + 1  # (the first manifest call may grow the scratch rows)

    # the scheduler's cycle: PreFilter -> Reserve by key, in queue order; every Reserve must be visible to the next PreFilter
    admitted = []
    for p in queue[:40]:
        a, b = ref.prefilter(p), dut.prefilter_key(*key(p))
        assert norm_prefilter(a) == norm_prefilter(b), key(p)
        if a["code"] == "Success":
            assert ref.reserve(p)["code"] == dut.reserve_key(*key(p))["code"] == "Success"
            admitted.append(p)
    assert admitted
    for t in throttles:
        k, nn = t["kind"], t["metadata"].get("namespace", "") + "/" + t["metadata"]["name"]
        a, b = ref.reserved(k, nn), dut.reserved(k, nn)
        assert sorted(a["pods"]) == sorted(b["pods"]) and norm_amount(a["amount"]) == norm_amount(b["amount"]), (nn, a, b)
    compare(queue)
    # bind half of the admitted pods (they leave the queue), un-reserve one, relabel some queued pods, edit a throttle, reconcile
    for i, p in enumerate(admitted):
        if i % 2 == 0:
            both(dict(p, spec=dict(p["spec"], nodeName="node-1"), status={"phase": "Running"}))
            assert dut.queue_row(*key(p)) == -1  # bound: it left the queue
    ref.unreserve(admitted[1]), dut.unreserve_key(*key(admitted[1]))
    still = [p for i, p in enumerate(queue) if not (p in admitted and admitted.index(p) % 2 == 0)]
    for p in rng.sample(still, 12):
        p["metadata"]["labels"] = rand_labels(rng)
        both(p)
    compare(still)
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    compare(still)
    throttles[3]["spec"]["threshold"] = {"resourceCounts": {"pod": 0}}
    both(throttles[3])
    compare(still[:30])
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    compare(still)
    gone = still[5]
    ref.delete("Pod", gone["metadata"]["name"], gone["metadata"]["namespace"]), dut.delete("Pod", gone["metadata"]["name"], gone["metadata"]["namespace"])
    with pytest.raises(RuntimeError, match="not in the informer cache"):
        dut.prefilter_key(*key(gone))
    newcomers = [rand_pod(rng, rng.choice(nss), f"n{i}", False) for i in range(80)]  # the queue outgrows its first capacity
    both(*newcomers)
    compare(newcomers + still[6:20])
    dut.close()


@pytest.mark.parametrize("seed", [11, 18, 19])
def test_admit_queue_equals_one_pod_per_cycle(oracle, new_plugin, seed):
    """kth_admit_queue == the scheduler's cycle (PreFilter, on Success Reserve) run pod by pod on the oracle: same verdict for
    every pod of the queue, same reservations afterwards -- in far fewer device passes than pods."""

    rng = random.Random(seed)
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    nss = [f"ns{i}" for i in range(5)]
    for n in nss:
        both(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
    throttles = [rand_throttle(rng, i, nss) for i in range(40)]
    for t in throttles:  # roomy thresholds: the queue has to fill them up pod by pod
        thr = t["spec"]["threshold"]
        if "resourceCounts" in thr:
            thr["resourceCounts"]["pod"] = rng.choice([2, 5, 9, 40])
        if "cpu" in thr.get("resourceRequests", {}):
            thr["resourceRequests"]["cpu"] = rng.choice(["1", "2500m", "7", "30"])
        t["spec"].pop("temporaryThresholdOverrides", None)
    both(*throttles)
    both(*[rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(40)])
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(150)]
    want = []
    for p in queue:  # one pod per scheduling cycle
        r = ref.prefilter(p)
        if r["code"] == "Success":
            assert ref.reserve(p)["code"] == "Success"
        want.append(norm_prefilter(r))
    got = dut.admit_queue(queue)
    assert [norm_prefilter(x["preFilter"]) for x in got["results"]] == want
    assert got["admitted"] == sum(w["code"] == "Success" for w in want) > 5
    assert 1 < got["rounds"] < len(queue) / 2, got["rounds"]  # conflicts force several passes, far fewer than pods
    for t in throttles:
        k, nn = t["kind"], t["metadata"].get("namespace", "") + "/" + t["metadata"]["name"]
        a, b = ref.reserved(k, nn), dut.reserved(k, nn)
        assert sorted(a["pods"]) == sorted(b["pods"]) and norm_amount(a["amount"]) == norm_amount(b["amount"]), (nn, a, b)
    dut.close()


def test_admit_queue_with_pods_that_already_hold_a_reservation(oracle, new_plugin):
    """Reserve is idempotent per pod (podResourceAmountMap.add overwrites, reserved_resource_amounts.go:131-136): a pod that was
    reserved in an earlier cycle and comes through the queue again -- or stands in it twice -- adds nothing when it is admitted
    again.  (Found by the event-stream chaos test, seed 171: the device's prefix sums counted such a pod a second time and
    rejected the pod behind it.)"""
    from test_scenarios import pod

    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    both(namespace("ns0", {"team": "a"}))
    both({"kind": "ClusterThrottle", "metadata": {"name": "ct"},
          "spec": {"throttlerName": THROTTLER, "threshold": {"resourceCounts": {"pod": 3}, "resourceRequests": {"cpu": "1"}},
                   "selector": {"selectorTerms": [{"podSelector": {}}]}}})
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    q = [pod("ns0", f"q{i}", "200m", {}, scheduler=SCHED) for i in range(5)]
    assert ref.prefilter(q[0])["code"] == dut.prefilter(q[0])["code"] == "Success"
    assert ref.reserve(q[0])["code"] == dut.reserve(q[0])["code"] == "Success"
    for queue in ([q[0], q[1], q[2], q[3]],          # q0 holds a reservation already: q1 and q2 still fit under pod <= 3
                  [q[3], q[3], q[4]]):               # the same pod twice
        want = []
        for p in queue:
            r = ref.prefilter(p)
            if r["code"] == "Success":
                assert ref.reserve(p)["code"] == "Success"
            want.append(norm_prefilter(r))
        got = dut.admit_queue(queue)
        assert [norm_prefilter(x["preFilter"]) for x in got["results"]] == want, (got, want)
        a, b = ref.reserved("ClusterThrottle", "/ct"), dut.reserved("ClusterThrottle", "/ct")
        assert sorted(a["pods"]) == sorted(b["pods"]) and norm_amount(a["amount"]) == norm_amount(b["amount"]), (a, b)
    assert sorted(dut.reserved("ClusterThrottle", "/ct")["pods"]) == ["ns0/q0", "ns0/q1", "ns0/q2"]
    dut.close()


@pytest.mark.parametrize("seed", [11, 19])
def test_admit_queue_with_negative_requests(oracle, new_plugin, seed):
    """Quantities are signed, and a negative request of an undecided pod LOWERS the load the pods behind it see: the device's
    fixpoint bounds that load with the undecided pods' negative parts from below and their positive parts from above.  Such a
    queue is admitted on the device (onDevice) with the verdicts and reservations of one pod per cycle.  The first queue is the
    smallest one the unsigned bounds got wrong: A (cpu -5, on t1 and on t2 with pod: 0) is rejected, so B (cpu 8) sees t1's
    5 + 8 > 10 -- under "Admitted + Undecided" it saw 5 - 5 + 8 and was admitted."""
    from test_scenarios import pod, throttle

    rng = random.Random(seed)
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    nss = [f"ns{i}" for i in range(3)]
    for n in nss:
        both(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
    throttles = [throttle("ns0", "t1", {"app": "x"}, cpu="10"), throttle("ns0", "t2", {"tier": "y"}, pod_cnt=0)]
    both(*throttles)
    both(pod("ns0", "r0", "5", {"app": "x"}, node="n1", phase="Running"))

    def more():  # after the two-pod queue: random throttles with roomy thresholds, as in test_admit_queue_equals_one_pod_per_cycle
        for i in range(30):
            t = rand_throttle(rng, i + 3, nss)
            thr = t["spec"]["threshold"]
            if "resourceCounts" in thr:
                thr["resourceCounts"]["pod"] = rng.choice([2, 5, 9, 40])
            if "cpu" in thr.get("resourceRequests", {}):
                thr["resourceRequests"]["cpu"] = rng.choice(["1", "2500m", "7", "30"])
            t["spec"].pop("temporaryThresholdOverrides", None)
            throttles.append(t)
            both(t)
        both(*[rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(30)])
        queue = []
        for i in range(120):
            p = rand_pod(rng, rng.choice(nss), f"q{i}", False)
            if rng.random() < 0.3:
                p["spec"]["containers"][0]["resources"]["requests"]["cpu"] = "-500m"
            queue.append(p)
        return queue

    verdicts = []
    for queue in ([pod("ns0", "a", "-5", {"app": "x", "tier": "y"}), pod("ns0", "b", "8", {"app": "x"})], None):
        queue = queue or more()
        ref.reconcile_all(NOW), dut.reconcile_all(NOW)
        want = []
        verdicts.append(want)
        for p in queue:  # one pod per scheduling cycle
            r = ref.prefilter(p)
            if r["code"] == "Success":
                assert ref.reserve(p)["code"] == "Success"
            want.append(norm_prefilter(r))
        got = dut.admit_queue(queue)
        assert got.get("onDevice") is True
        assert [norm_prefilter(x["preFilter"]) for x in got["results"]] == want
        assert got["admitted"] == sum(w["code"] == "Success" for w in want)
        for t in throttles:
            k, nn = t["kind"], t["metadata"].get("namespace", "") + "/" + t["metadata"]["name"]
            a, b = ref.reserved(k, nn), dut.reserved(k, nn)
            assert sorted(a["pods"]) == sorted(b["pods"]) and norm_amount(a["amount"]) == norm_amount(b["amount"]), (nn, a, b)
    assert [w["reasons"] for w in verdicts[0]] == [["throttle[pod-requests-exceeds-threshold]=ns0/t2"], ["throttle[insufficient]=ns0/t1"]]
    assert 5 < sum(w["code"] == "Success" for w in verdicts[1]) < len(queue) - 5
    dut.close()


def test_engine_limits_grow(oracle, new_plugin):
    """More label slots / resource columns / namespace labels than the engine was created with: the host layer re-creates
    the engine with larger limits and re-uploads its caches; decisions stay identical to the oracle's."""
    from test_scenarios import pod, throttle

    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    both(namespace("default"), throttle("default", "t", {"a": "1"}, pod_cnt=3, cpu="1"))
    both(pod("default", "p0", "300m", {"a": "1"}, node="n", phase="Running"))
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    assert norm_status(ref.status("t", "default")) == norm_status(dut.status("t", "default"))
    # 11 labels (> 8 slots), 6 resource names (> 4 columns), a namespace with 6 labels (> 4 slots)
    many = {f"k{i}": "v" for i in range(10)}
    many["a"] = "1"
    big = pod("default", "p1", "200m", many, node="n", phase="Running",
              requests={"memory": "1Gi", "nvidia.com/gpu": "1", "ephemeral-storage": "10Gi", "example.com/foo": "2", "hugepages-2Mi": "4Mi"})
    both(big, namespace("wide", {f"l{i}": "x" for i in range(5)}),
         {"kind": "ClusterThrottle", "metadata": {"name": "c"}, "spec": {"throttlerName": THROTTLER, "threshold": {"resourceRequests": {"example.com/foo": "3", "memory": "1536Mi"}},
                                                                       "selector": {"selectorTerms": [{"podSelector": {"matchLabels": {"k9": "v"}}, "namespaceSelector": {}}]}}})
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    for name, ns in (("t", "default"), ("c", "")):
        assert norm_status(ref.status(name, ns)) == norm_status(dut.status(name, ns))
    assert rl_values_of(dut.status("c")["used"]) == {"cpu": Fraction(1, 5), "memory": 2**30, "nvidia.com/gpu": 1, "ephemeral-storage": 10 * 2**30, "example.com/foo": 2, "hugepages-2Mi": 4 * 2**20}
    for p in (pod("default", "q0", "100m", many, requests={"example.com/foo": "2"}), pod("default", "q1", "600m", {"a": "1"}), pod("wide", "q2", "1", many, requests={"memory": "600Mi"})):
        assert norm_prefilter(ref.prefilter(p)) == norm_prefilter(dut.prefilter(p))
    dut.close()


def rl_values_of(amount):
    return {k: q(v) for k, v in amount.get("resourceRequests", {}).items()}


def test_delete_events(oracle, new_plugin):
    """Pod and throttle deletes (informer DeleteFunc): the row becomes a tombstone and is reused; used sums follow."""
    from test_scenarios import pod, throttle

    w = new_plugin(THROTTLER, SCHED)
    w.apply(namespace("default"), throttle("default", "t", {"a": "1"}, cpu="1"))
    for i in range(5):
        w.apply(pod("default", f"p{i}", "100m", {"a": "1"}, node="n", phase="Running"))
    w.reconcile_all(NOW)
    assert q(w.status("t", "default")["used"]["resourceRequests"]["cpu"]) == Fraction(1, 2)
    w.delete("Pod", "p1", "default")
    w.delete("Pod", "p3", "default")
    w.reconcile_all(NOW)
    s = w.status("t", "default")
    assert s["used"]["resourceCounts"]["pod"] == 3 and q(s["used"]["resourceRequests"]["cpu"]) == Fraction(3, 10)
    w.apply(pod("default", "p9", "700m", {"a": "1"}, node="n", phase="Running"))  # reuses a tombstone row
    w.reconcile_all(NOW)
    s = w.status("t", "default")
    assert s["used"]["resourceCounts"]["pod"] == 4 and q(s["used"]["resourceRequests"]["cpu"]) == 1 and s["throttled"]["resourceRequests"]["cpu"] is True
    w.delete("Throttle", "t", "default")
    assert w.prefilter(pod("default", "x", "1", {"a": "1"}))["code"] == "Success"
    w.close()


def test_column_scale_refinement(new_plugin):
    """A quantity finer than the column's scale (cpu below 1m) re-packs the column at a finer power of ten; sums stay exact."""
    from test_scenarios import pod, throttle

    w = new_plugin(THROTTLER, SCHED)
    w.apply(namespace("default"), throttle("default", "t", {"a": "1"}, cpu="1"))
    w.apply(pod("default", "p0", "100m", {"a": "1"}, node="n", phase="Running"))
    w.reconcile_all(NOW)
    w.apply(pod("default", "p1", "100u", {"a": "1"}, node="n", phase="Running"), pod("default", "p2", "1n", {"a": "1"}, node="n", phase="Running"))
    w.reconcile_all(NOW)
    assert q(w.status("t", "default")["used"]["resourceRequests"]["cpu"]) == Fraction(1, 10) + Fraction(1, 10**4) + Fraction(1, 10**9)
    r = w.prefilter(pod("default", "x", "899899999n", {"a": "1"}))  # 0.1 + 0.0001 + 1n + 0.899899999 == 1 exactly: not > threshold
    assert r["code"] == "Success"
    r = w.prefilter(pod("default", "y", "899900000n", {"a": "1"}))
    assert r["reasons"] == ["throttle[insufficient]=default/t"]
    w.close()


def test_gauges_follow_reconcile(new_plugin):
    """kth_metrics: series are recorded by reconcile (throttle_controller.go:159,187), only for reconciled (responsible)
    throttles, and stay after the throttle is deleted (a GaugeVec never drops a series)."""
    from test_scenarios import clthrottle, pod, throttle

    w = new_plugin(THROTTLER, SCHED)
    t = throttle("default", "t", {"a": "1"}, pod_cnt=2, cpu="1")
    t["metadata"]["uid"] = "uid-t"
    w.apply(namespace("default"), t, throttle("default", "other", {"a": "1"}, cpu="1", throttler="someone-else"),
            clthrottle("c", {"kubernetes.io/metadata.name": "default"}, {"a": "1"}, cpu="250m"))
    assert w.metrics() == ""  # nothing reconciled yet
    for i in range(3):
        w.apply(pod("default", f"p{i}", "100m", {"a": "1"}, node="n", phase="Running"))
    w.reconcile_all(NOW)
    s = {}
    for line in w.metrics().splitlines():
        if not line.startswith("#"):
            k, v = line.rsplit(" ", 1)
            s[k] = v
    lt = '{name="t",namespace="default",resource="%s",uid="uid-t"}'
    assert s["throttle_status_used_resourceCounts" + lt % "pod"] == "3"
    assert s["throttle_status_used_resourceRequests" + lt % "cpu"] == "300"
    assert s["throttle_status_throttled_resourceCounts" + lt % "pod"] == "1"
    assert s["throttle_status_throttled_resourceRequests" + lt % "cpu"] == "0"
    assert s["throttle_status_calculated_threshold_resourceRequests" + lt % "cpu"] == "1000"
    assert s["throttle_spec_threshold_resourceCounts" + lt % "pod"] == "2"
    lc = '{name="c",resource="%s",uid=""}'
    assert s["clusterthrottle_status_used_resourceRequests" + lc % "cpu"] == "300"
    assert s["clusterthrottle_status_throttled_resourceRequests" + lc % "cpu"] == "1"
    assert s["clusterthrottle_spec_threshold_resourceCounts" + lc % "pod"] == "0"
    assert not any('name="other"' in k for k in s)  # not ours: never enqueued, never recorded
    # a spec edit does not move the spec gauge until the next reconcile records it (the recorder runs inside reconcile)
    t2 = throttle("default", "t", {"a": "1"}, pod_cnt=7, cpu="1")
    t2["metadata"]["uid"] = "uid-t"
    w.apply(t2)
    assert f'throttle_spec_threshold_resourceCounts{lt % "pod"} 2' in w.metrics()
    w.reconcile_all(NOW)
    assert f'throttle_spec_threshold_resourceCounts{lt % "pod"} 7' in w.metrics()
    w.delete("Throttle", "t", "default")
    w.reconcile_all(NOW)
    assert "throttle_status_used_resourceCounts" + lt % "pod" in w.metrics()
    w.close()


def test_objects_beyond_the_limits_are_rejected_not_fatal(new_plugin):
    """A pod with more labels than KT_MAX_LABEL_SLOTS (32), a namespace likewise, or a 32nd distinct resource name is refused with
    an error for THAT object; the plugin keeps serving (the limits are checked before any state is touched)."""
    from test_scenarios import pod, throttle

    w = new_plugin(THROTTLER, SCHED)
    w.apply(namespace("default"), throttle("default", "t", {"a": "1"}, cpu="1"))
    w.apply(pod("default", "p0", "300m", {"a": "1"}, node="n", phase="Running"))
    with pytest.raises(RuntimeError, match="more than 32 labels"):
        w.apply(pod("default", "fat", "100m", {f"k{i}": "v" for i in range(33)}, node="n", phase="Running"))
    with pytest.raises(RuntimeError, match="more than 31 labels"):
        w.apply(namespace("fat-ns", {f"l{i}": "x" for i in range(33)}))
    with pytest.raises(RuntimeError, match="distinct resource names"):
        w.apply(pod("default", "greedy", "100m", {"a": "1"}, node="n", phase="Running", requests={f"example.com/r{i}": "1" for i in range(40)}))
    w.reconcile_all(NOW)
    s = w.status("t", "default")
    assert s["used"]["resourceCounts"]["pod"] == 1 and q(s["used"]["resourceRequests"]["cpu"]) == Fraction(3, 10)
    assert w.prefilter(pod("default", "x", "800m", {"a": "1"}))["reasons"] == ["throttle[insufficient]=default/t"]
    assert w.prefilter(pod("default", "y", "700m", {"a": "1"}))["code"] == "Success"
    w.close()


def test_selector_errors_q9(oracle, new_plugin):
    """Q9: a podSelector that LabelSelectorAsSelector rejects makes PreFilter return framework.Error with the conversion error
    for every pod the controller would have asked it about (plugin.go:154-156,166-168), and keeps that throttle -- only that
    one -- from being reconciled; a namespaceSelector that fails to convert is swallowed and simply never matches
    (clusterthrottle_selector.go:65-67,74-76)."""
    from test_scenarios import pod, throttle

    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    bad = {"matchExpressions": [{"key": "a", "operator": "In", "values": []}]}
    spec = lambda terms: {"throttlerName": THROTTLER, "threshold": {"resourceRequests": {"cpu": "1"}}, "selector": {"selectorTerms": terms}}
    both(namespace("default", {"team": "x"}), namespace("other", {"team": "y"}), throttle("default", "ok", {"a": "1"}, cpu="1"),
         {"kind": "ClusterThrottle", "metadata": {"name": "cbadns"}, "spec": spec([{"namespaceSelector": bad, "podSelector": {"matchLabels": {"a": "1"}}}])},
         pod("default", "p0", "300m", {"a": "1"}, node="n", phase="Running"), pod("other", "p1", "300m", {"a": "1"}, node="n", phase="Running"))
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    for name, ns in (("ok", "default"), ("cbadns", "")):
        assert norm_status(ref.status(name, ns)) == norm_status(dut.status(name, ns))
    assert "resourceCounts" not in dut.status("cbadns")["used"]  # the swallowed namespace-selector error: nothing ever matches
    probes = [pod("default", "x", "100m", {"a": "1"}), pod("other", "y", "100m", {"a": "1"}), pod("default", "z", "100m", {"q": "1"})]
    for p in probes:
        assert norm_prefilter(ref.prefilter(p)) == norm_prefilter(dut.prefilter(p))

    def verdict(w, p):  # what the scheduler sees of an Error status: the code and the message
        r = w.prefilter(p)
        return r["code"], r["reasons"]

    both({"kind": "Throttle", "metadata": {"namespace": "default", "name": "bad"}, "spec": spec([{"podSelector": bad}])})
    with pytest.raises(RuntimeError, match="values set can't be empty"):
        ref.reconcile_all(NOW)      # the oracle reports the failing key; the others were reconciled all the same
    dut.reconcile_all(NOW)
    assert norm_status(ref.status("ok", "default")) == norm_status(dut.status("ok", "default"))
    assert norm_status(ref.status("bad", "default")) == norm_status(dut.status("bad", "default"))  # untouched: never reconciled
    for p in probes:
        assert verdict(ref, p) == verdict(dut, p)
    assert verdict(dut, probes[0])[0] == "Error" and verdict(dut, probes[1])[0] != "Error"  # only the namespace of the broken Throttle
    both({"kind": "ClusterThrottle", "metadata": {"name": "cbadpod"}, "spec": spec([{"namespaceSelector": {"matchLabels": {"team": "y"}}, "podSelector": bad}])})
    for p in probes:
        assert verdict(ref, p) == verdict(dut, p)
    assert verdict(dut, probes[1])[0] == "Error"  # its namespaceSelector picks "other": pods there now get the conversion error
    dut.close()


def test_selector_error_behind_a_valid_term(oracle, new_plugin):
    """MatchesToPod walks the terms in order and returns at the first match (throttle_selector.go:30-42): a term that does not
    convert only hurts the pods that get as far as it.  A Throttle {valid term, broken term} is reconciled as long as every
    counted pod of its namespace matches the valid term, stops being reconciled when one does not, and PreFilter fails only for
    the pods that reach the broken term."""
    from test_scenarios import pod

    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    bad = {"matchExpressions": [{"key": "a", "operator": "Exists", "values": ["x"]}]}
    mixed = {"kind": "Throttle", "metadata": {"namespace": "default", "name": "mixed"},
             "spec": {"throttlerName": THROTTLER, "threshold": {"resourceCounts": {"pod": 2}, "resourceRequests": {"cpu": "1"}},
                      "selector": {"selectorTerms": [{"podSelector": {"matchLabels": {"a": "1"}}}, {"podSelector": bad}, {"podSelector": {"matchLabels": {"b": "1"}}}]}}}
    both(namespace("default"), namespace("other"), mixed)

    def reconcile_both():
        try:
            ref.reconcile_all(NOW)
            ok = True
        except RuntimeError:
            ok = False
        dut.reconcile_all(NOW)
        assert norm_status(ref.status("mixed", "default")) == norm_status(dut.status("mixed", "default"))
        return ok

    assert reconcile_both()  # no pod has asked the selector anything yet
    assert dut.status("mixed", "default")["calculatedThreshold"]["calculatedAtSet"] is True
    both(pod("default", "p0", "300m", {"a": "1"}, node="n", phase="Running"), pod("default", "p1", "300m", {"a": "1", "b": "1"}, node="n", phase="Succeeded"),
         pod("other", "elsewhere", "300m", {"c": "1"}, node="n", phase="Running"), pod("default", "unscheduled", "300m", {"c": "1"}))
    assert reconcile_both()
    assert dut.status("mixed", "default")["used"]["resourceCounts"]["pod"] == 1
    both(pod("default", "p2", "300m", {"b": "1"}, node="n", phase="Running"))  # matches only the term BEHIND the broken one
    assert not reconcile_both()
    assert dut.status("mixed", "default")["used"]["resourceCounts"]["pod"] == 1  # untouched
    for p in (pod("default", "x", "100m", {"a": "1"}), pod("default", "y", "100m", {"b": "1"}), pod("default", "z", "100m", {}), pod("other", "w", "100m", {"b": "1"})):
        a, b = ref.prefilter(p), dut.prefilter(p)
        assert (a["code"], a["reasons"]) == (b["code"], b["reasons"])
    both(pod("default", "p2", "300m", {"a": "1", "b": "1"}, node="n", phase="Running"))  # relabelled: now the valid term takes it
    both(pod("default", "p3", "400m", {"a": "1"}, node="n", phase="Running"))
    assert reconcile_both()
    assert dut.status("mixed", "default")["used"]["resourceCounts"]["pod"] == 3 and dut.status("mixed", "default")["throttled"]["resourceCounts"]["pod"] is True
    dut.close()


def test_clusterthrottle_selector_error_is_scoped_by_its_namespace_selector(oracle, new_plugin):
    """ClusterThrottleSelectorTerm.MatchesToPod checks the term's namespaceSelector FIRST (clusterthrottle_selector.go:71-87): a
    podSelector that does not convert only hurts pods of the namespaces that term selects, and only those that no EARLIER valid term
    took; pods elsewhere go on to the LATER terms.  One malformed ClusterThrottle scoped to one namespace must not fail PreFilter
    cluster-wide, and it is still reconciled as long as no counted pod runs into the broken term."""
    from test_scenarios import pod

    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    bad = {"matchExpressions": [{"key": "a", "operator": "Exists", "values": ["x"]}]}
    everywhere = {}
    only_x = {"matchLabels": {"team": "x"}}
    mixed = {"kind": "ClusterThrottle", "metadata": {"name": "mixed"},
             "spec": {"throttlerName": THROTTLER, "threshold": {"resourceCounts": {"pod": 3}, "resourceRequests": {"cpu": "2"}},
                      "selector": {"selectorTerms": [{"namespaceSelector": everywhere, "podSelector": {"matchLabels": {"a": "1"}}},
                                                     {"namespaceSelector": only_x, "podSelector": bad},
                                                     {"namespaceSelector": everywhere, "podSelector": {"matchLabels": {"b": "1"}}}]}}}
    both(namespace("nx", {"team": "x"}), namespace("ny", {"team": "y"}), mixed)

    def reconcile_both():
        try:
            ref.reconcile_all(NOW)
            ok = True
        except RuntimeError:
            ok = False
        dut.reconcile_all(NOW)
        assert norm_status(ref.status("mixed")) == norm_status(dut.status("mixed"))
        return ok

    def same_verdicts():
        out = []
        for p in (pod("nx", "x", "100m", {"a": "1"}), pod("nx", "y", "100m", {"b": "1"}), pod("nx", "z", "100m", {}),
                  pod("ny", "x", "100m", {"a": "1"}), pod("ny", "y", "100m", {"b": "1"}), pod("ny", "z", "100m", {})):
            a, b = ref.prefilter(p), dut.prefilter(p)
            assert (a["code"], a["reasons"]) == (b["code"], b["reasons"]), (p["metadata"], a, b)
            out.append(b["code"])
        return out

    assert reconcile_both()
    # nx: the valid first term saves a=1, everything else runs into the broken term; ny never sees it
    assert same_verdicts() == ["Success", "Error", "Error", "Success", "Success", "Success"]
    both(pod("nx", "p0", "300m", {"a": "1"}, node="n", phase="Running"), pod("ny", "p1", "300m", {"b": "1"}, node="n", phase="Running"),
         pod("ny", "p2", "300m", {"c": "1"}, node="n", phase="Running"))
    assert reconcile_both()  # nobody in nx reaches the broken term; ny's b=1 pod is counted through the term BEHIND it
    assert dut.status("mixed")["used"]["resourceCounts"]["pod"] == 2
    both(pod("nx", "p3", "300m", {"b": "1"}, node="n", phase="Running"))  # in nx, not taken by the first term: the broken one is next
    assert not reconcile_both()
    assert dut.status("mixed")["used"]["resourceCounts"]["pod"] == 2  # untouched
    same_verdicts()
    both(pod("nx", "p3", "300m", {"a": "1", "b": "1"}, node="n", phase="Running"))  # relabelled: the first term takes it
    assert reconcile_both()
    assert dut.status("mixed")["used"]["resourceCounts"]["pod"] == 3 and dut.status("mixed")["throttled"]["resourceCounts"]["pod"] is True
    same_verdicts()
    dut.close()


def test_q8_finished_pods_keep_their_reservation(oracle, new_plugin):
    """Q8: `terminatedPods = append(nonterminatedPods, pod)` (throttle_controller.go:241) leaves only the LAST finished match in
    the Throttle controller's list, so a reconcile un-reserves the running pods it observes and one finished pod; the other
    finished pods keep their reservation (and keep counting against later pods).  ClusterThrottles (correct code,
    clusterthrottle_controller.go:266) un-reserve all of them."""
    from test_scenarios import clthrottle, pod, throttle

    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    both(namespace("default"), throttle("default", "t", {"a": "1"}, cpu="10"), clthrottle("c", {"kubernetes.io/metadata.name": "default"}, {"a": "1"}, cpu="10"))
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    queue = [pod("default", f"q{i}", "1", {"a": "1"}) for i in range(4)]
    for p in queue:
        assert ref.prefilter(p)["code"] == dut.prefilter(p)["code"] == "Success"
        assert ref.reserve(p)["code"] == dut.reserve(p)["code"] == "Success"
    # q0 and q2 ran to completion before the next reconcile, q1 is running, q3 is still only reserved
    both(dict(queue[0], spec=dict(queue[0]["spec"], nodeName="n"), status={"phase": "Succeeded"}),
         dict(queue[1], spec=dict(queue[1]["spec"], nodeName="n"), status={"phase": "Running"}),
         dict(queue[2], spec=dict(queue[2]["spec"], nodeName="n"), status={"phase": "Failed"}))
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    for kind, nn in (("Throttle", "default/t"), ("ClusterThrottle", "/c")):
        a, b = ref.reserved(kind, nn), dut.reserved(kind, nn)
        assert sorted(a["pods"]) == sorted(b["pods"]) and norm_amount(a["amount"]) == norm_amount(b["amount"]), (nn, a, b)
    assert sorted(dut.reserved("Throttle", "default/t")["pods"]) == ["default/q0", "default/q3"]  # q2 (the last finished one) and q1 left
    assert dut.reserved("ClusterThrottle", "/c")["pods"] == ["default/q3"]
    for name, ns in (("t", "default"), ("c", "")):
        assert norm_status(ref.status(name, ns)) == norm_status(dut.status(name, ns))
    probe = pod("default", "x", "7500m", {"a": "1"})  # used 1 (q1) + reserved: 2 on the Throttle, 1 on the ClusterThrottle
    assert norm_prefilter(ref.prefilter(probe)) == norm_prefilter(dut.prefilter(probe))
    assert dut.prefilter(probe)["reasons"] == ["throttle[insufficient]=default/t"]
    dut.close()


# ---- random EVENT STREAMS: informer events, scheduling cycles and reconciles interleaved at random ---------------------------
TIMES = ["2026-01-01T00:00:00Z", "2026-01-15T12:00:00Z", "2026-03-01T12:00:00Z", "2025-12-31T23:59:59Z"]
def run_event_stream(oracle, new_plugin, seed, n_thr=14, n_ns=4, check_every_reconcile=False):
    rng = random.Random(seed)
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    nss = [f"ns{i}" for i in range(n_ns)]
    for n in nss: both(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
    throttles = [rand_throttle(rng, i, nss) for i in range(n_thr)]  # (tools/chaos_host.py also runs 80 of them: several 32-throttle words)
    both(*throttles)
    pods = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(60)]
    both(*pods)
    pending = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(40)]
    reserved = []
    gone = set()  # indices of throttles that are deleted right now (an edit brings them back under the same name)
    log = []
    for step in range(60):
        op = rng.random()
        if op < 0.2:
            now = rng.choice(TIMES); log.append(("reconcile", now))
            try: ref.reconcile_all(now)
            except RuntimeError: pass
            dut.reconcile_all(now)
            if check_every_reconcile:  # (tools/chaos_host.py: every status and reservation after EVERY reconcile, not only at the end)
                for i, t in enumerate(throttles):
                    ns = t["metadata"].get("namespace", "")
                    if i not in gone:
                        a, b = ref.status(t["metadata"]["name"], ns), dut.status(t["metadata"]["name"], ns)
                        assert norm_status(a) == norm_status(b), (seed, step, "status", t["metadata"], log[-5:], a, b)
                    k, nn = t["kind"], ns + "/" + t["metadata"]["name"]
                    a, b = ref.reserved(k, nn), dut.reserved(k, nn)
                    assert sorted(a["pods"]) == sorted(b["pods"]) and norm_amount(a["amount"]) == norm_amount(b["amount"]), (seed, step, "reserved", nn, log[-5:], a, b)
        elif op < 0.23:
            batch = rng.sample(pending, 6); log.append(("prefilter-batch", [p["metadata"]["name"] for p in batch]))
            want = [ref.prefilter(p) for p in batch]
            got = dut.prefilter_batch(batch)  # one device pass for the lot: independent checks against the same snapshot
            assert [(a["code"], a["reasons"]) for a in want] == [(b["code"], b["reasons"]) for b in got], (seed, step, log[-5:])
        elif op < 0.27:
            names = {p["metadata"]["name"] for p in reserved}
            queue = [p for p in rng.sample(pending, 8) if p["metadata"]["name"] not in names]; log.append(("admit-queue", len(queue)))
            want = []
            for p in queue:  # the scheduler's cycle, pod by pod
                r = ref.prefilter(p)
                if r["code"] == "Success":
                    assert ref.reserve(p)["code"] == "Success"
                want.append((r["code"], r["reasons"]))
            got = dut.admit_queue(queue)
            assert [(x["preFilter"]["code"], x["preFilter"]["reasons"]) for x in got["results"]] == want, (seed, step, log[-5:])
            reserved.extend(p for p, w in zip(queue, want) if w[0] == "Success")
        elif op < 0.45:
            p = rng.choice(pending); log.append(("prefilter", p["metadata"]["name"]))
            a, b = ref.prefilter(p), dut.prefilter(p)
            assert (a["code"], a["reasons"]) == (b["code"], b["reasons"]), (seed, step, log[-5:], a, b)
            if a["code"] == "Success" and rng.random() < 0.7:
                assert ref.reserve(p)["code"] == dut.reserve(p)["code"]
                reserved.append(p)
        elif op < 0.55 and reserved:
            p = reserved.pop(rng.randrange(len(reserved))); log.append(("bind-or-unreserve", p["metadata"]["name"]))
            if rng.random() < 0.6:
                both(dict(p, spec=dict(p["spec"], nodeName="node-2"), status={"phase": rng.choice(["Running", "Running", "Succeeded"])}))
            else:
                ref.unreserve(p); dut.unreserve(p)
        elif op < 0.64:
            p = rng.choice(pods); log.append(("relabel", p["metadata"]["name"]))
            p["metadata"]["labels"] = rand_labels(rng)
            if rng.random() < 0.3: p["status"] = {"phase": rng.choice(["Running", "Succeeded", "Failed"])}
            both(p)
        elif op < 0.68:
            i = rng.randrange(len(pods)); log.append(("mutate-pod", pods[i]["metadata"]["name"]))  # anything may change: requests, scheduler, node, phase
            pods[i] = rand_pod(rng, pods[i]["metadata"]["namespace"], pods[i]["metadata"]["name"], True)
            both(pods[i])
        elif op < 0.7 and reserved:
            p = rng.choice(reserved); log.append(("re-reserve", p["metadata"]["name"]))  # addPod overwrites the amount it kept
            p["spec"]["containers"][0]["resources"]["requests"]["cpu"] = rng.choice(CPUS)
            assert ref.reserve(p)["code"] == dut.reserve(p)["code"]
        elif op < 0.8:
            i = rng.randrange(len(throttles)); log.append(("edit-throttle", i))
            t = rand_throttle(rng, i, nss)
            t["kind"] = throttles[i]["kind"]; t["metadata"] = throttles[i]["metadata"]
            if t["kind"] == "Throttle":
                for term in t["spec"]["selector"]["selectorTerms"]: term.pop("namespaceSelector", None)
                if t["spec"]["selector"]["selectorTerms"] and rng.random() < 0.15:  # a podSelector that does not convert, at a random position (Q9)
                    rng.choice(t["spec"]["selector"]["selectorTerms"])["podSelector"] = rng.choice([
                        {"matchExpressions": [{"key": "team", "operator": "In", "values": []}]},
                        {"matchExpressions": [{"key": "env", "operator": "Exists", "values": ["a"]}]},
                        {"matchLabels": {"bad key!": "x"}}])
            throttles[i] = t
            gone.discard(i)
            both(t)
        elif op < 0.86:
            n = rng.choice(nss); log.append(("relabel-ns", n))  # also what brings a deleted namespace back
            both(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
        elif op < 0.88:
            n = rng.choice(nss); log.append(("delete-ns", n))  # the lister stops returning it; its pods and throttles stay
            ref.delete("Namespace", n), dut.delete("Namespace", n)
        elif op < 0.91 and len(gone) < 5:
            i = rng.randrange(len(throttles)); log.append(("delete-throttle", i))  # its reservations stay in the cache (no way to drop them)
            if i not in gone:
                gone.add(i)
                md = throttles[i]["metadata"]
                ref.delete(throttles[i]["kind"], md["name"], md.get("namespace", "")), dut.delete(throttles[i]["kind"], md["name"], md.get("namespace", ""))
        elif op < 0.95 and len(pods) > 20:
            p = pods.pop(rng.randrange(len(pods))); log.append(("delete-pod", p["metadata"]["name"]))  # informer Delete event
            ref.delete("Pod", p["metadata"]["name"], p["metadata"]["namespace"]), dut.delete("Pod", p["metadata"]["name"], p["metadata"]["namespace"])
        else:
            p = rand_pod(rng, rng.choice(nss), f"n{step}", True); pods.append(p); log.append(("new-pod", p["metadata"]["name"]))
            both(p)
    for now in (TIMES[1],):
        try: ref.reconcile_all(now)
        except RuntimeError: pass
        dut.reconcile_all(now)
    for i, t in enumerate(throttles):
        ns = t["metadata"].get("namespace", "")
        if i not in gone:
            a, b = ref.status(t["metadata"]["name"], ns), dut.status(t["metadata"]["name"], ns)
            assert norm_status(a) == norm_status(b), (seed, "status", t["metadata"], a, b)
        k, nn = t["kind"], ns + "/" + t["metadata"]["name"]
        a, b = ref.reserved(k, nn), dut.reserved(k, nn)
        assert sorted(a["pods"]) == sorted(b["pods"]), (seed, "reserved", nn, a, b)
    for p in pending:
        a, b = ref.prefilter(p), dut.prefilter(p)
        assert (a["code"], a["reasons"]) == (b["code"], b["reasons"]), (seed, "final", a, b)
    dut.close()


@pytest.mark.parametrize("seed", [0, 1, 2, 3, 4, 5, 8, 17])  # 8 and 17: a throttle is deleted and comes back while pods are reserved on it
def test_event_stream_chaos(oracle, new_plugin, seed):
    """Sixty random steps per seed -- reconciles at different clock times (override windows open and close), PreFilter + Reserve, batched
    PreFilter and queue admission,
    binds (some pods finish at once), Unreserve, pod relabels (reservation moves), pod deletes, throttle spec edits, throttle deletes
    and re-creations, namespace relabels and deletes, new pods -- applied to the oracle and to the plugin alike; every verdict on the way and every status, reservation and verdict at
    the end must agree.  (tools/chaos_host.py runs more seeds on the CPU double.)"""
    run_event_stream(oracle, new_plugin, seed)


def run_queue_stream(oracle, new_plugin, seed, n_thr=10, ns_deletes=False):
    """The RESIDENT scheduling queue under churn: the pending pods are delivered by the informer (they live in the device's
    pending table), PreFilter / Reserve / Unreserve address them by key, the whole queue is asked for in one call -- while
    throttles of both kinds are created, edited (new selector vocabulary: rows packed as 'some other value' are packed again),
    deleted and re-created (the device columns are laid out again), pods are relabelled, bound and deleted, namespaces relabelled.
    Every by-key verdict must equal the oracle's PreFilter of the same pod, every verdict byte of the queue call its code."""
    rng = random.Random(seed)
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    key = lambda p: (p["metadata"]["namespace"], p["metadata"]["name"])
    nss = [f"ns{i}" for i in range(5)]
    both(*[namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}) for n in nss])
    throttles = [rand_throttle(rng, i, nss) for i in range(n_thr)]
    both(*throttles)
    both(*[rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(50)])
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(36)]
    both(*queue)
    names = {"Success": 1, "UnschedulableAndUnresolvable": 2, "Error": 3}
    reserved, log = [], []
    for step in range(50):
        op = rng.random()
        if op < 0.12:
            now = rng.choice(TIMES); log.append(("reconcile", now))
            try: ref.reconcile_all(now)
            except RuntimeError: pass
            dut.reconcile_all(now)
        elif op < 0.40 and queue:
            p = rng.choice(queue); log.append(("prefilter-key", key(p)))
            a, b = ref.prefilter(p), dut.prefilter_key(*key(p))
            assert norm_prefilter(a) == norm_prefilter(b), (seed, step, log[-5:], a, b)
            if a["code"] == "Success" and rng.random() < 0.6:
                assert ref.reserve(p)["code"] == dut.reserve_key(*key(p))["code"] == "Success"
                if p not in reserved: reserved.append(p)
        elif op < 0.47 and queue:
            log.append(("prefilter-queue", len(queue)))
            verdicts = dut.prefilter_queue()
            for p in queue:
                row = dut.queue_row(*key(p))
                if row < 0:
                    assert p["spec"]["schedulerName"] != SCHED, (seed, step, key(p))
                    continue
                assert verdicts[row] == names[ref.prefilter(p)["code"]], (seed, step, log[-5:], key(p))
        elif op < 0.55 and reserved:
            p = reserved.pop(rng.randrange(len(reserved))); log.append(("bind-or-unreserve", key(p)))
            if rng.random() < 0.5:
                queue.remove(p)
                both(dict(p, spec=dict(p["spec"], nodeName="node-9"), status={"phase": "Running"}))
                assert dut.queue_row(*key(p)) == -1
            else:
                ref.unreserve(p), dut.unreserve_key(*key(p))
        elif op < 0.63 and queue:
            p = rng.choice(queue); log.append(("relabel-queued", key(p)))
            p["metadata"]["labels"] = rand_labels(rng)
            both(p)
        elif op < 0.78:
            i = rng.randrange(len(throttles) + 3); log.append(("apply-throttle", i))  # an edit, or a new one
            t = rand_throttle(rng, i, nss)
            if i < len(throttles):
                t["kind"] = throttles[i]["kind"]; t["metadata"] = throttles[i]["metadata"]
                if t["kind"] == "Throttle":
                    for term in t["spec"]["selector"]["selectorTerms"]: term.pop("namespaceSelector", None)
                throttles[i] = t
            else:
                t["metadata"]["name"] += f"-s{step}"
                throttles.append(t)
            both(t)
        elif op < 0.84 and len(throttles) > 4:
            t = throttles.pop(rng.randrange(len(throttles))); log.append(("delete-throttle", t["metadata"]["name"]))
            md = t["metadata"]
            ref.delete(t["kind"], md["name"], md.get("namespace", "")), dut.delete(t["kind"], md["name"], md.get("namespace", ""))
        elif op < 0.89:
            n = rng.choice(nss)
            if ns_deletes and rng.random() < 0.4:  # (tools/chaos_host.py) the lister stops returning it; its pods and throttles stay: Error verdicts
                log.append(("delete-ns", n)); ref.delete("Namespace", n), dut.delete("Namespace", n)
            else:
                log.append(("relabel-ns", n)); both(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
        elif op < 0.94 and len(queue) > 10:
            p = queue.pop(rng.randrange(len(queue))); log.append(("delete-queued", key(p)))
            if p in reserved: reserved.remove(p)
            ref.delete("Pod", p["metadata"]["name"], p["metadata"]["namespace"]), dut.delete("Pod", p["metadata"]["name"], p["metadata"]["namespace"])
        else:
            p = rand_pod(rng, rng.choice(nss), f"n{step}", False); queue.append(p); log.append(("new-queued", key(p)))
            both(p)
    for p in queue:
        a, b = ref.prefilter(p), dut.prefilter_key(*key(p))
        assert norm_prefilter(a) == norm_prefilter(b), (seed, "final", key(p), a, b)
    for t in throttles:
        k, nn = t["kind"], t["metadata"].get("namespace", "") + "/" + t["metadata"]["name"]
        a, b = ref.reserved(k, nn), dut.reserved(k, nn)
        assert sorted(a["pods"]) == sorted(b["pods"]) and norm_amount(a["amount"]) == norm_amount(b["amount"]), (seed, "reserved", nn, a, b)
    dut.close()


@pytest.mark.parametrize("seed", [0, 1, 2, 3, 2410, 2703, 2793])  # 2410 ...: a throttle edit, then a RECONCILE, then PreFilter by key -- the cached
def test_resident_queue_event_stream(oracle, new_plugin, seed):      # verdicts of the old throttle set must not answer (they did)
    """Random events against the resident scheduling queue, by key (tools/chaos_host.py runs more seeds on the CPU double)."""
    run_queue_stream(oracle, new_plugin, seed)


def rand_status(rng):
    """A status subresource as another writer (a restart, a second controller instance) may have left it."""
    st = {}
    if rng.random() < 0.8:
        ct = {"threshold": rand_amount(rng, 2)}
        if rng.random() < 0.7: ct["calculatedAt"] = rng.choice(TIMES)
        if rng.random() < 0.2: ct["messages"] = ["m"]
        st["calculatedThreshold"] = ct
    thr = {}
    if rng.random() < 0.6: thr["resourceCounts"] = {"pod": rng.random() < 0.3}
    if rng.random() < 0.7: thr["resourceRequests"] = {k: rng.random() < 0.3 for k in rng.sample(["cpu", "memory", "nvidia.com/gpu"], rng.randrange(0, 3))}
    if thr: st["throttled"] = thr
    if rng.random() < 0.8: st["used"] = rand_amount(rng, 3)
    return st


def run_status_stream(oracle, new_plugin, seed):
    """PreFilter reads the INFORMER COPY of .status (plugin.go:148-216 -> CheckThrottledFor with the status as it was last
    delivered): statuses arrive through the informer -- at start-up, from another writer -- stale or plain wrong, with or without
    calculatedAt (Q6: which threshold counts), with throttled flags and used amounts that have nothing to do with the pods;
    reconciles replace them only where apiequality.Semantic.DeepEqual says they differ.  Every verdict in between and every status
    after every reconcile must equal the oracle's."""
    rng = random.Random(seed)
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    nss = [f"ns{i}" for i in range(4)]
    both(*[namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}) for n in nss])
    throttles = [rand_throttle(rng, i, nss) for i in range(12)]
    both(*[dict(t, status=rand_status(rng)) if rng.random() < 0.7 else t for t in throttles])  # what the informer delivers at start-up
    both(*[rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(40)])
    pending = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(30)]
    log = []
    for step in range(40):
        op = rng.random()
        if op < 0.5:
            p = rng.choice(pending); log.append(("prefilter", p["metadata"]["name"]))
            a, b = ref.prefilter(p), dut.prefilter(p)
            assert norm_prefilter(a) == norm_prefilter(b), (seed, step, log[-5:], a, b)
            if a["code"] == "Success" and rng.random() < 0.5:
                assert ref.reserve(p)["code"] == dut.reserve(p)["code"]
        elif op < 0.7:
            i = rng.randrange(len(throttles)); log.append(("apply-status", i))  # another writer's status arrives through the informer
            both(dict(throttles[i], status=rand_status(rng)))
        elif op < 0.8:
            i = rng.randrange(len(throttles)); log.append(("edit-spec", i))   # a spec update: the status is kept
            t = rand_throttle(rng, i, nss); t["kind"] = throttles[i]["kind"]; t["metadata"] = throttles[i]["metadata"]
            if t["kind"] == "Throttle":
                for term in t["spec"]["selector"]["selectorTerms"]: term.pop("namespaceSelector", None)
            throttles[i] = t
            both(t)
        elif op < 0.9:
            now = rng.choice(TIMES); log.append(("reconcile", now))
            try: ref.reconcile_all(now)
            except RuntimeError: pass
            dut.reconcile_all(now)
            for t in throttles:
                ns = t["metadata"].get("namespace", "")
                a, b = ref.status(t["metadata"]["name"], ns), dut.status(t["metadata"]["name"], ns)
                assert norm_status(a) == norm_status(b), (seed, step, "status", t["metadata"], log[-5:], a, b)
        else:
            batch = rng.sample(pending, 5); log.append(("batch", 5))
            want = [ref.prefilter(p) for p in batch]
            got = dut.prefilter_batch(batch)
            assert [norm_prefilter(a) for a in want] == [norm_prefilter(b) for b in got], (seed, step, log[-5:])
    dut.close()


@pytest.mark.parametrize("seed", [0, 1, 2, 143])  # 143: `used: {resourceRequests: {}}` on a throttle that matches no pod -- nil and empty maps are EQUAL
def test_status_event_stream(oracle, new_plugin, seed):
    run_status_stream(oracle, new_plugin, seed)


EXTRA_RES = [f"vendor{i}.example.com/dev" for i in range(18)]
FINE = ["1n", "100n", "0.000001", "1u", "0.0015", "333m", "1.0000001"]
def grow_pod(rng, ns, name, running, stage):
    p = rand_pod(rng, ns, name, running)
    # stage grows: more labels (-> 16 / 32 label slots), more resource names (-> 8 / 16 / 31 columns), finer quantities (column re-scale)
    for i in range(rng.randrange(0, 1 + 4 * stage)):
        p["metadata"]["labels"][f"extra-{rng.randrange(0, 6 * stage + 1)}"] = rng.choice(VALS)
    reqs = p["spec"]["containers"][0]["resources"]["requests"]
    for r in rng.sample(EXTRA_RES[: 3 + 4 * stage], rng.randrange(0, min(3 + stage, 3 + 4 * stage))):
        reqs[r] = str(rng.randrange(0, 5))
    if rng.random() < 0.15 * stage: reqs["cpu"] = rng.choice(FINE)
    return p
def grow_throttle(rng, i, nss, stage):
    t = rand_throttle(rng, i, nss)
    rr = t["spec"]["threshold"].setdefault("resourceRequests", {})
    for r in rng.sample(EXTRA_RES[: 3 + 4 * stage], rng.randrange(0, 3)):
        rr[r] = str(rng.randrange(0, 9))
    if rng.random() < 0.1 * stage: rr["cpu"] = rng.choice(FINE + ["2", "0.5"])
    if rng.random() < 0.3 and t["spec"]["selector"]["selectorTerms"]:
        t["spec"]["selector"]["selectorTerms"][0]["podSelector"].setdefault("matchLabels", {})[f"extra-{rng.randrange(0, 6 * stage + 1)}"] = rng.choice(VALS)
    return t
def run_growth_stream(oracle, new_plugin, seed):
    rng = random.Random(seed)
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    key = lambda p: (p["metadata"]["namespace"], p["metadata"]["name"])
    nss = [f"ns{i}" for i in range(4)]
    both(*[namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}) for n in nss])
    throttles = [grow_throttle(rng, i, nss, 0) for i in range(10)]
    both(*throttles)
    pods = [grow_pod(rng, rng.choice(nss), f"p{i}", True, 0) for i in range(30)]
    both(*pods)
    queue = [grow_pod(rng, rng.choice(nss), f"q{i}", False, 0) for i in range(16)]
    both(*queue)
    reserved, log = [], []
    for step in range(48):
        stage = step // 12  # the limits are crossed as the stream goes on
        op = rng.random()
        if op < 0.12:
            now = rng.choice(TIMES); log.append(("reconcile", now))
            try: ref.reconcile_all(now)
            except RuntimeError: pass
            dut.reconcile_all(now)
            for t in throttles:
                ns = t["metadata"].get("namespace", "")
                a, b = ref.status(t["metadata"]["name"], ns), dut.status(t["metadata"]["name"], ns)
                assert norm_status(a) == norm_status(b), (seed, step, "status", t["metadata"], log[-5:], a, b)
        elif op < 0.35:
            p = rng.choice(queue); log.append(("prefilter-key", key(p)))
            a, b = ref.prefilter(p), dut.prefilter_key(*key(p))
            assert norm_prefilter(a) == norm_prefilter(b), (seed, step, log[-5:], a, b)
            if a["code"] == "Success" and rng.random() < 0.6:
                assert ref.reserve(p)["code"] == dut.reserve_key(*key(p))["code"] == "Success"
                if p not in reserved: reserved.append(p)
        elif op < 0.5:
            p = grow_pod(rng, rng.choice(nss), f"m{step}", False, stage); log.append(("prefilter-manifest", key(p)))
            a, b = ref.prefilter(p), dut.prefilter(p)
            assert norm_prefilter(a) == norm_prefilter(b), (seed, step, log[-5:], a, b)
            if a["code"] == "Success" and rng.random() < 0.4:
                assert ref.reserve(p)["code"] == dut.reserve(p)["code"]
        elif op < 0.7:
            p = grow_pod(rng, rng.choice(nss), f"n{step}", rng.random() < 0.6, stage); log.append(("new-pod", key(p)))
            both(p)
            if p["spec"]["nodeName"] == "" and p["status"]["phase"] == "Pending": queue.append(p)
        elif op < 0.85:
            i = rng.randrange(len(throttles) + 2); log.append(("apply-throttle", i))
            t = grow_throttle(rng, i, nss, stage)
            if i < len(throttles):
                t["kind"] = throttles[i]["kind"]; t["metadata"] = throttles[i]["metadata"]
                if t["kind"] == "Throttle":
                    for term in t["spec"]["selector"]["selectorTerms"]: term.pop("namespaceSelector", None)
                throttles[i] = t
            else:
                t["metadata"]["name"] += f"-s{step}"; throttles.append(t)
            both(t)
        elif op < 0.93 and reserved:
            p = reserved.pop(rng.randrange(len(reserved))); log.append(("unreserve", key(p)))
            ref.unreserve(p), dut.unreserve_key(*key(p))
        else:
            batch = rng.sample(queue, min(5, len(queue))); log.append(("admit-queue", len(batch)))
            names = {p["metadata"]["name"] for p in reserved}
            batch = [p for p in batch if p["metadata"]["name"] not in names]
            want = []
            for p in batch:
                r = ref.prefilter(p)
                if r["code"] == "Success": assert ref.reserve(p)["code"] == "Success"; reserved.append(p)
                want.append((r["code"], r["reasons"]))
            got = dut.admit_queue(batch)
            assert [(x["preFilter"]["code"], x["preFilter"]["reasons"]) for x in got["results"]] == want, (seed, step, log[-5:])
    for p in queue:
        a, b = ref.prefilter(p), dut.prefilter_key(*key(p))
        assert norm_prefilter(a) == norm_prefilter(b), (seed, "final", key(p), a, b)
    for t in throttles:
        k, nn = t["kind"], t["metadata"].get("namespace", "") + "/" + t["metadata"]["name"]
        a, b = ref.reserved(k, nn), dut.reserved(k, nn)
        assert sorted(a["pods"]) == sorted(b["pods"]) and norm_amount(a["amount"]) == norm_amount(b["amount"]), (seed, "reserved", nn, a, b)
    st = dut.queue_stats()
    dut.close()
    return st


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_growth_event_stream(oracle, new_plugin, seed):
    """A world that outgrows the engine's limits while it is in use: pods bring more and more labels (8 -> 16 -> 32 label slots)
    and resource names (4 -> 8 -> 16 -> 31 columns) and finer quantities (a column is re-scaled) -- the host layer re-creates the
    engine with larger limits and uploads its caches again, between PreFilter / Reserve by key and by manifest, reconciles, queue
    admissions and throttle edits.  Nothing may be lost on the way: verdicts, statuses and reservations equal the oracle's."""
    st = run_growth_stream(oracle, new_plugin, seed)
    assert st["resourceColumns"] > 8, st


def test_pods_of_a_namespace_the_lister_does_not_hold(oracle, new_plugin):
    """ClusterThrottleController.affectedPods walks the namespaces the lister returns (clusterthrottle_controller.go:227): pods of
    a namespace that was never seen, or was deleted, are not counted by ANY ClusterThrottle -- not even one whose namespaceSelector
    is empty -- while a namespaced Throttle (which never asks about the namespace) still counts them; PreFilter for such a pod
    fails in the ClusterThrottle controller with "not found" (:273-276)."""
    from test_scenarios import pod, throttle

    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    everywhere = {"kind": "ClusterThrottle", "metadata": {"name": "everywhere"},
                  "spec": {"throttlerName": THROTTLER, "threshold": {"resourceCounts": {"pod": 10}},
                           "selector": {"selectorTerms": [{"namespaceSelector": {}, "podSelector": {"matchLabels": {"a": "1"}}}]}}}
    notprod = {"kind": "ClusterThrottle", "metadata": {"name": "notprod"},
               "spec": {"throttlerName": THROTTLER, "threshold": {"resourceCounts": {"pod": 10}},
                        "selector": {"selectorTerms": [{"namespaceSelector": {"matchExpressions": [{"key": "env", "operator": "NotIn", "values": ["prod"]}]},
                                                        "podSelector": {}}]}}}
    both(namespace("seen", {"env": "dev"}), everywhere, notprod, throttle("ghost", "local", {"a": "1"}, pod_cnt=10),
         pod("seen", "p0", "100m", {"a": "1"}, node="n", phase="Running"), pod("ghost", "p1", "100m", {"a": "1"}, node="n", phase="Running"))

    def settle_and_compare():
        ref.reconcile_all(NOW), dut.reconcile_all(NOW)
        for name, ns in (("everywhere", ""), ("notprod", ""), ("local", "ghost")):
            assert norm_status(ref.status(name, ns)) == norm_status(dut.status(name, ns)), name
        for p in (pod("seen", "x", "100m", {"a": "1"}), pod("ghost", "y", "100m", {"a": "1"})):
            a, b = ref.prefilter(p), dut.prefilter(p)
            assert (a["code"], a["reasons"]) == (b["code"], b["reasons"])

    settle_and_compare()
    assert dut.status("everywhere")["used"]["resourceCounts"]["pod"] == 1 and dut.status("local", "ghost")["used"]["resourceCounts"]["pod"] == 1
    assert dut.prefilter(pod("ghost", "y", "100m", {"a": "1"}))["code"] == "Error"
    both(namespace("ghost", {"env": "dev"}))           # the namespace shows up
    settle_and_compare()
    assert dut.status("everywhere")["used"]["resourceCounts"]["pod"] == 2 and dut.status("notprod")["used"]["resourceCounts"]["pod"] == 2
    ref.delete("Namespace", "seen"), dut.delete("Namespace", "seen")   # and another one goes away
    settle_and_compare()
    assert dut.status("everywhere")["used"]["resourceCounts"]["pod"] == 1
    dut.close()
