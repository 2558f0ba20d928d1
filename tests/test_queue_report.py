"""kth_queue_report: the scheduling queue summarised per throttle in one device call, checked against the calls that define it.

The report must equal what kth_pre_filter_queue (the verdict counts), kth_affected_pods of every responsible throttle (the
per-status counts of its queued pods, and the ResourceAmountOfPod sum of the ones it holds back) and kth_pre_filter_key of every
queued pod (the pods one throttle alone blocks) say at the same moment.  Random worlds of test_plugin_vs_oracle, with a namespace
the lister never holds (Error pods), broken podSelectors, foreign throttles, tombstone rows of deleted queued pods, and every other
entry point run right before a report -- each runs device passes of its own, so a report that trusted the device's codes without
a pass at the current state would be caught.  Runs on the product (GPU) and on the product's host layer over an engine test
double whose kt_get_check_summary counts the recorded codes row by row (CPU)."""
import functools
import json
import os
import random
from decimal import Decimal

import pytest

from test_plugin_vs_oracle import VALS, rand_labels, rand_pod, rand_throttle
from test_reconcile_keys import BROKEN, _build
from test_scenarios import NOW, SCHED, THROTTLER, namespace, pod, throttle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUB = os.path.join(ROOT, "tests", "host_stub")


@pytest.fixture(scope="module")
def host_on_oracle_summary(oracle):
    """kt_host.cc linked against the oracle-backed engine test double plus its kt_reconcile_throttles, kt_get_match_columns,
    kt_match_pods and kt_get_check_summary (tests/host_stub/engine_oracle_summary.cc; it has no kt_check_pending_rows, so
    prefilter_keys is left out there); host.Plugin's signature.  CPU only; says nothing about the kernels."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_summary.cc")]
    deps = [os.path.join(STUB, f) for f in ("engine_oracle.cc", "engine_oracle_reconcile.cc", "engine_oracle_match_pods.cc")] + [os.path.join(ROOT, "oracle", "libkt_oracle.so")] + \
        [os.path.join(ROOT, "kube_throttler_b200", "csrc", f) for f in ("kt_json.h", "kt_quantity.h")] + \
        [os.path.join(ROOT, "include", f) for f in ("kt_b200.h", "kt_host.h")]
    lib = _build("libkt_hostoracle_summary.so", srcs, deps,
                 ["-L", os.path.join(ROOT, "oracle"), "-lkt_oracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    return functools.partial(host.Plugin, library=lib)


@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def new_plugin(request):
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle_summary")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin


STATUS_FIELD = {"active": "active", "insufficient": "insufficient", "pod-requests-exceeds-threshold": "podRequestsExceedsThreshold"}
REASON_KIND = {"throttle": "Throttle", "clusterthrottle": "ClusterThrottle"}


class World:
    """The manifests a plugin was given, so that the contract can be derived from the plugin's own calls."""

    def __init__(self, dut):
        self.dut, self.pods, self.thr, self.order = dut, {}, {}, []

    def apply(self, *ms):
        for m in ms:
            self.dut.apply(m)
            md = m["metadata"]
            if m["kind"] == "Pod":
                self.pods[md["namespace"] + "/" + md["name"]] = m
            elif m["kind"] in ("Throttle", "ClusterThrottle"):
                key = md.get("namespace", "") + "/" + md["name"]
                if (m["kind"], key) not in self.thr:
                    self.order.append((m["kind"], key))
                self.thr[(m["kind"], key)] = m

    def delete(self, kind, key):
        ns, _, name = key.partition("/")
        self.dut.delete(kind, name, ns)
        if kind == "Pod":
            self.pods.pop(key, None)
        else:
            self.thr.pop((kind, key), None)
            self.order.remove((kind, key))


def amount_of(dut, pod):
    """ResourceAmountOfPod through the plugin's own library (kth_eval)."""
    from kube_throttler_b200 import host

    return host._result(dut._L.kth_eval(json.dumps({"fn": "ResourceAmountOfPod", "pod": pod}).encode()))


def expected_report(w):
    """The report as the defining calls give it."""
    dut = w.dut
    verdicts = list(dut.prefilter_queue())
    want = {"queued": sum(v != 0 for v in verdicts), "success": verdicts.count(1), "unschedulable": verdicts.count(2),
            "error": verdicts.count(3), "throttles": []}
    only = {}
    for key, p in w.pods.items():
        ns, _, name = key.partition("/")
        if dut.queue_row(ns, name) < 0:
            continue
        r = dut.prefilter_key(ns, name)
        if r["code"] == "UnschedulableAndUnresolvable" and len(r["reasons"]) == 1:
            head, names = r["reasons"][0].split("=", 1)
            if "," not in names:
                k = (REASON_KIND[head.split("[")[0]], names)
                only[k] = only.get(k, 0) + 1
    for kind, key in w.order:
        t = w.thr[(kind, key)]
        if t["spec"]["throttlerName"] != THROTTLER:
            continue
        ns, _, name = key.partition("/")
        entry = {"key": key, "kind": kind, "active": 0, "insufficient": 0, "podRequestsExceedsThreshold": 0, "onlyBlocker": only.get((kind, key), 0)}
        try:
            queued = dut.affected_pods(name, ns)["queued"]
        except RuntimeError:  # a counted pod reaches a broken podSelector: affectedPods has no answer to compare with
            entry["heldBack"] = None
            want["throttles"].append(entry)
            continue
        pods, reqs = 0, {}
        for q in queued:
            if q["status"] == "not-throttled":
                continue
            entry[STATUS_FIELD[q["status"]]] += 1
            pods += 1
            for rn, v in amount_of(dut, w.pods[q["pod"]])["resourceRequests"].items():
                reqs[rn] = reqs.get(rn, Decimal(0)) + Decimal(v)
        entry["heldBack"] = {"resourceCounts": {"pod": pods}, "resourceRequests": reqs} if pods else {}
        want["throttles"].append(entry)
    return want


def normalised(report, want):
    """The report with its decimal strings as Decimals; entries whose affectedPods failed compare on their other fields."""
    out = dict(report, throttles=[])
    for e, ew in zip(report["throttles"], want["throttles"] + [None] * len(report["throttles"])):
        e = dict(e)
        hb = e["heldBack"]
        if "resourceRequests" in hb:
            hb = dict(hb, resourceRequests={k: Decimal(v) for k, v in hb["resourceRequests"].items()})
        e["heldBack"] = None if ew is not None and ew["heldBack"] is None else hb
        if ew is not None and ew["heldBack"] is None:
            for f in ("active", "insufficient", "podRequestsExceedsThreshold"):
                e[f] = ew[f]
        out["throttles"].append(e)
    return out


def has_prefilter_keys(dut):
    return hasattr(dut._L, "kt_check_pending_rows")  # (not in the CPU double)


def check(w, where=""):
    got = w.dut.queue_report()
    want = expected_report(w)
    assert normalised(got, want) == want, where
    return got


def random_world(dut, rng, n_thr=30, n_run=200, n_queue=60):
    w = World(dut)
    nss = [f"ns{i}" for i in range(5)]
    for n in nss[:4]:  # ns4 is never applied: its queued pods' PreFilter is an Error (ClusterThrottle controller)
        w.apply(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
    w.apply(*[rand_throttle(rng, i, nss) for i in range(n_thr)])
    w.apply(*[rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(n_run)])
    dut.reconcile_all(NOW)
    w.apply(*[rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(n_queue)])
    return w, nss


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_report_equals_its_definition(new_plugin, seed):
    rng = random.Random(seed)
    w, nss = random_world(new_plugin(THROTTLER, SCHED), rng)
    got = check(w, "fresh world")
    assert got["error"] > 0 and got["unschedulable"] > 0 and got["success"] > 0, got
    assert any(e["onlyBlocker"] for e in got["throttles"]) and any(e["heldBack"] for e in got["throttles"])
    assert {e["key"] for e in got["throttles"]} == {k for (_, k), t in w.thr.items() if t["spec"]["throttlerName"] == THROTTLER}
    assert w.dut.queue_report() == got  # twice in a row: the same answer
    w.dut.close()


def test_report_after_every_other_entry_point(new_plugin):
    """Each step runs some other call, which may change the state or run a device pass of its own; the report right after it
    must be that of the state now."""
    rng = random.Random(7)
    w, nss = random_world(new_plugin(THROTTLER, SCHED), rng, n_thr=24, n_run=150, n_queue=50)
    dut = w.dut
    queued = lambda: [k for k in w.pods if dut.queue_row(*k.split("/", 1)) >= 0]
    manifests = lambda k: [rand_pod(rng, rng.choice(nss), f"m{rng.randrange(10**6)}", False) for _ in range(k)]
    steps = [
        ("reconcile_all", lambda: dut.reconcile_all(NOW)),
        ("reconcile keys", lambda: dut.reconcile([k for (_, k) in w.order[:5]], NOW)),
        ("prefilter manifest", lambda: dut.prefilter(manifests(1)[0])),
        ("prefilter_batch", lambda: dut.prefilter_batch(manifests(20))),
        ("admit_queue", lambda: dut.admit_queue(manifests(6))),
        ("reserve_key", lambda: [dut.reserve_key(*k.split("/", 1)) for k in queued()[:6]]),
        ("unreserve_key", lambda: [dut.unreserve_key(*k.split("/", 1)) for k in queued()[:3]]),
        ("affected_pods", lambda: [dut.affected_pods(k.split("/", 1)[1], k.split("/", 1)[0]) for (kind, k) in w.order[:6]
                                   if w.thr[(kind, k)]["spec"]["throttlerName"] == THROTTLER]),
        ("prefilter_key", lambda: [dut.prefilter_key(*k.split("/", 1)) for k in queued()[:10]]),
        ("prefilter_queue", lambda: dut.prefilter_queue()),
        ("apply_events", lambda: dut.apply_events([{"type": "MODIFIED", "object": dict(p, metadata=dict(p["metadata"], labels=rand_labels(rng)))}
                                                   for p in rng.sample(list(w.pods.values()), 10)])),
        ("relabel pods", lambda: w.apply(*[dict(p, metadata=dict(p["metadata"], labels=rand_labels(rng))) for p in rng.sample(list(w.pods.values()), 15)])),
        ("bind queued pods", lambda: w.apply(*[dict(w.pods[k], spec=dict(w.pods[k]["spec"], nodeName="node-2"), status={"phase": "Running"})
                                              for k in queued()[:4]])),
        ("delete queued pods", lambda: [w.delete("Pod", k) for k in queued()[-4:]]),  # tombstone rows in the queue table
        ("new queued pods", lambda: w.apply(*[rand_pod(rng, rng.choice(nss), f"n{rng.randrange(10**6)}", False) for _ in range(8)])),
        ("new throttles", lambda: w.apply(*[rand_throttle(rng, 100 + rng.randrange(10**6), nss) for _ in range(40)])),  # more words
        ("edit a throttle", lambda: w.apply(dict(w.thr[w.order[1]], spec=dict(w.thr[w.order[1]]["spec"], threshold={"resourceCounts": {"pod": 1}})))),
        ("delete throttles", lambda: [w.delete(*w.order[i]) for i in (5, 3)]),  # columns handed out again, creation order
        ("re-create a throttle", lambda: w.apply(rand_throttle(rng, 3, nss))),
        ("relabel a namespace", lambda: w.apply(namespace("ns1", {"team": rng.choice(VALS), "env": rng.choice(VALS)}))),
        ("apply the missing namespace", lambda: w.apply(namespace("ns4", {"team": "a"}))),
        ("reconcile_all", lambda: dut.reconcile_all(NOW)),
    ]
    if has_prefilter_keys(dut):
        steps.insert(9, ("prefilter_keys", lambda: dut.prefilter_keys(queued()[:10])))
    for name, step in steps:
        step()
        check(w, f"after {name}")
    dut.close()


def test_report_leaves_every_other_answer_unchanged(new_plugin):
    """The same event stream with and without reports in between: every other call answers the same."""

    def stream(with_reports):
        rng = random.Random(11)
        w, nss = random_world(new_plugin(THROTTLER, SCHED), rng, n_thr=16, n_run=100, n_queue=40)
        dut, out = w.dut, []
        keys = [k for k in w.pods if dut.queue_row(*k.split("/", 1)) >= 0]
        calls = [lambda: dut.prefilter_key(*keys[0].split("/", 1)), lambda: dut.reserve_key(*keys[1].split("/", 1)),
                 lambda: [dut.status(k.split("/", 1)[1], k.split("/", 1)[0]) for (kind, k) in w.order if w.thr[(kind, k)]["spec"]["throttlerName"] == THROTTLER],
                 lambda: dut.prefilter_queue().tolist(), lambda: dut.reconcile_all(NOW), lambda: dut.metrics(),
                 lambda: [dut.reserved(kind, k) for (kind, k) in w.order],
                 lambda: dut.prefilter_keys(keys[:12]) if has_prefilter_keys(dut) else None,
                 lambda: dut.admit_queue([rand_pod(rng, "ns0", "m0", False)]), lambda: dut.reconcile_all(NOW)]
        for c in calls:
            if with_reports:
                dut.queue_report()
            out.append(c())
        stats = dut.queue_stats()
        dut.close()
        return out, {k: v for k, v in stats.items() if k not in ("passes", "hits")}

    assert stream(False) == stream(True)


def test_broken_selectors_error_pods_and_foreign_throttles(new_plugin):
    dut = new_plugin(THROTTLER, SCHED)
    w = World(dut)
    w.apply(namespace("default", {"team": "a"}), namespace("other", {"team": "b"}))
    mixed = {"kind": "Throttle", "metadata": {"namespace": "default", "name": "mixed"},
             "spec": {"throttlerName": THROTTLER, "threshold": {"resourceCounts": {"pod": 1}},
                      "selector": {"selectorTerms": [{"podSelector": {"matchLabels": {"a": "1"}}}, {"podSelector": BROKEN[0]}]}}}
    w.apply(mixed, throttle("default", "t1", {"a": "1"}, pod_cnt=1), throttle("default", "foreign", {"a": "1"}, pod_cnt=0, throttler="other-throttler"),
            throttle("other", "t2", {"b": "1"}, cpu="200m"))
    w.apply(pod("default", "run", "100m", {"a": "1"}, node="n", phase="Running"))
    dut.reconcile_all(NOW)
    # queued: one the valid term of `mixed` matches (no error), one that reaches the broken term (Error), one in an unknown
    # namespace (Error in the ClusterThrottle controller), and one that only t2 holds back
    w.apply(pod("default", "q0", "100m", {"a": "1"}), pod("default", "q1", "100m", {"c": "1"}), pod("nowhere", "q2", "300m", {"b": "1"}),
            pod("other", "q3", "300m", {"b": "1"}))
    got = check(w)
    assert [e["key"] for e in got["throttles"]] == ["default/mixed", "default/t1", "other/t2"]  # the foreign one is absent
    assert got["error"] == 2 and got["queued"] == 4
    by_key = {e["key"]: e for e in got["throttles"]}
    assert by_key["other/t2"]["onlyBlocker"] == 1 and by_key["other/t2"]["podRequestsExceedsThreshold"] == 1
    assert by_key["other/t2"]["heldBack"] == {"resourceCounts": {"pod": 1}, "resourceRequests": {"cpu": "0.3"}}
    assert by_key["default/mixed"]["onlyBlocker"] == 0  # q0 is held back by mixed and t1 together
    w.delete("Pod", "other/q3")  # its row stays behind as a tombstone
    got = check(w, "after a delete")
    assert {e["key"]: e["heldBack"] for e in got["throttles"]}["other/t2"] == {}
    dut.close()


def test_world_without_throttles_and_without_a_queue(new_plugin):
    dut = new_plugin(THROTTLER, SCHED)
    assert dut.queue_report() == {"queued": 0, "success": 0, "unschedulable": 0, "error": 0, "throttles": []}
    w = World(dut)
    w.apply(namespace("default"), pod("default", "q0", "100m", {"a": "1"}), pod("nowhere", "q1", "100m", {}))
    assert check(w) == {"queued": 2, "success": 1, "unschedulable": 0, "error": 1, "throttles": []}
    w.apply(throttle("default", "t", {"a": "1"}, pod_cnt=0))
    got = check(w, "one throttle")
    assert got["throttles"] == [{"key": "default/t", "kind": "Throttle", "active": 0, "insufficient": 0, "podRequestsExceedsThreshold": 1,
                                 "onlyBlocker": 1, "heldBack": {"resourceCounts": {"pod": 1}, "resourceRequests": {"cpu": "0.1"}}}]
    dut.close()


def test_report_device_cost(host_on_oracle_summary):
    """At most one pass per report, and none when the cached verdicts are current and the device's codes belong to a pass at this
    state: the last report's or kth_affected_pods'.  Any other call in between may have run a pass at another state, so the
    report runs its own even when every cached verdict is current."""
    import ctypes as C

    dut = host_on_oracle_summary(THROTTLER, SCHED)
    L = dut._L
    L.kt_test_device_calls.argtypes = [C.POINTER(C.c_int64)]
    L.kt_test_device_calls.restype = None

    def passes():
        out = (C.c_int64 * 2)()
        L.kt_test_device_calls(out)
        return out[1]

    def report_passes():
        before = passes()
        dut.queue_report()
        return passes() - before

    rng = random.Random(5)
    w, _ = random_world(dut, rng, n_thr=12, n_run=60, n_queue=30)
    report_passes()
    assert report_passes() == 0
    ours = [k for (kind, k) in w.order if w.thr[(kind, k)]["spec"]["throttlerName"] == THROTTLER]
    dut.affected_pods(ours[0].split("/", 1)[1], ours[0].split("/", 1)[0])
    assert report_passes() == 0
    dut.status(ours[0].split("/", 1)[1], ours[0].split("/", 1)[0])  # (the cached verdicts stay current)
    assert report_passes() == 1
    queued = [k for k in w.pods if dut.queue_row(*k.split("/", 1)) >= 0]
    dut.reserve_key(*queued[0].split("/", 1))  # voids cached verdicts: the refresh is the report's one pass
    assert report_passes() == 1
    check(w)
    dut.close()
