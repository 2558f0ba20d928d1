"""End-to-end decision vectors of the reference's integration suite and README walk-through, replayed on
BOTH implementations of the plugin surface through the same test bodies:
  [oracle]  the object-level ORACLE (plugin PreFilter/Reserve + both controllers), CPU only;
  [b200]    the PRODUCT: include/kt_host.h above the CUDA engine (marked gpu: every match, sum and compare
            of these scenarios runs in the sm_90a kernels, the host only packs and spells).

The integration suite needs Go + kind + a real kube-scheduler, none of which exist here; its scenarios
are deterministic decision sequences, so they are transcribed as golden vectors:
  test/integration/throttle_test.go:41-197, clusterthrottle_test.go:40-195,
  clusterthrottle_stress_test.go:33-86, README.md:230-374 (example/*.yaml).
"""
from fractions import Fraction

import pytest

from test_oracle_kat import q, rl_values

NOW = "2026-01-01T00:00:00Z"
SCHED = "my-scheduler"
THROTTLER = "kube-throttler"


def pod(ns, name, cpu=None, labels=None, node="", phase="Pending", requests=None, scheduler=SCHED):
    """util_pod_test.go:34-46 MakePod(ns, name, cpuReq).Label(k, v)"""
    reqs = dict(requests or {})
    if cpu is not None:
        reqs["cpu"] = cpu
    return {"kind": "Pod", "metadata": {"namespace": ns, "name": name, "labels": labels or {}},
            "spec": {"schedulerName": scheduler, "nodeName": node, "containers": [{"name": "c", "resources": {"requests": reqs}}]},
            "status": {"phase": phase}}


def throttle(ns, name, pod_sel, pod_cnt=None, cpu=None, extra=None, throttler=THROTTLER, overrides=None):
    """util_throttle_test.go:32-86 MakeThrottle(ns,name).PodSelector(k,v).ThresholdPod(n).ThresholdCpu(q)"""
    thr = {}
    if pod_cnt is not None:
        thr["resourceCounts"] = {"pod": pod_cnt}
    rr = dict(extra or {})
    if cpu is not None:
        rr["cpu"] = cpu
    if rr:
        thr["resourceRequests"] = rr
    spec = {"throttlerName": throttler, "threshold": thr, "selector": {"selectorTerms": [{"podSelector": {"matchLabels": pod_sel}}]}}
    if overrides:
        spec["temporaryThresholdOverrides"] = overrides
    return {"kind": "Throttle", "metadata": {"namespace": ns, "name": name}, "spec": spec}


def clthrottle(name, ns_sel, pod_sel, pod_cnt=None, cpu=None):
    """util_clusterthrottle_test.go:32-100 MakeClusterThrottle(name).Selectors(...)"""
    thr = {}
    if pod_cnt is not None:
        thr["resourceCounts"] = {"pod": pod_cnt}
    if cpu is not None:
        thr["resourceRequests"] = {"cpu": cpu}
    return {"kind": "ClusterThrottle", "metadata": {"name": name},
            "spec": {"throttlerName": THROTTLER, "threshold": thr,
                     "selector": {"selectorTerms": [{"namespaceSelector": {"matchLabels": ns_sel}, "podSelector": {"matchLabels": pod_sel}}]}}}


def namespace(name, labels=None):
    l = {"kubernetes.io/metadata.name": name}
    l.update(labels or {})
    return {"kind": "Namespace", "metadata": {"name": name, "labels": l}}


@pytest.fixture(params=["oracle", "host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def new_world(request, oracle):
    """Constructor of a plugin world: NewPlugin(name, targetSchedulerName) on the object-level oracle, on the product's HOST layer
    over an engine test double that evaluates with the columnar oracle (CPU: checks kt_host.cc, not the kernels), or on the
    product itself (GPU)."""
    if request.param == "oracle":
        return oracle.World
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle")
    from kube_throttler_b200 import host  # the product path: fails loudly without the CUDA library / a GPU

    return host.Plugin


class Cluster:
    """A miniature scheduler loop: PreFilter -> (Success) Reserve -> bind (nodeName set, pod informer
    sees it) -> reconcile.  Mirrors what the integration suite observes through the API server."""

    def __init__(self, new_world):
        self.w = new_world(THROTTLER, SCHED)
        self.w.apply(namespace("default"))

    def try_schedule(self, p):
        r = self.w.prefilter(p)
        if r["code"] != "Success":
            return r
        assert self.w.reserve(p)["code"] == "Success"
        bound = dict(p, spec=dict(p["spec"], nodeName="node-1"), status={"phase": "Running"})
        self.w.apply(bound)
        return r

    def settle(self):
        self.w.reconcile_all(NOW)

    def status(self, name, ns="default"):
        s = self.w.status(name, ns)
        return {"pod": s["used"].get("resourceCounts", {}).get("pod"),
                "cpu": q(s["used"].get("resourceRequests", {}).get("cpu", "0")),
                "podThrottled": s["throttled"]["resourceCounts"]["pod"],
                "cpuThrottled": s["throttled"].get("resourceRequests", {}).get("cpu")}


LBL = {"throttle": "test-throttle"}


@pytest.fixture
def cluster(new_world):
    return Cluster(new_world)


# ---- throttle_test.go:41-65 --------------------------------------------------------------------
def test_within_threshold(cluster):
    cluster.w.apply(throttle("default", "test-throttle", LBL, pod_cnt=2, cpu="1"))
    cluster.settle()
    assert cluster.try_schedule(pod("default", "pod", "500m", LBL))["code"] == "Success"
    cluster.settle()
    assert cluster.status("test-throttle") == {"pod": 1, "cpu": Fraction(1, 2), "podThrottled": False, "cpuThrottled": False}


# ---- throttle_test.go:77-101: count throttled -> active -----------------------------------------
def test_resource_count_active(cluster):
    cluster.w.apply(throttle("default", "test-throttle", LBL, pod_cnt=2, cpu="1"))
    cluster.settle()
    for i in (1, 2):
        assert cluster.try_schedule(pod("default", f"pod{i}", "100m", LBL))["code"] == "Success"
        cluster.settle()
    assert cluster.status("test-throttle") == {"pod": 2, "cpu": Fraction(1, 5), "podThrottled": True, "cpuThrottled": False}
    r = cluster.try_schedule(pod("default", "pod3", "100m", LBL))
    assert r["code"] == "UnschedulableAndUnresolvable"
    assert r["reasons"] == ["throttle[active]=default/test-throttle"]


# ---- throttle_test.go:102-123: request throttled -> active --------------------------------------
def test_resource_request_active(cluster):
    cluster.w.apply(throttle("default", "test-throttle", LBL, pod_cnt=2, cpu="1"))
    cluster.settle()
    assert cluster.try_schedule(pod("default", "pod1", "1", LBL))["code"] == "Success"
    cluster.settle()
    assert cluster.status("test-throttle") == {"pod": 1, "cpu": 1, "podThrottled": False, "cpuThrottled": True}
    r = cluster.try_schedule(pod("default", "pod2", "500m", LBL))
    assert r["reasons"] == ["throttle[active]=default/test-throttle"]


# ---- throttle_test.go:124-145: insufficient -----------------------------------------------------
def test_resource_request_insufficient(cluster):
    cluster.w.apply(throttle("default", "test-throttle", LBL, pod_cnt=2, cpu="1"))
    cluster.settle()
    assert cluster.try_schedule(pod("default", "pod1", "900m", LBL))["code"] == "Success"
    cluster.settle()
    assert cluster.status("test-throttle") == {"pod": 1, "cpu": Fraction(9, 10), "podThrottled": False, "cpuThrottled": False}
    r = cluster.try_schedule(pod("default", "pod2", "500m", LBL))
    assert r["reasons"] == ["throttle[insufficient]=default/test-throttle"]


# ---- throttle_test.go:146-164: pod-requests-exceeds-threshold + event ----------------------------
def test_pod_requests_exceeds_threshold(cluster):
    cluster.w.apply(throttle("default", "test-throttle", LBL, pod_cnt=2, cpu="1"))
    cluster.settle()
    r = cluster.try_schedule(pod("default", "pod", "1.1", LBL))
    assert r["code"] == "UnschedulableAndUnresolvable"
    assert r["reasons"] == ["throttle[pod-requests-exceeds-threshold]=default/test-throttle"]
    assert r["event"]["reason"] == "ResourceRequestsExceedsThrottleThreshold" and r["event"]["type"] == "Warning"
    assert r["event"]["message"].endswith("resource requests exceeds their thresholds: default/test-throttle")
    s = cluster.status("test-throttle")
    assert s["podThrottled"] is False and s["cpuThrottled"] is False


# ---- throttle_test.go:167-197: 20 x 50m exactly fills cpu=1; the 21st is `active` (Q2) -----------
@pytest.mark.parametrize("reconcile_between", [True, False])
def test_many_pods_at_once(cluster, reconcile_between):
    cluster.w.apply(throttle("default", "test-throttle", LBL, cpu="1"))
    cluster.settle()
    for i in range(20):
        # without reconciles the reservation cache alone must carry the admitted amounts (S4 uses `>`)
        assert cluster.try_schedule(pod("default", f"pod-{i}", "50m", LBL))["code"] == "Success", i
        if reconcile_between:
            cluster.settle()
    if not reconcile_between:
        # 20 reserved, none observed: used+reserved == threshold -> step 3 (onEqual=true for Throttle) says active
        r = cluster.w.prefilter(pod("default", "pod-20", "50m", LBL))
        assert r["reasons"] == ["throttle[active]=default/test-throttle"]
    cluster.settle()
    assert cluster.status("test-throttle") == {"pod": 20, "cpu": 1, "podThrottled": False, "cpuThrottled": True}
    assert cluster.w.reserved("Throttle", "default/test-throttle")["pods"] == []  # reconcile un-reserves observed pods
    r = cluster.try_schedule(pod("default", "pod-20", "50m", LBL))
    assert r["reasons"] == ["throttle[active]=default/test-throttle"]


# ---- clusterthrottle_test.go twins (ns selector kubernetes.io/metadata.name=default) --------------
CL_NS = {"kubernetes.io/metadata.name": "default"}


def test_clusterthrottle_twins(cluster):
    cluster.w.apply(clthrottle("test-clthr", CL_NS, LBL, pod_cnt=2, cpu="1"))
    cluster.settle()
    assert cluster.try_schedule(pod("default", "pod1", "900m", LBL))["code"] == "Success"
    cluster.settle()
    s = cluster.status("test-clthr", "")
    assert s == {"pod": 1, "cpu": Fraction(9, 10), "podThrottled": False, "cpuThrottled": False}
    r = cluster.try_schedule(pod("default", "pod2", "500m", LBL))
    assert r["reasons"] == ["clusterthrottle[insufficient]=/test-clthr"]  # ClusterThrottle prints "/name" (plugin.go:289-294)
    r = cluster.try_schedule(pod("default", "big", "1.1", LBL))
    assert r["reasons"] == ["clusterthrottle[pod-requests-exceeds-threshold]=/test-clthr"]
    assert r["event"]["message"].endswith(": /test-clthr")
    # a pod in a namespace the selector does not cover is unaffected
    cluster.w.apply(namespace("other"))
    assert cluster.try_schedule(pod("other", "free", "10", LBL))["code"] == "Success"


def test_q1_step3_asymmetry(cluster):
    """used+reserved == threshold: Throttle -> active (S3 onEqual hard-coded true, throttle_types.go:143),
    ClusterThrottle -> insufficient (S3 uses PreFilter's false, clusterthrottle_types.go:45).

    The stale status (used observed, throttled flag not yet recomputed) is what PreFilter sees between the
    pod event and the next reconcile; at reconcile time S2 would say `active` for both kinds."""
    cluster.w.apply(throttle("default", "thr", LBL, cpu="1"), clthrottle("clthr", CL_NS, LBL, cpu="1"))
    stale = {"calculatedThreshold": {"threshold": {"resourceRequests": {"cpu": "1"}}, "calculatedAt": NOW},
             "used": {"resourceCounts": {"pod": 1}, "resourceRequests": {"cpu": "1"}},
             "throttled": {"resourceCounts": {"pod": False}, "resourceRequests": {"cpu": False}}}
    t = throttle("default", "thr", LBL, cpu="1")
    t["status"] = stale
    c = clthrottle("clthr", CL_NS, LBL, cpu="1")
    c["status"] = stale
    cluster.w.apply(t, c)
    r = cluster.w.prefilter(pod("default", "p", "100m", LBL))
    assert r["reasons"] == ["throttle[active]=default/thr", "clusterthrottle[insufficient]=/clthr"] or \
        r["reasons"] == ["clusterthrottle[insufficient]=/clthr", "throttle[active]=default/thr"]
    assert r["throttle"]["active"] == ["default/thr"] and r["clusterthrottle"]["insufficient"] == ["/clthr"]


# ---- clusterthrottle_stress_test.go:33-86 --------------------------------------------------------
def test_clusterthrottle_stress(new_world):
    w = new_world(THROTTLER, SCHED)
    n_clthr, n_ns, n_pods = 50, 10, 10
    for i in range(n_clthr):
        w.apply(clthrottle(f"clthr-{i}", {"targetns": "true"}, {"clthr-target": "true"}, pod_cnt=n_ns * n_pods, cpu=f"{n_ns * n_pods}m"))
    w.reconcile_all(NOW)
    for i in range(n_ns):
        w.apply(namespace(f"ns-{i}", {"targetns": "true"}))
        for j in range(n_pods):
            p = pod(f"ns-{i}", f"pod-{j}", "1m", {"clthr-target": "true"})
            r = w.prefilter(p)
            assert r["code"] == "Success", (i, j, r)
            w.reserve(p)
            w.apply(dict(p, spec=dict(p["spec"], nodeName="n"), status={"phase": "Running"}))
    w.reconcile_all(NOW)
    for i in range(n_clthr):
        s = w.status(f"clthr-{i}")
        assert s["used"]["resourceCounts"]["pod"] == 100 and q(s["used"]["resourceRequests"]["cpu"]) == Fraction(1, 10)
        assert s["throttled"] == {"resourceCounts": {"pod": True}, "resourceRequests": {"cpu": True}}
    r = w.prefilter(pod("ns-0", "late", "1m", {"clthr-target": "true"}))
    assert r["code"] == "UnschedulableAndUnresolvable" and len(r["clusterthrottle"]["active"]) == n_clthr


# ---- README.md:230-374 walk-through with example/*.yaml -------------------------------------------
def test_readme_walkthrough(cluster):
    T1 = {"throttle": "t1"}
    cluster.w.apply(throttle("default", "t1", T1, pod_cnt=5, cpu="200m", extra={"memory": "1Gi"}))
    cluster.settle()
    assert cluster.try_schedule(pod("default", "pod1", "200m", T1))["code"] == "Success"
    cluster.settle()
    s = cluster.w.status("t1", "default")
    assert s["throttled"]["resourceRequests"] == {"cpu": True, "memory": False}
    # README.md:284 says pod2 (300m vs cpu=200m) is "active"; by code it is S1 pod-requests-exceeds-threshold
    r = cluster.try_schedule(pod("default", "pod2", "300m", T1))
    assert r["reasons"] == ["throttle[pod-requests-exceeds-threshold]=default/t1"]
    # pod1m asks only for memory: admitted while cpu is throttled (README.md:287-309)
    assert cluster.try_schedule(pod("default", "pod1m", None, T1, requests={"memory": "512Mi"}))["code"] == "Success"
    cluster.settle()
    s = cluster.w.status("t1", "default")
    assert s["used"]["resourceCounts"]["pod"] == 2
    assert rl_values(s["used"]["resourceRequests"]) == {"cpu": Fraction(1, 5), "memory": 536870912}
    # threshold cpu 200m -> 700m: pod2 fits, pod3 (300m) is insufficient (README.md:311-374)
    cluster.w.apply(throttle("default", "t1", T1, pod_cnt=5, cpu="700m", extra={"memory": "1Gi"}))
    cluster.settle()
    assert cluster.try_schedule(pod("default", "pod2", "300m", T1))["code"] == "Success"
    cluster.settle()
    assert cluster.w.status("t1", "default")["throttled"]["resourceRequests"] == {"cpu": False, "memory": False}
    r = cluster.try_schedule(pod("default", "pod3", "300m", T1))
    assert r["reasons"] == ["throttle[insufficient]=default/t1"]


# ---- quirks ---------------------------------------------------------------------------------------
def test_q3_zero_pods_never_count_throttled(cluster):
    """threshold pod:0 with no matched pods: used.Counts is nil -> status.throttled.pod stays false (Q3),
    yet every matching pod is pod-requests-exceeds-threshold by S1 (1 > 0, Q4)."""
    cluster.w.apply(throttle("default", "t", LBL, pod_cnt=0))
    cluster.settle()
    assert cluster.w.status("t", "default")["throttled"]["resourceCounts"]["pod"] is False
    r = cluster.w.prefilter(pod("default", "p", "1m", LBL))
    assert r["reasons"] == ["throttle[pod-requests-exceeds-threshold]=default/t"]


def test_q10_reason_order(cluster):
    """plugin.go:182-213: clthr[exceeds], thr[exceeds], clthr[active], thr[active], clthr[insufficient], thr[insufficient]"""
    A, B, C = {"a": "1"}, {"b": "1"}, {"c": "1"}
    all_l = {**A, **B, **C}
    cluster.w.apply(
        throttle("default", "t-exceeds", A, cpu="100m"), clthrottle("c-exceeds", CL_NS, A, cpu="100m"),
        throttle("default", "t-insuff", C, cpu="1200m"), clthrottle("c-insuff", CL_NS, C, cpu="1200m"),
        throttle("default", "t-active", B, pod_cnt=1), clthrottle("c-active", CL_NS, B, pod_cnt=1),
    )
    cluster.settle()
    assert cluster.try_schedule(pod("default", "filler-b", "1m", B))["code"] == "Success"
    assert cluster.try_schedule(pod("default", "filler-c", "1", C))["code"] == "Success"
    cluster.settle()
    r = cluster.w.prefilter(pod("default", "p", "500m", all_l))
    assert r["code"] == "UnschedulableAndUnresolvable"
    assert r["reasons"] == [
        "clusterthrottle[pod-requests-exceeds-threshold]=/c-exceeds", "throttle[pod-requests-exceeds-threshold]=default/t-exceeds",
        "clusterthrottle[active]=/c-active", "throttle[active]=default/t-active",
        "clusterthrottle[insufficient]=/c-insuff", "throttle[insufficient]=default/t-insuff"]
    assert r["event"]["message"].endswith(": /c-exceeds,default/t-exceeds")


def test_not_responsible_and_other_scheduler(cluster):
    cluster.w.apply(throttle("default", "foreign", LBL, pod_cnt=0, throttler="someone-else"), throttle("default", "ours", LBL, cpu="1"))
    cluster.settle()
    assert cluster.w.prefilter(pod("default", "p", "1m", LBL))["code"] == "Success"  # foreign throttle ignored
    # a running pod of another scheduler is not counted (shouldCountIn)
    cluster.w.apply(pod("default", "alien", "900m", LBL, node="n", phase="Running", scheduler="default-scheduler"))
    cluster.w.apply(pod("default", "done", "900m", LBL, node="n", phase="Succeeded"))
    cluster.w.apply(pod("default", "unbound", "900m", LBL, node="", phase="Pending"))
    cluster.settle()
    assert cluster.status("ours")["pod"] is None and cluster.status("ours")["cpu"] == 0


def test_override_replaces_threshold_in_check(cluster):
    """An active override replaces the whole threshold (Q7): the spec's pod:1 limit disappears."""
    ovr = [{"begin": "2025-12-01T00:00:00Z", "end": "2026-02-01T00:00:00Z", "threshold": {"resourceRequests": {"cpu": "5"}}}]
    cluster.w.apply(throttle("default", "t", LBL, pod_cnt=1, cpu="200m", overrides=ovr))
    cluster.settle()
    for i in range(3):
        assert cluster.try_schedule(pod("default", f"p{i}", "1", LBL))["code"] == "Success"
        cluster.settle()
    s = cluster.w.status("t", "default")
    assert s["calculatedThreshold"]["threshold"] == {"resourceRequests": {"cpu": "5"}}
    assert s["throttled"] == {"resourceCounts": {"pod": False}, "resourceRequests": {"cpu": False}}


def test_missing_namespace_is_an_error(new_world):
    w = new_world(THROTTLER, SCHED)
    w.apply(clthrottle("c", {}, LBL, cpu="1"))
    r = w.prefilter(pod("ghost", "p", "1m", LBL))
    assert r["code"] == "Error" and "not found" in r["reasons"][0]


def test_reserve_unreserve_roundtrip(cluster):
    cluster.w.apply(throttle("default", "t", LBL, cpu="1"), clthrottle("c", CL_NS, LBL, cpu="1"))
    cluster.settle()
    p = pod("default", "p", "600m", LBL)
    assert cluster.w.prefilter(p)["code"] == "Success"
    cluster.w.reserve(p)
    assert cluster.w.reserved("Throttle", "default/t")["pods"] == ["default/p"]
    assert cluster.w.reserved("ClusterThrottle", "/c")["pods"] == ["default/p"]
    assert q(cluster.w.reserved("Throttle", "default/t")["amount"]["resourceRequests"]["cpu"]) == Fraction(3, 5)
    p2 = pod("default", "p2", "600m", LBL)
    assert cluster.w.prefilter(p2)["code"] == "UnschedulableAndUnresolvable"  # 600m reserved + 600m > 1
    cluster.w.unreserve(p)
    assert cluster.w.reserved("Throttle", "default/t")["pods"] == []
    assert cluster.w.prefilter(p2)["code"] == "Success"
