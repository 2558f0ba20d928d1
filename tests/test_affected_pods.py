"""kth_affected_pods: the pods a throttle counts and the queued pods it holds back, read from the device's relations.

Compared with the object-level oracle on the random worlds of test_plugin_vs_oracle.  affectedPods (throttle_controller.go:221-246,
clusterthrottle_controller.go:224-270) is the counted pods whose affected throttles include the throttle, so the oracle's answer
is its PreFilter breakdown (affectedThrottles) of every counted pod, inverted; an affectedPods error is what the oracle's
reconcile of the throttle returns.  The queued pods' statuses are compared with PreFilter by key.  Runs on the product (GPU)
and on the product's host layer over the engine test double that evaluates with the columnar oracle (CPU)."""
import os
import random
import subprocess

import pytest

from test_plugin_vs_oracle import VALS, rand_labels, rand_pod, rand_throttle
from test_scenarios import NOW, SCHED, THROTTLER, namespace, pod, throttle


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host_on_oracle_columns(oracle):
    """kt_host.cc linked against the oracle-backed engine test double plus its kt_get_match_columns
    (tests/host_stub/engine_oracle_columns.cc); host.Plugin's signature.  CPU only; says nothing about the kernels."""
    import ctypes
    import functools

    from kube_throttler_b200 import host

    out = os.path.join(ROOT, "tests", "_build", "libkt_hostoracle_columns.so")
    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(ROOT, "tests", "host_stub", "engine_oracle_columns.cc")]
    deps = srcs + [os.path.join(ROOT, "tests", "host_stub", "engine_oracle.cc")] + \
        [os.path.join(ROOT, "kube_throttler_b200", "csrc", f) for f in ("kt_json.h", "kt_quantity.h")] + \
        [os.path.join(ROOT, "include", f) for f in ("kt_b200.h", "kt_host.h")] + [os.path.join(ROOT, "oracle", "libkt_oracle.so")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(f) for f in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        tmp = out + f".{os.getpid()}.tmp"
        subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-o", tmp] + srcs +
                       ["-L", os.path.join(ROOT, "oracle"), "-lkt_oracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")], check=True)
        os.replace(tmp, out)
    return functools.partial(host.Plugin, library=ctypes.CDLL(out))


@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def new_plugin(request):
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle_columns")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin


def pod_nn(p):
    return p["metadata"]["namespace"] + "/" + p["metadata"]["name"]


def oracle_affected_pods(ref, running):
    """{throttle nn: (non-terminated, terminated)} from the oracle's affectedThrottles of every counted pod (shouldCountIn:
    our scheduler, bound).  PreFilter computes the Throttle half before the ClusterThrottle half, so a pod of a namespace the
    lister does not hold still has its Throttle breakdown, and affects no ClusterThrottle."""
    out = {}
    for p in running:
        if p["spec"]["schedulerName"] != SCHED or not p["spec"]["nodeName"]:
            continue
        r = ref.prefilter(p)
        assert r["code"] != "Error" or "not found" in r["reasons"][0], r  # (the random worlds have no broken selectors)
        finished = p["status"]["phase"] in ("Succeeded", "Failed")
        for ctl in ("throttle", "clusterthrottle"):
            if ctl == "clusterthrottle" and r["code"] == "Error":
                continue
            for nn in r[ctl]["affected"]:
                out.setdefault((ctl, nn), ([], []))[finished].append(pod_nn(p))
    return out


BUCKETS = (("active", "active"), ("insufficient", "insufficient"), ("podRequestsExceedsThreshold", "pod-requests-exceeds-threshold"))


def by_key(names):
    return sorted(names, key=lambda s: tuple(s.split("/", 1)))


def ident(t):
    return t["metadata"]["name"], t["metadata"].get("namespace", "")


def nn_of(t):
    return t["metadata"].get("namespace", "") + "/" + t["metadata"]["name"]


def expected_queued(ref, dut, thr, pods):
    """{pod: status} of the queued pods whose PreFilter lists thr among the affected throttles of its kind, and the queued pods
    whose PreFilter fails on a broken podSelector (no per-throttle answer to compare with).  The statuses are the oracle's
    breakdown, which PreFilter by key must agree with; a pod of a namespace the lister does not hold fails in the ClusterThrottle
    controller only, after the Throttle controller answered."""
    ctl = "throttle" if thr["kind"] == "Throttle" else "clusterthrottle"
    want, unknown = {}, set()
    for p in pods:
        key = (p["metadata"]["namespace"], p["metadata"]["name"])
        if dut.queue_row(*key) < 0:
            continue
        r, by_key_r = ref.prefilter(p), dut.prefilter_key(*key)
        assert (by_key_r["code"], by_key_r["reasons"]) == (r["code"], r["reasons"]), key
        if r["code"] == "Error" and not (ctl == "throttle" and "not found" in r["reasons"][0]):
            unknown.add("/".join(key))
            continue
        if nn_of(thr) not in r[ctl]["affected"]:
            continue
        status = "not-throttled"
        for field, name in BUCKETS:
            if nn_of(thr) in r[ctl][field]:
                status = name
        want["/".join(key)] = status
    return want, unknown


def compare_all(ref, dut, throttles, running, queue):
    """affected_pods of every throttle == the oracle's affectedPods; queued statuses == PreFilter by key."""
    answered = 0
    want_all = oracle_affected_pods(ref, running)
    for t in throttles:
        name, ns = ident(t)
        if t["spec"]["throttlerName"] != THROTTLER:
            with pytest.raises(RuntimeError, match="belongs to throttler"):
                dut.affected_pods(name, ns)
            continue
        got = dut.affected_pods(name, ns)
        answered += 1
        pods, terminated = want_all.get(("throttle" if t["kind"] == "Throttle" else "clusterthrottle", nn_of(t)), ([], []))
        assert got["pods"] == by_key(pods), nn_of(t)
        assert got["terminatedPods"] == by_key(terminated), nn_of(t)
        q, unknown = expected_queued(ref, dut, t, running + queue)  # (a "running" pod without a node is queued too)
        listed = [e["pod"] for e in got["queued"]]
        assert listed == by_key(listed)
        assert {e["pod"]: e["status"] for e in got["queued"] if e["pod"] not in unknown} == q, nn_of(t)
    return answered


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_world(oracle, new_plugin, seed):
    rng = random.Random(seed)
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    nss = [f"ns{i}" for i in range(5)]
    for n in nss[:4]:  # ns4 is never applied: a namespace the lister does not hold
        both(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
    throttles = [rand_throttle(rng, i, nss) for i in range(40)]
    both(*throttles)
    running = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(300)]
    both(*running)
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(80)]
    both(*queue)  # delivered by the informer: the resident scheduling queue
    assert compare_all(ref, dut, throttles, running, queue) > 20
    stats = [dut.affected_pods(*ident(t)) for t in throttles[:5] if t["spec"]["throttlerName"] == THROTTLER]
    assert any(s["pods"] for s in stats) or any(s["queued"] for s in stats)
    # reservations, a reconcile, relabelled and finished pods, then once more
    for p in queue[:30]:
        key = (p["metadata"]["namespace"], p["metadata"]["name"])
        if dut.queue_row(*key) >= 0 and ref.prefilter(p)["code"] == "Success":
            assert ref.reserve(p)["code"] == dut.reserve_key(*key)["code"] == "Success"
    for p in rng.sample(running, 30):
        p["metadata"]["labels"] = rand_labels(rng)
        if rng.random() < 0.3:
            p["status"] = {"phase": "Succeeded"}
        both(p)
    compare_all(ref, dut, throttles, running, queue)
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    compare_all(ref, dut, throttles, running, queue)
    dut.close()


def test_selector_errors_and_unknown_throttles(oracle, new_plugin):
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    bad = {"matchExpressions": [{"key": "a", "operator": "Exists", "values": ["x"]}]}
    mixed = {"kind": "Throttle", "metadata": {"namespace": "default", "name": "mixed"},
             "spec": {"throttlerName": THROTTLER, "threshold": {"resourceCounts": {"pod": 2}},
                      "selector": {"selectorTerms": [{"podSelector": {"matchLabels": {"a": "1"}}}, {"podSelector": bad}]}}}
    both(namespace("default"), mixed, throttle("default", "foreign", {"a": "1"}, pod_cnt=1, throttler="other-throttler"))
    both(pod("default", "p0", "100m", {"a": "1"}, node="n", phase="Running"))
    assert dut.affected_pods("mixed", "default") == {"pods": ["default/p0"], "terminatedPods": [], "queued": []}
    both(pod("default", "p1", "100m", {"b": "1"}, node="n", phase="Running"))  # reaches the broken term
    with pytest.raises(RuntimeError) as want:  # the only throttle of the world whose reconcile can fail: its affectedPods error
        ref.reconcile_all(NOW)
    with pytest.raises(RuntimeError) as got:
        dut.affected_pods("mixed", "default")
    assert str(got.value) == str(want.value)
    with pytest.raises(RuntimeError, match="not found"):
        dut.affected_pods("nobody", "default")
    with pytest.raises(RuntimeError, match="not found"):
        dut.affected_pods("mixed")  # no ClusterThrottle of that name
    with pytest.raises(RuntimeError, match="belongs to throttler"):
        dut.affected_pods("foreign", "default")
    dut.close()


def test_clusterthrottle_selector_error_is_scoped_by_its_namespace_selector(oracle, new_plugin):
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    bad = {"matchExpressions": [{"key": "a", "operator": "In", "values": []}]}
    team_a = {"matchLabels": {"team": "a"}}
    ct = {"kind": "ClusterThrottle", "metadata": {"name": "ct"},
          "spec": {"throttlerName": THROTTLER, "threshold": {"resourceCounts": {"pod": 5}},
                   "selector": {"selectorTerms": [{"namespaceSelector": team_a, "podSelector": {"matchLabels": {"x": "1"}}},
                                                  {"namespaceSelector": team_a, "podSelector": bad}]}}}
    both(namespace("na", {"team": "a"}), namespace("nb", {"team": "b"}), ct)
    both(pod("na", "p0", "100m", {"x": "1"}, node="n", phase="Running"), pod("nb", "p1", "100m", {"y": "1"}, node="n", phase="Running"))
    ref.reconcile_all(NOW)  # nobody reaches the broken term: no error
    assert dut.affected_pods("ct") == {"pods": ["na/p0"], "terminatedPods": [], "queued": []}
    both(pod("na", "p2", "100m", {"y": "1"}, node="n", phase="Failed"))  # a counted pod of a team-a namespace reaches it
    with pytest.raises(RuntimeError) as want:
        ref.reconcile_all(NOW)
    with pytest.raises(RuntimeError) as got:
        dut.affected_pods("ct")
    assert str(got.value) == str(want.value)
    dut.close()


def test_two_running_pods_and_one_queued_active(oracle, new_plugin):
    """throttle_test.go (2): a pod-count threshold of 2 filled by two running pods; the third pod waits, throttled [active]."""
    dut = new_plugin(THROTTLER, SCHED)
    lbl = {"throttle": "t1"}
    dut.apply(namespace("default"), throttle("default", "t1", lbl, pod_cnt=2),
              pod("default", "pod-1", "100m", lbl, node="n", phase="Running"), pod("default", "pod-2", "100m", lbl, node="n", phase="Running"),
              pod("default", "done", "100m", lbl, node="n", phase="Succeeded"), pod("default", "other", "100m", {"x": "y"}, node="n", phase="Running"))
    dut.reconcile_all(NOW)
    dut.apply(pod("default", "pod-3", "100m", lbl))
    assert dut.prefilter_key("default", "pod-3")["reasons"] == ["throttle[active]=default/t1"]
    assert dut.affected_pods("t1", "default") == {"pods": ["default/pod-1", "default/pod-2"], "terminatedPods": ["default/done"],
                                                  "queued": [{"pod": "default/pod-3", "status": "active"}]}
    dut.close()


def run_stream(new_plugin, seed, probe):
    """One event stream; `probe` is called between the steps.  Returns every output of the stream's own calls."""
    rng = random.Random(seed)
    dut = new_plugin(THROTTLER, SCHED)
    out = []
    nss = [f"ns{i}" for i in range(3)]
    throttles = [rand_throttle(rng, i, nss) for i in range(12)]
    steps = [lambda: [dut.apply(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)})) for n in nss],
             lambda: [dut.apply(t) for t in throttles]]
    running = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(80)]
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(30)]
    keys = [(p["metadata"]["namespace"], p["metadata"]["name"]) for p in queue]
    steps += [lambda: [dut.apply(p) for p in running], lambda: dut.reconcile_all(NOW), lambda: [dut.apply(p) for p in queue],
              lambda: [dut.prefilter_key(*k) for k in keys]]
    steps += [lambda k=k: (dut.prefilter_key(*k), dut.reserve_key(*k)) for k in keys[:8]]
    steps += [lambda: dut.prefilter_queue().tolist(), lambda: dut.reconcile_all(NOW), lambda: [dut.prefilter_key(*k) for k in keys],
              lambda: dut.unreserve_key(*keys[0]), lambda: dut.prefilter(queue[3]), lambda: dut.queue_stats(), lambda: dut.metrics()]
    steps += [lambda: [dut.status(*ident(t)) for t in throttles if t["spec"]["throttlerName"] == THROTTLER],
              lambda: [dut.reserved(t["kind"], nn_of(t)) for t in throttles]]
    for step in steps:
        out.append(step())
        probe(dut, throttles)
    dut.close()
    return out


@pytest.mark.parametrize("seed", [0, 1])
def test_calls_leave_every_other_result_unchanged(new_plugin, seed):
    def ask(dut, throttles):
        for t in throttles:
            if t["spec"]["throttlerName"] == THROTTLER:
                try:
                    dut.affected_pods(*ident(t))
                except RuntimeError:
                    pass

    assert run_stream(new_plugin, seed, lambda dut, thr: None) == run_stream(new_plugin, seed, ask)
