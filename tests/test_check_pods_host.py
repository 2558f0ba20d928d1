"""Manifest PreFilter, Reserve and Unreserve, the reservation move of a pod update, the un-reservation of a pod delete,
kth_pre_filter_batch and the host-orchestrated rounds of kth_admit_queue check their pods with one kt_check_pods call each: the
cost follows the pods' namespaces, with no scratch row uploaded and no pass over the scheduling queue.

Random event streams and scheduling cycles run on three parties fed the same events: the plugin under test, a twin whose engine
double has no kt_check_pods (so it keeps the scratch-row pass), and the object-level oracle.  After every step the plugin must
return exactly what the twin returns (results, warnings, errors, round counts, statuses, reservations, gauges, PreFilter by key)
and agree with the oracle; kth_queue_stats' passes and hits may only be lower.  For informer-held pods, PreFilter by key must
equal the entry kth_pre_filter_keys gives.  On the engine double that counts its calls (CPU) a manifest PreFilter, Reserve or
Unreserve makes one kt_check_pods call and no kt_evaluate and no pending-row upload."""
import ctypes as C
import functools
import os
import random

import pytest

from test_plugin_vs_oracle import VALS, norm_amount, norm_prefilter, norm_status, rand_labels, rand_pod, rand_throttle
from test_prefilter_keys import host_on_oracle_check_rows  # noqa: F401 (fixture)
from test_reconcile_keys import BROKEN, _build
from test_scenarios import NOW, SCHED, THROTTLER, namespace, pod, throttle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUB = os.path.join(ROOT, "tests", "host_stub")
CALLS = ("check_pods", "evaluate", "pending_uploads")


@pytest.fixture(scope="module")
def host_on_oracle_check_pods(oracle):
    """kt_host.cc linked against the oracle-backed engine test double with kt_check_pods and call counters
    (tests/host_stub/engine_oracle_check_pods.cc); host.Plugin's signature plus `.calls()`."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_check_pods.cc")]
    deps = [os.path.join(STUB, f) for f in ("engine_oracle.cc", "engine_oracle_check_rows.cc")] + [os.path.join(ROOT, "oracle", "libkt_oracle.so")] + \
        [os.path.join(ROOT, "kube_throttler_b200", "csrc", f) for f in ("kt_json.h", "kt_quantity.h")] + \
        [os.path.join(ROOT, "include", f) for f in ("kt_b200.h", "kt_host.h")]
    lib = _build("libkt_hostoracle_check_pods.so", srcs, deps,
                 ["-L", os.path.join(ROOT, "oracle"), "-lkt_oracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    lib.kt_test_check_pods_calls.argtypes = [C.POINTER(C.c_int64)]
    lib.kt_test_check_pods_calls.restype = None

    def calls():
        out = (C.c_int64 * len(CALLS))()
        lib.kt_test_check_pods_calls(out)
        return dict(zip(CALLS, out))

    make = functools.partial(host.Plugin, library=lib)
    make.calls = calls
    return make


@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def new_plugin(request):
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle_check_pods")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin


def nn(p):
    return p["metadata"]["namespace"] + "/" + p["metadata"]["name"]


def outcome(f, *args):
    """A call's result, or its error text (both parties must fail alike)."""
    try:
        return f(*args)
    except RuntimeError as e:
        return {"error": str(e)}


class Three:
    """The plugin under test, the scratch-row twin and the object oracle, driven by the same events."""

    def __init__(self, ref, dut, twin):
        self.ref, self.dut, self.twin = ref, dut, twin
        self.throttles = {}

    def same(self, name, *args, oracle=True):
        a = outcome(getattr(self.dut, name), *args)
        b = outcome(getattr(self.twin, name), *args)
        assert a == b, (name, args, a, b)
        if oracle and name in ("prefilter", "reserve", "unreserve"):
            want = getattr(self.ref, name)(*args)
            if name == "prefilter":
                assert norm_prefilter(a) == norm_prefilter(want), (args, a, want)
            elif name == "reserve":  # (the oracle's Unreserve returns nothing; the reservations are compared afterwards)
                assert a["code"] == want["code"], (name, args, a, want)
        return a

    def apply(self, *ms):
        for m in ms:
            self.ref.apply(m)
            self.same("apply", m, oracle=False)
            if m["kind"] in ("Throttle", "ClusterThrottle"):
                self.throttles[(m["kind"], m["metadata"].get("namespace", "") + "/" + m["metadata"]["name"])] = m

    def delete(self, kind, name, ns=""):
        self.ref.delete(kind, name, ns)
        self.same("delete", kind, name, ns, oracle=False)

    def compare(self, queue, held, where):
        for (kind, key) in self.throttles:
            ns, _, name = key.partition("/")
            a, b = self.dut.status(name, ns), self.twin.status(name, ns)
            assert a == b, (where, key)
            assert norm_status(a) == norm_status(self.ref.status(name, ns)), (where, key)
            a, b, c = self.dut.reserved(kind, key), self.twin.reserved(kind, key), self.ref.reserved(kind, key)
            assert a == b, (where, key, a, b)
            assert sorted(a["pods"]) == sorted(c["pods"]) and norm_amount(a["amount"]) == norm_amount(c["amount"]), (where, key, a, c)
        for p in queue:
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if self.dut.queue_row(*k) >= 0:
                self.same("prefilter_key", *k, oracle=False)
        # informer-held pods that are not queued are checked like manifests: the same entry kth_pre_filter_keys gives
        keys = [nn(p) for p in held]
        if keys:
            listed = self.same("prefilter_keys", keys, oracle=False)
            for key, entry in zip(keys, listed):
                ns, _, name = key.partition("/")
                assert self.same("prefilter_key", ns, name, oracle=False) == entry, (where, key)
        assert self.dut.metrics() == self.twin.metrics(), where
        a, b = self.dut.queue_stats(), self.twin.queue_stats()
        assert a["passes"] <= b["passes"] and a["hits"] <= b["hits"], (where, a, b)
        assert {k: v for k, v in a.items() if k not in ("passes", "hits")} == {k: v for k, v in b.items() if k not in ("passes", "hits")}, (where, a, b)


def run_stream(oracle, new_plugin, twin_plugin, seed, steps=70, n_thr=16, n_ns=4, broken=False):
    rng = random.Random(seed)
    w = Three(oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED), twin_plugin(THROTTLER, SCHED))
    nss = [f"ns{i}" for i in range(n_ns)]
    w.apply(*[namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}) for n in nss])
    throttles = [rand_throttle(rng, i, nss) for i in range(n_thr)]
    if broken:  # a podSelector that does not convert: PreFilter answers Error, and admit_queue takes the host rounds
        throttles[0] = dict(throttles[0], spec=dict(throttles[0]["spec"], selector={"selectorTerms": [{"podSelector": BROKEN}]}))
    w.apply(*throttles)
    running = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(40)]
    w.apply(*running)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(20)]
    w.apply(*queue)
    w.ref.reconcile_all(NOW)
    w.same("reconcile_all", NOW, oracle=False)
    manifests = [rand_pod(rng, rng.choice(nss), f"m{i}", False) for i in range(30)]
    reserved, seen = [], set()
    for step in range(steps):
        op = rng.random()
        where = (seed, step)
        if op < 0.2:  # the scheduling cycle of a manifest: PreFilter, Reserve on Success
            p = rng.choice(manifests)
            r = w.same("prefilter", p)
            seen.add(r["code"])
            if r["code"] == "Success" and rng.random() < 0.7:
                w.same("reserve", p)
                reserved.append(p)
                seen.add("reserve")
        elif op < 0.27 and reserved:  # Unreserve
            w.same("unreserve", reserved.pop(rng.randrange(len(reserved))))
            seen.add("unreserve")
        elif op < 0.37:  # a reserved pod is bound: the informer sees it
            if reserved:
                p = reserved.pop(rng.randrange(len(reserved)))
                if p in manifests:
                    manifests.remove(p)
                p = dict(p, spec=dict(p["spec"], nodeName="node-2"), status={"phase": "Running"})
                running.append(p)
                w.apply(p)
        elif op < 0.5:  # relabel a running pod: its reservation moves with it
            p = rng.choice(running)
            p["metadata"]["labels"] = rand_labels(rng)
            w.apply(p)
            seen.add("update")
        elif op < 0.57 and len(running) > 5:  # delete a pod: it is un-reserved
            p = running.pop(rng.randrange(len(running)))
            w.delete("Pod", p["metadata"]["name"], p["metadata"]["namespace"])
            seen.add("delete")
        elif op < 0.65:
            w.same("prefilter_batch", rng.sample(manifests, rng.randint(1, 20)), oracle=False)
            seen.add("batch")
        elif op < 0.72:  # a sorted queue admitted one pod per cycle (device fixpoint, or host rounds)
            batch = rng.sample(manifests, rng.randint(1, 25))
            got = w.same("admit_queue", batch, oracle=False)
            if "error" not in got:
                for p, r in zip(batch, got["results"]):  # the oracle admits them one per cycle
                    want = w.ref.prefilter(p)
                    assert norm_prefilter(r["preFilter"]) == norm_prefilter(want), (where, nn(p))
                    if want["code"] == "Success":
                        w.ref.reserve(p)
                        reserved.append(p)
                seen.add("admit")
        elif op < 0.8:  # PreFilter / Reserve of a queued pod by key
            p = rng.choice(queue)
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if w.dut.queue_row(*k) >= 0 and w.same("prefilter_key", *k, oracle=False)["code"] == "Success":
                w.ref.reserve(p)
                w.same("reserve_key", *k, oracle=False)
        elif op < 0.88:
            w.ref.reconcile_all(NOW)
            w.same("reconcile_all", NOW, oracle=False)
        else:  # a new manifest or a new running pod, maybe with a resource nobody asked for before
            bound = rng.random() < 0.5
            p = rand_pod(rng, rng.choice(nss + ["elsewhere"]), f"n{step}", bound)
            if rng.random() < 0.2:
                p["spec"]["containers"][0]["resources"]["requests"]["example.com/widget"] = str(rng.randint(1, 3))
            if bound:
                running.append(p)
                w.apply(p)
            else:
                manifests.append(p)
        held = [p for p in running[:6] if p["spec"]["schedulerName"] == SCHED]
        w.compare(queue, held, where)
    for x in (w.dut, w.twin, w.ref):
        x.close()
    return seen


@pytest.mark.parametrize("seed", [0, 1, 2, 4])
def test_manifest_stream(oracle, new_plugin, host_on_oracle_check_rows, seed):  # noqa: F811
    seen = run_stream(oracle, new_plugin, host_on_oracle_check_rows, seed)
    assert {"Success", "reserve", "update", "batch", "admit"} <= seen, seen


@pytest.mark.parametrize("seed", [10, 11])
def test_manifest_stream_broken_selector(oracle, new_plugin, host_on_oracle_check_rows, seed):  # noqa: F811
    seen = run_stream(oracle, new_plugin, host_on_oracle_check_rows, seed, broken=True)
    assert {"admit", "batch"} <= seen, seen


def test_manifest_calls(oracle, host_on_oracle_check_pods):
    """On the counting double: a manifest PreFilter, Reserve and Unreserve each make one kt_check_pods call, no kt_evaluate and
    no pending-row upload -- also with a long resident queue; a batch makes one call for all its pods."""
    ref, dut = oracle.World(THROTTLER, SCHED), host_on_oracle_check_pods(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    lbl = {"app": "x"}
    both(namespace("na"), namespace("nb"), throttle("na", "a", lbl, pod_cnt=3), throttle("nb", "b", lbl, cpu="1"))
    both(*[pod("na" if i % 2 else "nb", f"q{i}", "100m", lbl) for i in range(200)])
    both(pod("na", "run", "100m", lbl, node="n", phase="Running"))
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    dut.prefilter_queue()
    m = pod("na", "m", "100m", lbl)
    for call in ("prefilter", "reserve", "unreserve", "prefilter"):
        before = host_on_oracle_check_pods.calls()
        got, want = getattr(dut, call)(m), getattr(ref, call)(m)
        assert got["code"] == "Success" and want.get("code", "Success") == "Success", (call, got, want)
        after = host_on_oracle_check_pods.calls()
        d = {k: after[k] - before[k] for k in CALLS}
        assert d == {"check_pods": 1, "evaluate": 0, "pending_uploads": 0}, (call, d)
    batch = [pod("nb", f"b{i}", "500m", lbl) for i in range(40)]
    before = host_on_oracle_check_pods.calls()
    got = dut.prefilter_batch(batch)
    assert [norm_prefilter(r) for r in got] == [norm_prefilter(ref.prefilter(p)) for p in batch]
    after = host_on_oracle_check_pods.calls()
    assert after["check_pods"] - before["check_pods"] == 1 and after["evaluate"] == before["evaluate"], (before, after)
    dut.close()
    ref.close()
