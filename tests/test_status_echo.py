"""The status echo: reconcile writes a throttle's status, the Go side sends it with UpdateStatus, and the informer hands the same
Throttle back as a MODIFIED event.  Such an event -- and any other one whose spec equals the stored one (a status written by
another replica) -- must not recompile the selector tables or void the whole scheduling queue's cached verdicts: only that
column's status goes to the device again (kt_update_status_rows), and Reserve / Unreserve send only the columns whose
reservations changed (kt_update_reserved_rows).

Random streams interleave reconciles by key followed by their echoes, other writers' statuses, Reserve, PreFilter by key, spec
edits, pod binds and relabels.  After every step the plugin must agree with the object oracle (statuses, reservations, PreFilter
by key, gauges) and, result for result, with a twin plugin fed the same events whose engine double has no column deltas (so it
uploads whole tables, as before).  On the engine test double that counts its calls (CPU) an echo makes no kt_upload_throttles
and at most one kt_update_status_rows call, a Reserve one kt_update_reserved_rows and no kt_set_reserved call, and a spec edit
still recompiles the tables."""
import ctypes as C
import functools
import json
import os
import random

import pytest

from test_plugin_vs_oracle import CPUS, VALS, rand_labels, rand_pod, rand_status, rand_throttle
from test_reconcile_keys import TIMES, Twin, _build, host_on_oracle_reconcile, key_oracle, nn_of  # noqa: F401 (fixtures)
from test_scenarios import NOW, SCHED, THROTTLER, namespace, pod, throttle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUB = os.path.join(ROOT, "tests", "host_stub")
CALLS = ("upload_throttles", "upload_status", "set_reserved", "update_status_rows", "update_reserved_rows", "evaluate")


@pytest.fixture(scope="module")
def host_on_oracle_throttle_rows(oracle):
    """kt_host.cc linked against the oracle-backed engine test double with the column deltas and call counters
    (tests/host_stub/engine_oracle_throttle_rows.cc); host.Plugin's signature plus `.calls()`."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_throttle_rows.cc")]
    deps = [os.path.join(STUB, f) for f in ("engine_oracle.cc", "engine_oracle_reconcile.cc")] + [os.path.join(ROOT, "oracle", "libkt_oracle.so")] + \
        [os.path.join(ROOT, "kube_throttler_b200", "csrc", f) for f in ("kt_json.h", "kt_quantity.h")] + \
        [os.path.join(ROOT, "include", f) for f in ("kt_b200.h", "kt_host.h")]
    lib = _build("libkt_hostoracle_throttle_rows.so", srcs, deps,
                 ["-L", os.path.join(ROOT, "oracle"), "-lkt_oracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    lib.kt_test_throttle_calls.argtypes = [C.POINTER(C.c_int64)]
    lib.kt_test_throttle_calls.restype = None

    def calls():
        out = (C.c_int64 * len(CALLS))()
        lib.kt_test_throttle_calls(out)
        return dict(zip(CALLS, out))

    make = functools.partial(host.Plugin, library=lib)
    make.calls = calls
    return make


@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def new_plugin(request):
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle_throttle_rows")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin


class Counter:
    """Calls of the counting double between two points of a test; a no-op on the product."""

    def __init__(self, make):
        self.read = getattr(make, "calls", None)
        self.mark()

    def mark(self):
        self.at = self.read() if self.read else None

    def since(self):
        if not self.read:
            return None
        now = self.read()
        return {k: now[k] - self.at[k] for k in CALLS}


class EchoTwin(Twin):
    """The oracle and the plugin (Twin), plus a second plugin on whole-table uploads that must answer exactly as the plugin."""

    def __init__(self, ref, dut, full):
        super().__init__(ref, dut)
        self.full = full

    def apply(self, *ms):
        super().apply(*ms)
        for m in ms:
            self.full.apply(m)

    def reconcile(self, keys, now):
        got = super().reconcile(keys, now)
        assert self.full.reconcile(keys, now) == got, keys
        return got

    def echo(self, keys):
        """What the informer delivers after UpdateStatus of each key: the stored spec with the status the plugin holds."""
        for key in keys:
            ns, _, name = key.partition("/")
            t = self.live[("ClusterThrottle" if ns == "" else "Throttle", key)]
            self.apply(dict(t, status=json.loads(self.dut.status_manifest(name, ns))))

    def compare(self, queue, where):
        super().compare(queue, where)
        for (kind, key) in self.live:
            ns, _, name = key.partition("/")
            assert self.dut.status(name, ns) == self.full.status(name, ns), (where, key)
            assert self.dut.status_manifest(name, ns) == self.full.status_manifest(name, ns), (where, key)
            assert self.dut.reserved(kind, key) == self.full.reserved(kind, key), (where, key)
        for p in queue:
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if self.dut.queue_row(*k) >= 0:
                assert self.dut.prefilter_key(*k) == self.full.prefilter_key(*k), (where, k)
        assert self.dut.metrics() == self.full.metrics(), where


def run_echo_stream(key_oracle, new_plugin, full_plugin, seed, steps=60, n_thr=14, n_ns=4):
    rng = random.Random(seed)
    ref, dut, full = key_oracle(), new_plugin(THROTTLER, SCHED), full_plugin(THROTTLER, SCHED)
    w = EchoTwin(ref, dut, full)
    cnt = Counter(new_plugin)
    nss = [f"ns{i}" for i in range(n_ns)]
    for n in nss:
        w.apply(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
    throttles = [rand_throttle(rng, i, nss) for i in range(n_thr)]
    w.apply(*throttles)
    pods = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(50)]
    w.apply(*pods)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(30)]
    w.apply(*queue)
    reserved, seen = [], {"echo": 0, "reserve": 0, "edit": 0}
    for step in range(steps):
        op = rng.random()
        where = (seed, step)
        if op < 0.35:  # reconcile(key) of a few throttles, then the informer echoes every status it wrote
            keys = [nn_of(t) for t in rng.sample(throttles, rng.randint(1, 4))]
            got = w.reconcile(keys, rng.choice(TIMES))
            dut.prefilter_queue()  # the reconcile's own status writes reach the device here
            cnt.mark()
            w.echo(got["changed"])
            dut.prefilter_queue()
            c = cnt.since()
            if c is not None:
                assert c["upload_throttles"] == 0 and c["upload_status"] == 0 and c["update_status_rows"] == 0, (where, c)
            seen["echo"] += bool(got["changed"])
        elif op < 0.55:  # PreFilter, and Reserve on Success
            p = rng.choice(queue)
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if dut.queue_row(*k) >= 0 and ref.prefilter(p)["code"] == "Success":
                dut.prefilter_queue()
                holders = lambda: {key for (kind, key) in w.live if nn_of(p) in dut.reserved(kind, key)["pods"]}
                before = holders()
                cnt.mark()
                assert ref.reserve(p)["code"] == dut.reserve_key(*k)["code"] == full.reserve_key(*k)["code"] == "Success", where
                dut.prefilter_key(*k)  # the reserved pod's own verdict is void: this pass sends the reservations
                c = cnt.since()
                new = bool(holders() - before)
                if c is not None:
                    assert c["set_reserved"] == 0 and c["upload_throttles"] == 0 and c["update_reserved_rows"] <= 1, (where, c)
                    assert c["update_reserved_rows"] == 1 or not new, (where, c)
                seen["reserve"] += new
                reserved.append(p)
        elif op < 0.62:  # another writer's status through the informer, spec unchanged
            i = rng.randrange(len(throttles))
            w.apply(dict(throttles[i], status=rand_status(rng)))
        elif op < 0.7:  # a spec edit: the tables are compiled again
            i = rng.randrange(len(throttles))
            t = rand_throttle(rng, i, nss)
            t["kind"], t["metadata"] = throttles[i]["kind"], throttles[i]["metadata"]
            if t["kind"] == "Throttle":
                for term in t["spec"]["selector"]["selectorTerms"]:
                    term.pop("namespaceSelector", None)
            changed = t["spec"] != throttles[i]["spec"]
            throttles[i] = t
            cnt.mark()
            w.apply(t)
            dut.prefilter_queue()
            c = cnt.since()
            if c is not None and changed:
                assert c["upload_throttles"] == 1, (where, c)
            seen["edit"] += changed
        elif op < 0.78 and reserved:  # bind
            p = reserved.pop(rng.randrange(len(reserved)))
            queue.remove(p)
            p = dict(p, spec=dict(p["spec"], nodeName="node-2"), status={"phase": rng.choice(["Running", "Running", "Succeeded"])})
            pods.append(p)
            w.apply(p)
        elif op < 0.88:
            p = rng.choice(pods)
            p["metadata"]["labels"] = rand_labels(rng)
            w.apply(p)
        else:
            p = rand_pod(rng, rng.choice(nss), f"n{step}", True)
            p["spec"]["containers"][0]["resources"]["requests"]["cpu"] = rng.choice(CPUS)
            pods.append(p)
            w.apply(p)
        w.compare(queue, where)
    for x in (dut, full, ref):
        x.close()
    return seen


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_echo_stream(key_oracle, new_plugin, host_on_oracle_reconcile, seed):
    seen = run_echo_stream(key_oracle, new_plugin, host_on_oracle_reconcile, seed)
    assert seen["echo"] >= 3 and seen["edit"] >= 1, seen


def test_echo_keeps_unaffected_verdicts(key_oracle, new_plugin):
    """Two Throttles in two namespaces, a queued pod in each: after one pass over the queue, a reconcile of throttle a that changes
    its status and the echo of that status, the pod a does not affect is answered from the cached verdicts (a hit, no pass); the
    pod it affects is checked again.  An echo of an unchanged status voids nothing."""
    ref, dut = key_oracle(), new_plugin(THROTTLER, SCHED)
    w = Twin(ref, dut)
    cnt = Counter(new_plugin)
    lbl = {"app": "x"}
    ta, tb = throttle("na", "a", lbl, pod_cnt=5), throttle("nb", "b", lbl, pod_cnt=1)
    w.apply(namespace("na"), namespace("nb"), ta, tb)
    w.apply(pod("na", "run", "100m", lbl, node="n", phase="Running"))
    qa, qb = pod("na", "qa", "100m", lbl), pod("nb", "qb", "100m", lbl)
    w.apply(qa, qb)
    dut.prefilter_queue()
    got = w.reconcile(["na/a"], NOW)
    assert got["changed"] == ["na/a"]
    dut.prefilter_queue()  # the reconcile's status write voided qa's verdict: one pass
    cnt.mark()
    before = dut.queue_stats()
    w.apply(dict(ta, status=json.loads(dut.status_manifest("a", "na"))))  # the echo
    for p in (qb, qa):
        a, b = ref.prefilter(p), dut.prefilter_key(p["metadata"]["namespace"], p["metadata"]["name"])
        assert (a["code"], a["reasons"]) == (b["code"], b["reasons"])
    after = dut.queue_stats()
    assert after["passes"] == before["passes"] and after["hits"] == before["hits"] + 2, (before, after)
    c = cnt.since()
    if c is not None:
        assert c["upload_throttles"] == 0 and c["upload_status"] == 0 and c["update_status_rows"] == 0 and c["evaluate"] == 0, c
    # another writer's status for throttle b: only qb's verdict is void
    w.apply(dict(tb, status={"used": {"resourceCounts": {"pod": 1}}, "throttled": {"resourceCounts": {"pod": True}},
                             "calculatedThreshold": {"threshold": {"resourceCounts": {"pod": 1}}, "calculatedAt": NOW}}))
    before = dut.queue_stats()
    a, b = ref.prefilter(qa), dut.prefilter_key("na", "qa")
    assert (a["code"], a["reasons"]) == (b["code"], b["reasons"])
    mid = dut.queue_stats()
    assert mid["passes"] == before["passes"] and mid["hits"] == before["hits"] + 1, (before, mid)
    a, b = ref.prefilter(qb), dut.prefilter_key("nb", "qb")
    assert (a["code"], a["reasons"]) == (b["code"], b["reasons"]) and b["code"] != "Success"
    assert dut.queue_stats()["passes"] == mid["passes"] + 1
    c = cnt.since()
    if c is not None:
        assert c["upload_throttles"] == 0 and c["upload_status"] == 0 and c["update_status_rows"] == 1, c
    # Reserve of qa: one column delta for the reservation of throttle a, qb's verdict stays cached
    assert dut.prefilter_key("na", "qa")["code"] == "Success"
    cnt.mark()
    before = dut.queue_stats()
    assert ref.reserve(qa)["code"] == dut.reserve_key("na", "qa")["code"] == "Success"
    assert dut.reserved("Throttle", "na/a")["pods"] == ["na/qa"]
    a, b = ref.prefilter(qa), dut.prefilter_key("na", "qa")
    assert (a["code"], a["reasons"]) == (b["code"], b["reasons"])
    a, b = ref.prefilter(qb), dut.prefilter_key("nb", "qb")
    assert (a["code"], a["reasons"]) == (b["code"], b["reasons"])
    after = dut.queue_stats()
    assert after["passes"] == before["passes"] + 1 and after["hits"] == before["hits"] + 2, (before, after)
    c = cnt.since()
    if c is not None:
        assert c["update_reserved_rows"] == 1 and c["set_reserved"] == 0 and c["upload_throttles"] == 0, c
    w.compare([qa, qb], "end")
    dut.close()
    ref.close()
