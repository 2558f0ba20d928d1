"""Namespace events on the row path: a Namespace created, relabelled or deleted sends only its own row to the device
(kt_update_namespace_rows) and voids only the cached PreFilter verdicts of the queued pods in that namespace.

Random streams mix namespace creations, relabels (ClusterThrottle namespaceSelectors flip both ways), deletions and
re-creations with throttle edits, pod events, Reserve, PreFilter and reconcile.  After every step the plugin must agree with the
object oracle (statuses, reservations, PreFilter by key, gauges) and, result for result, with a twin plugin fed the same events
whose engine double has no kt_update_namespace_rows (so it uploads every namespace row, as before): PreFilter by key and by
manifest, reconcile, affected pods, the queue report and the metrics.  Some streams also go through kth_apply_events, which cuts
its batch at a Namespace event.  On the engine test double that counts its calls (CPU) a Namespace event makes one
kt_update_namespace_rows and no kt_upload_namespaces or kt_upload_throttles, and only the queued pods of that namespace lose
their cached verdict."""
import ctypes as C
import functools
import json
import os
import random

import pytest

from test_plugin_vs_oracle import VALS, rand_labels, rand_pod, rand_throttle
from test_reconcile_keys import TIMES, Twin, _build, host_on_oracle_reconcile, key_oracle, nn_of  # noqa: F401 (fixtures)
from test_scenarios import NOW, SCHED, THROTTLER, clthrottle, namespace, pod, throttle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUB = os.path.join(ROOT, "tests", "host_stub")
CALLS = ("upload_throttles", "upload_status", "set_reserved", "update_status_rows", "update_reserved_rows", "evaluate")
NS_CALLS = ("upload_namespaces", "update_namespace_rows")


@pytest.fixture(scope="module")
def host_on_oracle_namespace_rows(oracle):
    """kt_host.cc linked against the oracle-backed engine test double with the namespace row deltas and call counters
    (tests/host_stub/engine_oracle_namespace_rows.cc); host.Plugin's signature plus `.calls()`."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_namespace_rows.cc")]
    deps = [os.path.join(STUB, f) for f in ("engine_oracle.cc", "engine_oracle_reconcile.cc", "engine_oracle_throttle_rows.cc")] + \
        [os.path.join(ROOT, "oracle", "libkt_oracle.so")] + \
        [os.path.join(ROOT, "kube_throttler_b200", "csrc", f) for f in ("kt_json.h", "kt_quantity.h")] + \
        [os.path.join(ROOT, "include", f) for f in ("kt_b200.h", "kt_host.h")]
    lib = _build("libkt_hostoracle_namespace_rows.so", srcs, deps,
                 ["-L", os.path.join(ROOT, "oracle"), "-lkt_oracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    for fn, n in (("kt_test_throttle_calls", CALLS), ("kt_test_namespace_calls", NS_CALLS)):
        getattr(lib, fn).argtypes = [C.POINTER(C.c_int64)]
        getattr(lib, fn).restype = None

    def calls():
        a, b = (C.c_int64 * len(CALLS))(), (C.c_int64 * len(NS_CALLS))()
        lib.kt_test_throttle_calls(a)
        lib.kt_test_namespace_calls(b)
        return dict(zip(CALLS + NS_CALLS, list(a) + list(b)))

    make = functools.partial(host.Plugin, library=lib)
    make.calls = calls
    return make


@pytest.fixture(scope="module")
def product_full_path(kt):
    """kt_host.cc linked against the product library but built without its kt_update_namespace_rows reference
    (tests/host_stub/no_namespace_rows.h): the same device calls as host.Plugin, with every namespace row uploaded whole."""
    from kube_throttler_b200 import host

    pkg = os.path.join(ROOT, "kube_throttler_b200")
    srcs = [os.path.join(pkg, "csrc", "kt_host.cc")]
    deps = [os.path.join(STUB, "no_namespace_rows.h"), os.path.join(pkg, "libkt_b200.so")] + \
        [os.path.join(pkg, "csrc", f) for f in ("kt_json.h", "kt_quantity.h")] + [os.path.join(ROOT, "include", f) for f in ("kt_b200.h", "kt_host.h")]
    lib = _build("libkt_host_full_namespaces.so", srcs, deps,
                 ["-Dkt_update_namespace_rows=kt_update_namespace_rows_absent", "-include", os.path.join(STUB, "no_namespace_rows.h"),
                  "-L", pkg, "-lkt_b200", "-Wl,-rpath," + pkg])
    return functools.partial(host.Plugin, library=lib)


@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def plugins(request):
    """(the plugin on the row path, its twin on whole namespace uploads)"""
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle_namespace_rows"), request.getfixturevalue("host_on_oracle_reconcile")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin, request.getfixturevalue("product_full_path")


@pytest.fixture
def new_plugin(plugins):
    return plugins[0]


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
        return {k: now[k] - self.at[k] for k in now}


def outcome(f, *args):
    try:
        return f(*args)
    except Exception as e:  # the same refusal on both sides
        return ("error", str(e))


class NsTwin(Twin):
    """The oracle and the plugin (Twin), plus a second plugin on whole namespace uploads that must answer exactly as the plugin."""

    def __init__(self, ref, dut, full):
        super().__init__(ref, dut)
        self.full = full

    def apply(self, *ms):
        super().apply(*ms)
        for m in ms:
            self.full.apply(m)

    def delete(self, kind, name, ns=""):
        super().delete(kind, name, ns)
        self.full.delete(kind, name, ns)

    def events(self, evs):
        """The same events through kth_apply_events on both plugins, one by one on the oracle."""
        for e in evs:
            if e["type"] == "DELETED":
                o = e["object"]
                self.ref.delete(o["kind"], o["metadata"]["name"], o["metadata"].get("namespace", ""))
            else:
                self.ref.apply(e["object"])
        got = outcome(self.dut.apply_events, evs)
        assert outcome(self.full.apply_events, evs) == got
        if isinstance(got, tuple):  # an engine double without kt_match_pods: the events one by one
            for e in evs:
                o = e["object"]
                for p in (self.dut, self.full):
                    if e["type"] == "DELETED":
                        p.delete(o["kind"], o["metadata"]["name"], o["metadata"].get("namespace", ""))
                    else:
                        p.apply(o)
        return got

    def reconcile(self, keys, now):
        got = super().reconcile(keys, now)
        assert self.full.reconcile(keys, now) == got, keys
        return got

    def compare(self, queue, where, manifests=()):
        super().compare(queue, where)
        for p in queue:
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if self.dut.queue_row(*k) >= 0:
                assert self.dut.prefilter_key(*k) == self.full.prefilter_key(*k), (where, k)
        for p in manifests:
            a, b = outcome(self.dut.prefilter, p), outcome(self.full.prefilter, p)
            assert a == b, (where, p["metadata"])
            want = self.ref.prefilter(p)
            if isinstance(a, dict):
                assert (a["code"], a["reasons"]) == (want["code"], want["reasons"]), (where, p["metadata"], a, want)
        for (kind, key) in self.live:
            ns, _, name = key.partition("/")
            assert outcome(self.dut.affected_pods, name, ns) == outcome(self.full.affected_pods, name, ns), (where, key)
        assert outcome(self.dut.queue_report) == outcome(self.full.queue_report), where
        assert self.dut.metrics() == self.full.metrics(), where


def ns_labels(rng):
    lab = {}
    if rng.random() < 0.8:
        lab["team"] = rng.choice(VALS)
    if rng.random() < 0.7:
        lab["env"] = rng.choice(VALS)
    return lab


def rand_cluster(rng, i):
    """A ClusterThrottle whose namespaceSelectors use every operator (and empty selectors)."""
    sels = [{}, {"matchLabels": {"team": rng.choice(VALS)}},
            {"matchExpressions": [{"key": "env", "operator": "NotIn", "values": [rng.choice(VALS)]}]},
            {"matchExpressions": [{"key": "team", "operator": "Exists"}]},
            {"matchExpressions": [{"key": "env", "operator": "DoesNotExist"}]},
            {"matchExpressions": [{"key": "team", "operator": "In", "values": rng.sample(VALS, 2)}]}]
    t = clthrottle(f"c{i}", rng.choice(sels), {"matchLabels": {"app": rng.choice(VALS)}} if rng.random() < 0.5 else {}, pod_cnt=rng.randint(1, 6))
    if rng.random() < 0.3:
        t["spec"]["selector"]["selectorTerms"].append({"podSelector": {"matchLabels": {"tier": rng.choice(VALS)}}, "namespaceSelector": rng.choice(sels)})
    return t


def run_stream(key_oracle, new_plugin, full_plugin, seed, steps=60, n_thr=12, n_ns=5, batched=False):
    rng = random.Random(seed)
    ref, dut, full = key_oracle(), new_plugin(THROTTLER, SCHED), full_plugin(THROTTLER, SCHED)
    w = NsTwin(ref, dut, full)
    cnt = Counter(new_plugin)
    nss = [f"ns{i}" for i in range(n_ns)]
    alive = set(nss)
    for n in nss:
        w.apply(namespace(n, ns_labels(rng)))
    throttles = [rand_throttle(rng, i, nss) for i in range(n_thr)] + [rand_cluster(rng, i) for i in range(6)]
    w.apply(*throttles)
    pods = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(40)]
    w.apply(*pods)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(30)]
    w.apply(*queue)
    seen = {"create": 0, "relabel": 0, "delete": 0, "recreate": 0}
    for step in range(steps):
        op = rng.random()
        where = (seed, step)
        manifests = []
        if op < 0.4:  # a Namespace event
            kind = rng.choice(["create", "relabel", "relabel", "delete", "recreate"])
            gone = [n for n in nss if n not in alive]
            if kind == "create" or (kind == "recreate" and not gone):
                n = f"ns{len(nss)}"
                nss.append(n)
                kind = "create"
            elif kind == "recreate":
                n = rng.choice(gone)
            elif not alive:
                continue
            else:
                n = rng.choice(sorted(alive))
            dut.prefilter_queue()
            full.prefilter_queue()
            before = dut.queue_stats()
            cnt.mark()
            if kind == "delete":
                if batched:
                    w.events([{"type": "DELETED", "object": namespace(n)}])
                else:
                    w.delete("Namespace", n)
                alive.discard(n)
            else:
                m = namespace(n, ns_labels(rng))
                if batched:
                    w.events([{"type": "ADDED" if kind != "relabel" else "MODIFIED", "object": m}])
                else:
                    w.apply(m)
                alive.add(n)
            seen[kind] += 1
            # every queued pod outside n keeps its cached verdict; the pods in n are checked again by one pass
            others = [p for p in queue if p["metadata"]["namespace"] != n]
            for p in others:
                dut.prefilter_key(p["metadata"]["namespace"], p["metadata"]["name"])
            mid = dut.queue_stats()
            c = cnt.since()
            if c is not None:
                assert mid["passes"] == before["passes"], (where, before, mid)
                assert c["update_namespace_rows"] <= 1 and c["upload_namespaces"] == 0 and c["upload_throttles"] == 0, (where, c)
            mine = [p for p in queue if p["metadata"]["namespace"] == n and dut.queue_row(n, p["metadata"]["name"]) >= 0]
            if mine:
                dut.prefilter_key(mine[0]["metadata"]["namespace"], mine[0]["metadata"]["name"])
                if c is not None:
                    assert dut.queue_stats()["passes"] == mid["passes"] + 1, where
                    assert cnt.since()["update_namespace_rows"] == 1, where
        elif op < 0.5:  # a throttle spec edit (everything is uploaded again)
            i = rng.randrange(len(throttles))
            t = rand_throttle(rng, i, nss) if throttles[i]["kind"] == "Throttle" else rand_cluster(rng, int(throttles[i]["metadata"]["name"][1:]))
            if t["kind"] != throttles[i]["kind"]:
                continue
            t["metadata"] = throttles[i]["metadata"]
            throttles[i] = t
            w.apply(t)
        elif op < 0.62:  # reconcile of a few keys
            keys = [nn_of(t) for t in rng.sample(throttles, rng.randint(1, 4))]
            w.reconcile(keys, rng.choice(TIMES))
        elif op < 0.72:  # PreFilter and Reserve of a queued pod
            p = rng.choice(queue)
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if dut.queue_row(*k) >= 0 and ref.prefilter(p)["code"] == "Success":
                assert ref.reserve(p)["code"] == dut.reserve_key(*k)["code"] == full.reserve_key(*k)["code"] == "Success", where
        elif op < 0.82:  # a pod relabel, or a new pod (possibly in a namespace nobody created)
            if rng.random() < 0.5:
                p = rng.choice(pods)
                p["metadata"]["labels"] = rand_labels(rng)
            else:
                p = rand_pod(rng, rng.choice(nss + ["ghost"]), f"n{step}", rng.random() < 0.5)
                (pods if p["spec"].get("nodeName") else queue).append(p)
            w.apply(p)
        else:  # manifests PreFilter: namespaces alive, deleted, never seen
            manifests = [rand_pod(rng, rng.choice(nss + ["nowhere"]), f"m{step}_{j}", False) for j in range(3)]
        w.compare(queue, where, manifests)
    for x in (dut, full, ref):
        x.close()
    return seen


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_namespace_stream(key_oracle, plugins, seed):
    seen = run_stream(key_oracle, *plugins, seed)
    assert min(seen.values()) >= 1, seen


@pytest.mark.parametrize("seed", [10, 11])
def test_namespace_stream_batched(key_oracle, plugins, seed):
    """The same streams through kth_apply_events: the batch is cut at each Namespace event."""
    seen = run_stream(key_oracle, *plugins, seed, batched=True)
    assert seen["relabel"] >= 1, seen


def test_namespace_event_voids_only_its_pods(key_oracle, new_plugin):
    """A ClusterThrottle selecting team=a, a queued pod in each of two namespaces: after one pass over the queue, relabelling na
    out of the selector answers qb from the cache and checks qa again, and so do deleting na and re-creating it."""
    ref, dut = key_oracle(), new_plugin(THROTTLER, SCHED)
    w = Twin(ref, dut)
    cnt = Counter(new_plugin)
    lbl = {"app": "x"}
    ct = clthrottle("c", {"matchLabels": {"team": "a"}}, lbl, pod_cnt=1)
    w.apply(namespace("na", {"team": "a"}), namespace("nb", {"team": "a"}), ct, throttle("nb", "t", lbl, pod_cnt=5))
    w.apply(pod("na", "run", "100m", lbl, node="n", phase="Running"), pod("nb", "run", "100m", lbl, node="n", phase="Running"))
    w.reconcile_all(NOW)
    qa, qb = pod("na", "qa", "100m", lbl), pod("nb", "qb", "100m", lbl)
    w.apply(qa, qb)
    dut.prefilter_queue()

    def check(p):
        a, b = ref.prefilter(p), dut.prefilter_key(p["metadata"]["namespace"], p["metadata"]["name"])
        assert (a["code"], a["reasons"]) == (b["code"], b["reasons"]), (a, b)
        return b

    for labels, gone in (({"team": "b"}, False), (None, True), ({"team": "a"}, False)):
        cnt.mark()
        before = dut.queue_stats()
        if gone:
            w.delete("Namespace", "na")
        else:
            w.apply(namespace("na", labels))
        check(qb)
        mid = dut.queue_stats()
        assert mid["passes"] == before["passes"] and mid["hits"] == before["hits"] + 1, (before, mid)
        check(qa)
        assert dut.queue_stats()["passes"] == mid["passes"] + 1
        c = cnt.since()
        if c is not None:
            assert c["update_namespace_rows"] == 1 and c["upload_namespaces"] == 0 and c["upload_throttles"] == 0, c
            assert c["upload_status"] == 0 and c["set_reserved"] == 0, c
    # a namespace with more labels than the engine's slots re-creates the engine: everything is uploaded again
    cnt.mark()
    w.apply(namespace("nc", {f"k{i}": "v" for i in range(9)}))
    check(qa)
    check(qb)
    c = cnt.since()
    if c is not None:
        assert c["upload_namespaces"] == 1 and c["update_namespace_rows"] == 0 and c["upload_throttles"] == 1, c
    # and a throttle change takes the namespaces with it as before
    cnt.mark()
    w.apply(namespace("nd", {"team": "a"}), clthrottle("c2", {}, lbl, pod_cnt=3))
    check(qa)
    c = cnt.since()
    if c is not None:
        assert c["upload_namespaces"] == 1 and c["update_namespace_rows"] == 0 and c["upload_throttles"] == 1, c
    w.compare([qa, qb], "end")
    dut.close()
    ref.close()


def test_namespace_rows_on_the_full_path_without_the_call(key_oracle, host_on_oracle_reconcile):
    """An engine without kt_update_namespace_rows (the older doubles) keeps the whole upload, and the same answers."""
    ref, dut = key_oracle(), host_on_oracle_reconcile(THROTTLER, SCHED)
    w = Twin(ref, dut)
    lbl = {"app": "x"}
    w.apply(namespace("na", {"team": "a"}), clthrottle("c", {"matchLabels": {"team": "a"}}, lbl, pod_cnt=1))
    w.apply(pod("na", "run", "100m", lbl, node="n", phase="Running"))
    q = pod("na", "q", "100m", lbl)
    w.apply(q)
    for labels in ({"team": "b"}, {"team": "a"}):
        w.apply(namespace("na", labels))
        w.compare([q], labels)
    dut.close()
    ref.close()
