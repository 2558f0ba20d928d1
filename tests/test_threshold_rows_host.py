"""Threshold and override edits on the column path: a Throttle or ClusterThrottle event that changes spec.threshold or
spec.temporaryThresholdOverrides and nothing else of the spec sends only that column's threshold columns to the device
(kt_update_threshold_rows) and voids only the cached PreFilter verdicts of the queued pods that throttle affects.

Random streams mix threshold and override edits (values, presence, overrides added, removed, edited and reordered, parse errors,
open ends) with selector and throttlerName edits and edits bringing a new resource name (both still recompile the tables),
reconciles by key and their echoes, Reserve, PreFilter by key and binds; some streams go through kth_apply_events.  After every
step the plugin must agree with the object oracle (statuses, reservations, PreFilter by key, gauges, requeues) and, result for
result, with a twin plugin fed the same events that uploads the throttles whole on every spec edit (on the CPU an engine double
without the call, on the GPU a build of the host layer without it): statuses, reservations, PreFilter by key, affected pods, the
queue report and the metrics.  On the engine test double that counts its calls (CPU) a threshold-only or override-only edit makes
one kt_update_threshold_rows and no kt_upload_throttles, and only the queued pods of that throttle lose their cached verdict."""
import ctypes as C
import copy
import functools
import json
import os
import random

import pytest

from test_plugin_vs_oracle import VALS, rand_amount, rand_labels, rand_pod, rand_status, rand_throttle
from test_reconcile_keys import TIMES, Twin, _build, host_on_oracle_reconcile, key_oracle, nn_of  # noqa: F401 (fixtures)
from test_scenarios import NOW, SCHED, THROTTLER, clthrottle, namespace, pod, throttle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUB = os.path.join(ROOT, "tests", "host_stub")
CALLS = ("upload_throttles", "upload_status", "set_reserved", "update_status_rows", "update_reserved_rows", "evaluate")
HOST_DEPS = [os.path.join(ROOT, "kube_throttler_b200", "csrc", f) for f in ("kt_json.h", "kt_quantity.h")] + \
    [os.path.join(ROOT, "include", f) for f in ("kt_b200.h", "kt_host.h")]
ORACLE_LINK = ["-L", os.path.join(ROOT, "oracle"), "-lkt_oracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")]
ORACLE_DEPS = [os.path.join(STUB, f) for f in ("engine_oracle.cc", "engine_oracle_reconcile.cc", "engine_oracle_throttle_rows.cc")] + \
    [os.path.join(ROOT, "oracle", "libkt_oracle.so")]


def _counting(lib, extra=()):
    lib.kt_test_throttle_calls.argtypes = [C.POINTER(C.c_int64)]
    lib.kt_test_throttle_calls.restype = None
    for fn in extra:
        getattr(lib, fn).argtypes = []
        getattr(lib, fn).restype = C.c_int64

    def calls():
        out = (C.c_int64 * len(CALLS))()
        lib.kt_test_throttle_calls(out)
        got = dict(zip(CALLS, out))
        if extra:
            got["update_threshold_rows"] = lib.kt_test_threshold_calls()
        return got

    return calls


@pytest.fixture(scope="module")
def host_on_oracle_threshold_rows(oracle):
    """kt_host.cc linked against the oracle-backed engine test double with the threshold column deltas and call counters
    (tests/host_stub/engine_oracle_threshold_rows.cc); host.Plugin's signature plus `.calls()`."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_threshold_rows.cc")]
    lib = _build("libkt_hostoracle_threshold_rows.so", srcs, ORACLE_DEPS + HOST_DEPS, ORACLE_LINK)
    make = functools.partial(host.Plugin, library=lib)
    make.calls = _counting(lib, ("kt_test_threshold_calls",))
    return make


@pytest.fixture(scope="module")
def host_on_oracle_whole_thresholds(oracle):
    """The same host layer on the engine double without kt_update_threshold_rows (engine_oracle_throttle_rows.cc): every
    threshold or override edit recompiles and uploads the throttles whole."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_throttle_rows.cc")]
    lib = _build("libkt_hostoracle_throttle_rows.so", srcs, ORACLE_DEPS[:2] + ORACLE_DEPS[3:] + HOST_DEPS, ORACLE_LINK)
    make = functools.partial(host.Plugin, library=lib)
    make.calls = _counting(lib)
    return make


@pytest.fixture(scope="module")
def product_full_thresholds(kt):
    """kt_host.cc linked against the product library but built without its kt_update_threshold_rows reference
    (tests/host_stub/no_threshold_rows.h): the same device calls as host.Plugin, with every spec edit uploaded whole."""
    from kube_throttler_b200 import host

    pkg = os.path.join(ROOT, "kube_throttler_b200")
    srcs = [os.path.join(pkg, "csrc", "kt_host.cc")]
    deps = [os.path.join(STUB, "no_threshold_rows.h"), os.path.join(pkg, "libkt_b200.so")] + HOST_DEPS
    lib = _build("libkt_host_full_thresholds.so", srcs, deps,
                 ["-Dkt_update_threshold_rows=kt_update_threshold_rows_absent", "-include", os.path.join(STUB, "no_threshold_rows.h"),
                  "-L", pkg, "-lkt_b200", "-Wl,-rpath," + pkg])
    return functools.partial(host.Plugin, library=lib)


@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def plugins(request):
    """(the plugin on the column path, its twin on whole throttle uploads)"""
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle_threshold_rows"), request.getfixturevalue("host_on_oracle_whole_thresholds")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin, request.getfixturevalue("product_full_thresholds")


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


class SpecTwin(Twin):
    """The oracle and the plugin (Twin), plus a second plugin on whole throttle uploads that must answer exactly as the plugin."""

    def __init__(self, ref, dut, full):
        super().__init__(ref, dut)
        self.full = full

    def apply(self, *ms):
        super().apply(*ms)
        for m in ms:
            self.full.apply(m)

    def events(self, evs):
        """The same events through kth_apply_events on both plugins, one by one on the oracle."""
        for e in evs:
            self.ref.apply(e["object"])
            o = e["object"]
            if o["kind"] in ("Throttle", "ClusterThrottle"):
                self.live[(o["kind"], nn_of(o))] = o
        got = outcome(self.dut.apply_events, evs)
        assert outcome(self.full.apply_events, evs) == got
        if isinstance(got, tuple):  # an engine double without kt_match_pods: the events one by one
            for e in evs:
                for p in (self.dut, self.full):
                    p.apply(e["object"])
        return got

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
            assert self.dut.reserved(kind, key) == self.full.reserved(kind, key), (where, key)
            assert outcome(self.dut.affected_pods, name, ns) == outcome(self.full.affected_pods, name, ns), (where, key)
        for p in queue:
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if self.dut.queue_row(*k) >= 0:
                assert self.dut.prefilter_key(*k) == self.full.prefilter_key(*k), (where, k)
        assert outcome(self.dut.queue_report) == outcome(self.full.queue_report), where
        assert self.dut.metrics() == self.full.metrics(), where


OVR_BEGIN = ["", "2025-12-01T00:00:00Z", "2026-01-10T00:00:00Z", "2026-06-01T00:00:00Z", "garbage"]
OVR_END = ["", "2026-02-01T00:00:00+09:00", "2025-12-15T00:00:00Z", "2026-01-20T00:00:00Z", "not-a-time"]


def rand_override(rng):
    return {"begin": rng.choice(OVR_BEGIN), "end": rng.choice(OVR_END), "threshold": rand_amount(rng, rng.choice([1, 2]))}


def edit_overrides(rng, spec):
    """Overrides added, removed, edited or reordered, or a count 0 -> 3 / 3 -> 0."""
    ovs = list(spec.get("temporaryThresholdOverrides", []))
    how = rng.choice(["add", "remove", "edit", "reorder", "three", "none"])
    if how == "add" or (how in ("remove", "edit", "reorder") and not ovs):
        ovs.insert(rng.randint(0, len(ovs)), rand_override(rng))
    elif how == "remove":
        ovs.pop(rng.randrange(len(ovs)))
    elif how == "edit":
        i = rng.randrange(len(ovs))
        ovs[i] = dict(ovs[i], **{rng.choice(["begin", "end", "threshold"]): None})
        ovs[i] = {k: (v if v is not None else rand_override(rng)[k]) for k, v in ovs[i].items()}
    elif how == "reorder":
        ovs.append(rand_override(rng))
        rng.shuffle(ovs)
    elif how == "three":
        ovs = [rand_override(rng) for _ in range(3)]
    else:
        ovs = []
    if ovs:
        spec["temporaryThresholdOverrides"] = ovs
    else:
        spec.pop("temporaryThresholdOverrides", None)


def run_stream(key_oracle, new_plugin, full_plugin, seed, steps=70, n_thr=14, n_ns=4, batched=False):
    rng = random.Random(seed)
    ref, dut, full = key_oracle(), new_plugin(THROTTLER, SCHED), full_plugin(THROTTLER, SCHED)
    w = SpecTwin(ref, dut, full)
    cnt = Counter(new_plugin)
    nss = [f"ns{i}" for i in range(n_ns)]
    for n in nss:
        w.apply(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
    throttles = [rand_throttle(rng, i, nss) for i in range(n_thr)]
    for t in throttles:
        if t["kind"] == "Throttle":
            for term in t["spec"]["selector"]["selectorTerms"]:
                term.pop("namespaceSelector", None)
    w.apply(*throttles)
    pods = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(40)]
    w.apply(*pods)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(30)]
    w.apply(*queue)
    names = set()  # resource names a spec edit brought so far
    reserved, seen = [], {"threshold": 0, "override": 0, "other": 0, "delta": 0, "full": 0}
    for step in range(steps):
        op = rng.random()
        where = (seed, step)
        if op < 0.4:  # a spec edit: threshold, overrides, both; or a selector / throttlerName / new resource name edit
            i = rng.randrange(len(throttles))
            t = copy.deepcopy(throttles[i])
            t.pop("status", None)
            what = rng.choice(["threshold", "threshold", "override", "override", "both", "selector", "throttler", "resource"])
            spec = t["spec"]
            if what in ("threshold", "both"):
                spec["threshold"] = rand_amount(rng)
            if what in ("override", "both"):
                edit_overrides(rng, spec)
            if what == "selector":
                spec["selector"]["selectorTerms"] = [{"podSelector": {"matchLabels": {"app": rng.choice(VALS)}}}]
            if what == "throttler":
                spec["throttlerName"] = "foreign" if spec["throttlerName"] == THROTTLER else THROTTLER
            fresh_name = False
            if what == "resource":
                name = rng.choice(["ephemeral-storage", "example.com/fpga"])
                fresh_name = name not in names
                names.add(name)
                spec["threshold"] = dict(spec["threshold"], resourceRequests={name: "3"})
            tables_changed = what in ("selector", "throttler") and (spec["selector"], spec["throttlerName"]) != \
                (throttles[i]["spec"]["selector"], throttles[i]["spec"]["throttlerName"])
            throttles[i] = t
            dut.prefilter_queue()
            full.prefilter_queue()
            cnt.mark()
            if batched:
                w.events([{"type": "MODIFIED", "object": t}])
            else:
                w.apply(t)
            dut.prefilter_queue()
            c = cnt.since()
            if c is not None:
                if what in ("threshold", "override", "both"):
                    # (a new resource name or a finer scale in the new amounts moves every column: the whole path)
                    assert c["update_threshold_rows"] <= 1, (where, c)
                    assert c["upload_throttles"] + c["update_threshold_rows"] <= 1, (where, c)
                    seen["delta"] += c["update_threshold_rows"]
                    seen["full"] += c["upload_throttles"]
                elif tables_changed or fresh_name:  # the tables, the responsibility flag or the column layout: the whole path
                    assert c["upload_throttles"] == 1 and c["update_threshold_rows"] == 0, (where, what, c)
                elif what != "resource":  # an unchanged selector or throttlerName: nothing to send
                    assert c["upload_throttles"] == 0 and c["update_threshold_rows"] == 0, (where, what, c)
            seen["threshold" if what in ("threshold", "both") else "override" if what == "override" else "other"] += 1
        elif op < 0.6:  # reconcile(key) of a few throttles, then the informer echoes every status it wrote
            keys = [nn_of(t) for t in rng.sample(throttles, rng.randint(1, 4))]
            got = w.reconcile(keys, rng.choice(TIMES))
            w.echo(got["changed"])
        elif op < 0.72:  # PreFilter, and Reserve on Success
            p = rng.choice(queue)
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if dut.queue_row(*k) >= 0 and ref.prefilter(p)["code"] == "Success":
                assert ref.reserve(p)["code"] == dut.reserve_key(*k)["code"] == full.reserve_key(*k)["code"] == "Success", where
                reserved.append(p)
        elif op < 0.78:  # another writer's status, spec unchanged
            i = rng.randrange(len(throttles))
            w.apply(dict(throttles[i], status=rand_status(rng)))
        elif op < 0.85 and reserved:  # bind
            p = reserved.pop(rng.randrange(len(reserved)))
            queue.remove(p)
            p = dict(p, spec=dict(p["spec"], nodeName="node-2"), status={"phase": rng.choice(["Running", "Running", "Succeeded"])})
            pods.append(p)
            w.apply(p)
        elif op < 0.92:
            p = rng.choice(pods)
            p["metadata"]["labels"] = rand_labels(rng)
            w.apply(p)
        else:
            p = rand_pod(rng, rng.choice(nss), f"n{step}", False)
            queue.append(p)
            w.apply(p)
        w.compare(queue, where)
    for x in (dut, full, ref):
        x.close()
    return seen


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_threshold_stream(key_oracle, plugins, seed):
    seen = run_stream(key_oracle, *plugins, seed)
    assert seen["threshold"] >= 1 and seen["override"] >= 1 and seen["other"] >= 1, seen
    if getattr(plugins[0], "calls", None):
        assert seen["delta"] >= 3, seen


@pytest.mark.parametrize("seed", [10, 11])
def test_threshold_stream_batched(key_oracle, plugins, seed):
    """The same kind of stream with every spec edit through kth_apply_events."""
    seen = run_stream(key_oracle, *plugins, seed, batched=True)
    assert seen["threshold"] + seen["override"] >= 2, seen


def test_threshold_edit_voids_only_its_pods(key_oracle, host_on_oracle_threshold_rows):
    """Two Throttles in two namespaces, a queued pod in each: after one pass over the queue, an edit of throttle a's threshold or
    overrides makes one kt_update_threshold_rows and no upload; qb is answered from the cache, qa is checked again.  Selector and
    throttlerName edits still recompile the tables."""
    make = host_on_oracle_threshold_rows
    ref, dut = key_oracle(), make(THROTTLER, SCHED)
    w = Twin(ref, dut)
    cnt = Counter(make)
    lbl = {"app": "x"}
    ta, tb = throttle("na", "a", lbl, pod_cnt=5), throttle("nb", "b", lbl, pod_cnt=1)
    w.apply(namespace("na"), namespace("nb"), ta, tb)
    w.apply(pod("na", "run", "100m", lbl, node="n", phase="Running"), pod("nb", "run", "100m", lbl, node="n", phase="Running"))
    w.reconcile_all(NOW)
    qa, qb = pod("na", "qa", "100m", lbl), pod("nb", "qb", "100m", lbl)
    w.apply(qa, qb)
    dut.prefilter_queue()

    def check(p):
        a, b = ref.prefilter(p), dut.prefilter_key(p["metadata"]["namespace"], p["metadata"]["name"])
        assert (a["code"], a["reasons"]) == (b["code"], b["reasons"]), (a, b)
        return b

    ovr = [{"begin": "", "end": "", "threshold": {"resourceCounts": {"pod": 1}}},
           {"begin": "2025-01-01T00:00:00Z", "end": "", "threshold": {"resourceCounts": {"pod": 9}}},
           {"begin": "garbage", "end": "", "threshold": {"resourceCounts": {"pod": 2}}}]
    edits = [throttle("na", "a", lbl, pod_cnt=1),  # threshold only: qa becomes throttled
             throttle("na", "a", lbl, pod_cnt=1, overrides=ovr),  # 0 -> 3 overrides
             throttle("na", "a", lbl, pod_cnt=1, overrides=ovr[::-1]),  # reordered
             throttle("na", "a", lbl, pod_cnt=1, overrides=[ovr[1]]),  # 3 -> 1
             throttle("na", "a", lbl, pod_cnt=5)]  # 1 -> 0, threshold back
    for e in edits:
        w.apply(e)
        w.reconcile(["na/a"], NOW)  # the new threshold reaches the status through reconcile
        dut.prefilter_queue()
        cnt.mark()
        before = dut.queue_stats()
        w.apply(dict(e, spec=dict(e["spec"], threshold={"resourceCounts": {"pod": 4}})))  # the edit under test
        check(qb)
        mid = dut.queue_stats()
        assert mid["passes"] == before["passes"] and mid["hits"] == before["hits"] + 1, (e, before, mid)
        check(qa)
        assert dut.queue_stats()["passes"] == mid["passes"] + 1, e
        c = cnt.since()
        assert c["update_threshold_rows"] == 1 and c["upload_throttles"] == 0, (e, c)
        assert c["upload_status"] == 0 and c["set_reserved"] == 0, (e, c)
        w.apply(e)
    # selector and throttlerName edits recompile the tables, as before
    for e in (throttle("na", "a", {"app": "y"}, pod_cnt=5), throttle("na", "a", {"app": "y"}, pod_cnt=5, throttler="foreign")):
        cnt.mark()
        w.apply(e)
        check(qa)
        c = cnt.since()
        assert c["upload_throttles"] == 1 and c["update_threshold_rows"] == 0, (e, c)
    w.compare([qa, qb], "end")
    dut.close()
    ref.close()
