"""Throttle deletions and selector edits on the column path: a deleted Throttle or ClusterThrottle becomes a column that matches
nothing, and an edit of its selector terms or throttlerName that keeps its kind and namespace and mentions no label key or value
the dictionaries lack recompiles only its column (kt_update_selector_rows); neither re-lays out the columns nor voids the cached
PreFilter verdicts of the whole scheduling queue.

Random streams interleave deletions, selector edits within and beyond the label vocabulary, throttlerName flips, re-creations of
deleted names, threshold edits, Namespace relabels, pod events, reconciles with their echoes and PreFilter / Reserve by key; some
streams go through kth_apply_events.  After every step the plugin must agree with the object oracle and, result for result, with
a twin plugin fed the same events that uploads the throttles whole (on the CPU an engine double without the call, on the GPU a
build of the host layer without it): statuses, reservations, PreFilter by key, affected pods, the queue report and the metrics.
On the engine double that counts its calls (CPU), deletions and in-vocabulary edits take the delta, while vocabulary growth,
creations and a deletion that would leave more than half the columns holes upload the throttles whole."""
import copy
import functools
import os
import random

import pytest

from test_plugin_vs_oracle import VALS, rand_amount, rand_labels, rand_pod, rand_status, rand_throttle
from test_reconcile_keys import TIMES, Twin, _build, key_oracle, nn_of  # noqa: F401 (fixtures)
from test_scenarios import NOW, SCHED, THROTTLER, namespace, pod, throttle
from test_threshold_rows_host import HOST_DEPS, ORACLE_DEPS, ORACLE_LINK, ROOT, STUB, Counter, SpecTwin, _counting


@pytest.fixture(scope="module")
def host_on_oracle_selector_rows(oracle):
    """kt_host.cc linked against the oracle-backed engine double with the selector column deltas and call counters
    (tests/host_stub/engine_oracle_selector_rows.cc); host.Plugin's signature plus `.calls()`."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_selector_rows.cc")]
    deps = ORACLE_DEPS + [os.path.join(STUB, "engine_oracle_threshold_rows.cc")] + HOST_DEPS
    lib = _build("libkt_hostoracle_selector_rows.so", srcs, deps, ORACLE_LINK)
    make = functools.partial(host.Plugin, library=lib)
    counted = _counting(lib, ("kt_test_threshold_calls", "kt_test_selector_calls"))

    def calls():
        got = counted()
        got["update_selector_rows"] = lib.kt_test_selector_calls()
        return got

    make.calls = calls
    return make


@pytest.fixture(scope="module")
def host_on_oracle_whole_selectors(oracle):
    """The same host layer on the engine double without kt_update_selector_rows (engine_oracle_threshold_rows.cc): every deletion
    and selector edit uploads the throttles whole."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_threshold_rows.cc")]
    lib = _build("libkt_hostoracle_threshold_rows.so", srcs, ORACLE_DEPS + HOST_DEPS, ORACLE_LINK)
    return functools.partial(host.Plugin, library=lib)


@pytest.fixture(scope="module")
def product_full_selectors(kt):
    """kt_host.cc linked against the product library but built without its kt_update_selector_rows reference
    (tests/host_stub/no_selector_rows.h): the same device calls as host.Plugin, with every deletion and selector edit uploaded
    whole."""
    from kube_throttler_b200 import host

    pkg = os.path.join(ROOT, "kube_throttler_b200")
    srcs = [os.path.join(pkg, "csrc", "kt_host.cc")]
    deps = [os.path.join(STUB, "no_selector_rows.h"), os.path.join(pkg, "libkt_b200.so")] + HOST_DEPS
    lib = _build("libkt_host_full_selectors.so", srcs, deps,
                 ["-Dkt_update_selector_rows=kt_update_selector_rows_absent", "-include", os.path.join(STUB, "no_selector_rows.h"),
                  "-L", pkg, "-lkt_b200", "-Wl,-rpath," + pkg])
    return functools.partial(host.Plugin, library=lib)


@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def plugins(request):
    """(the plugin on the column path, its twin on whole throttle uploads)"""
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle_selector_rows"), request.getfixturevalue("host_on_oracle_whole_selectors")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin, request.getfixturevalue("product_full_selectors")


class SelectorTwin(SpecTwin):
    def delete(self, kind, name, ns=""):
        super().delete(kind, name, ns)
        self.full.delete(kind, name, ns)


def strip_status(t):
    t = copy.deepcopy(t)
    t.pop("status", None)
    return t


def run_stream(key_oracle, new_plugin, full_plugin, seed, steps=80, n_thr=14, n_ns=4, batched=False):
    rng = random.Random(seed)
    ref, dut, full = key_oracle(), new_plugin(THROTTLER, SCHED), full_plugin(THROTTLER, SCHED)
    w = SelectorTwin(ref, dut, full)
    cnt = Counter(new_plugin)
    nss = [f"ns{i}" for i in range(n_ns)]
    for n in nss:
        w.apply(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
    throttles = [rand_throttle(rng, i, nss) for i in range(n_thr)]
    for t in throttles:
        if t["kind"] == "Throttle":
            for term in t["spec"]["selector"]["selectorTerms"]:
                term.pop("namespaceSelector", None)
    # every selector the stream swaps in was applied once: the dictionaries hold its keys and values
    pool = {k: [copy.deepcopy(t["spec"]["selector"]) for t in throttles if t["kind"] == k] for k in ("Throttle", "ClusterThrottle")}
    w.apply(*throttles)
    live = {i: True for i in range(n_thr)}
    pods = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(40)]
    w.apply(*pods)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(30)]
    w.apply(*queue)
    reserved, seen = [], {"delete": 0, "edit": 0, "flip": 0, "grow": 0, "create": 0, "delta": 0, "full": 0}

    def send(t):
        if batched:
            w.events([{"type": "MODIFIED", "object": t}])
        else:
            w.apply(t)

    for step in range(steps):
        op = rng.random()
        where = (seed, step)
        if op < 0.42:  # a deletion, a re-creation or a selector / throttlerName edit
            i = rng.randrange(n_thr)
            t = strip_status(throttles[i])
            kind, name, ns = t["kind"], t["metadata"]["name"], t["metadata"].get("namespace", "")
            what = "create" if not live[i] else rng.choice(["delete", "delete", "edit", "edit", "flip", "grow"])
            if what == "edit":
                t["spec"]["selector"] = copy.deepcopy(rng.choice(pool[kind]))
                if rng.random() < 0.3:
                    t["spec"]["threshold"] = rand_amount(rng)
            elif what == "flip":
                t["spec"]["throttlerName"] = "foreign" if t["spec"]["throttlerName"] == THROTTLER else THROTTLER
            elif what == "grow":  # a label value no selector mentioned before
                term = {"podSelector": {"matchLabels": {"app": f"v{seed}-{step}"}}}
                if kind == "ClusterThrottle":
                    term["namespaceSelector"] = {}
                t["spec"]["selector"] = {"selectorTerms": [term]}
            changed = what in ("delete", "create", "grow") or (t["spec"]["selector"], t["spec"]["throttlerName"]) != \
                (throttles[i]["spec"]["selector"], throttles[i]["spec"]["throttlerName"])
            dut.prefilter_queue()
            full.prefilter_queue()
            st = dut.queue_stats()
            cnt.mark()
            if what == "delete":
                w.delete(kind, name, ns)
                live[i] = False
            else:
                throttles[i] = t
                live[i] = True
                send(t)
            dut.prefilter_queue()
            c = cnt.since()
            seen[what] += 1
            if c is not None and changed:
                holes = st["throttleColumns"] - st["liveThrottles"] + 1
                if what in ("edit", "flip") or (what == "delete" and 2 * holes <= st["throttleColumns"]):
                    # (no call yet when the queue is answered from the cache: the column goes with the next sync)
                    assert c["update_selector_rows"] <= 1 and c["upload_throttles"] == 0, (where, what, c)
                    seen["delta"] += c["update_selector_rows"]
                else:  # a creation, vocabulary growth, or more than half the columns holes
                    assert c["upload_throttles"] == 1 and c["update_selector_rows"] == 0, (where, what, st, c)
                    seen["full"] += 1
        elif op < 0.48:  # a threshold edit of a live throttle
            i = rng.choice([j for j in live if live[j]] or [0])
            if live[i]:
                t = strip_status(throttles[i])
                t["spec"]["threshold"] = rand_amount(rng)
                throttles[i] = t
                send(t)
        elif op < 0.53:  # a Namespace relabel
            w.apply(namespace(rng.choice(nss), {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
        elif op < 0.65:  # reconcile(key) of a few throttles, then the informer echoes every status it wrote
            keys = [nn_of(t) for t in rng.sample(throttles, rng.randint(1, 4))]
            got = w.reconcile(keys, rng.choice(TIMES))
            w.echo([k for k in got["changed"]])
        elif op < 0.75:  # PreFilter, and Reserve on Success
            p = rng.choice(queue)
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if dut.queue_row(*k) >= 0 and ref.prefilter(p)["code"] == "Success":
                assert ref.reserve(p)["code"] == dut.reserve_key(*k)["code"] == full.reserve_key(*k)["code"] == "Success", where
                reserved.append(p)
        elif op < 0.8:  # another writer's status, spec unchanged
            i = rng.randrange(n_thr)
            if live[i]:
                w.apply(dict(throttles[i], status=rand_status(rng)))
        elif op < 0.86 and reserved:  # bind
            p = reserved.pop(rng.randrange(len(reserved)))
            queue.remove(p)
            p = dict(p, spec=dict(p["spec"], nodeName="node-2"), status={"phase": rng.choice(["Running", "Running", "Succeeded"])})
            pods.append(p)
            w.apply(p)
        elif op < 0.93:
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
def test_selector_stream(key_oracle, plugins, seed):
    seen = run_stream(key_oracle, *plugins, seed)
    assert seen["delete"] >= 1 and seen["edit"] + seen["flip"] >= 1 and seen["create"] >= 1, seen
    if getattr(plugins[0], "calls", None):
        assert seen["delta"] >= 3 and seen["full"] >= 1, seen


@pytest.mark.parametrize("seed", [10, 11])
def test_selector_stream_batched(key_oracle, plugins, seed):
    """The same kind of stream with every edit through kth_apply_events."""
    seen = run_stream(key_oracle, *plugins, seed, batched=True)
    assert seen["delete"] + seen["edit"] + seen["flip"] >= 2, seen


def test_selector_delta_voids_only_its_pods(key_oracle, host_on_oracle_selector_rows):
    """Throttles in two namespaces, a queued pod in each: after one pass over the queue, a selector edit or a deletion of throttle
    a makes one kt_update_selector_rows and no upload; qb is answered from the cache, qa is checked again.  A selector with a new
    label value, a re-creation and a deletion past half the columns upload the throttles whole."""
    make = host_on_oracle_selector_rows
    ref, dut = key_oracle(), make(THROTTLER, SCHED)
    w = Twin(ref, dut)
    cnt = Counter(make)
    x, y = {"app": "x"}, {"app": "y"}
    w.apply(namespace("na"), namespace("nb"))
    w.apply(throttle("na", "a", x, pod_cnt=1), throttle("na", "a2", y, pod_cnt=5), throttle("nb", "b", x, pod_cnt=1),
            throttle("nb", "b2", y, pod_cnt=5))
    w.apply(pod("na", "run", "100m", x, node="n", phase="Running"), pod("nb", "run", "100m", x, node="n", phase="Running"))
    w.reconcile_all(NOW)
    qa, qb = pod("na", "qa", "100m", x), pod("nb", "qb", "100m", x)
    w.apply(qa, qb)

    def check(p):
        a, b = ref.prefilter(p), dut.prefilter_key(p["metadata"]["namespace"], p["metadata"]["name"])
        assert (a["code"], a["reasons"]) == (b["code"], b["reasons"]), (a, b)
        return b

    def delta(apply, n_selector, n_upload):
        dut.prefilter_queue()
        cnt.mark()
        before = dut.queue_stats()
        apply()
        check(qb)
        mid = dut.queue_stats()
        assert mid["passes"] == before["passes"] and mid["hits"] == before["hits"] + 1, (before, mid)
        check(qa)
        assert dut.queue_stats()["passes"] == mid["passes"] + 1
        c = cnt.since()
        assert c["update_selector_rows"] == n_selector and c["upload_throttles"] == n_upload, c
        assert c["upload_status"] == 0 and c["set_reserved"] == 0, c

    # a's selector swapped for a2's (the dictionaries hold app=y): qa is no longer throttled by a
    delta(lambda: w.apply(throttle("na", "a", y, pod_cnt=1)), 1, 0)
    assert check(qa)["code"] == "Success"
    delta(lambda: w.apply(throttle("na", "a", x, pod_cnt=1)), 1, 0)  # and back
    assert check(qa)["code"] != "Success"
    delta(lambda: w.apply(throttle("na", "a", x, pod_cnt=1, throttler="foreign")), 1, 0)  # responsibility off
    delta(lambda: w.apply(throttle("na", "a", x, pod_cnt=1)), 1, 0)  # and on
    delta(lambda: w.delete("Throttle", "a", "na"), 1, 0)  # a hole: 1 of 4 columns
    assert check(qa)["code"] == "Success"
    st = dut.queue_stats()
    assert st["throttleColumns"] == 4 and st["liveThrottles"] == 3, st
    # the whole path: a new label value, then a re-creation (which compacts the hole), then holes past half
    for f in (lambda: w.apply(throttle("na", "a2", {"app": "new"}, pod_cnt=5)), lambda: w.apply(throttle("na", "a", x, pod_cnt=1))):
        cnt.mark()
        f()
        check(qa)
        c = cnt.since()
        assert c["upload_throttles"] == 1 and c["update_selector_rows"] == 0, c
    assert dut.queue_stats()["throttleColumns"] == 4
    cnt.mark()
    w.delete("Throttle", "a", "na")
    w.delete("Throttle", "a2", "na")
    w.delete("Throttle", "b2", "nb")  # 3 holes of 4 columns
    check(qb)
    c = cnt.since()
    assert c["update_selector_rows"] == 0 and c["upload_throttles"] == 1, c  # the third hole passes half: the whole path
    assert dut.queue_stats()["throttleColumns"] == 1
    w.compare([qa, qb], "end")
    dut.close()
    ref.close()
