"""Throttle and ClusterThrottle creations on the column path: a creation whose selectors mention only known label keys and values
(and, for a Throttle, a namespace the plugin already knows) fills a hole or is appended at the end (kt_append_throttle_rows),
placed so that it adds no 32-throttle word to any namespace's word list beyond what it must; it neither re-lays out the columns
nor voids the cached PreFilter verdicts of the whole scheduling queue.

Random streams interleave creations of new names, re-creations of deleted names, deletions, selector and threshold edits,
Namespace relabels, pod events, reconciles with their echoes and PreFilter / Reserve by key; some streams go through
kth_apply_events.  After every step the plugin must agree with the object oracle and, result for result, with a twin plugin fed
the same events that uploads the throttles whole for every creation (on the CPU an engine double without the call, on the GPU
a build of the host layer without it).  On the engine double that counts its calls (CPU), in-group and new-group creations
make no kt_upload_throttles, out-of-group and out-of-vocabulary creations make one, and only the queued pods of the namespaces
a new throttle can reach are checked again."""
import copy
import functools
import os
import random

import pytest

from test_plugin_vs_oracle import VALS, rand_amount, rand_labels, rand_pod, rand_status, rand_throttle
from test_reconcile_keys import TIMES, Twin, _build, key_oracle, nn_of  # noqa: F401 (fixtures)
from test_scenarios import NOW, SCHED, THROTTLER, namespace, pod, throttle
from test_selector_rows_host import SelectorTwin, strip_status
from test_threshold_rows_host import HOST_DEPS, ORACLE_DEPS, ORACLE_LINK, ROOT, STUB, Counter, _counting


@pytest.fixture(scope="module")
def host_on_oracle_append_rows(oracle):
    """kt_host.cc linked against the oracle-backed engine double with the column appends and call counters
    (tests/host_stub/engine_oracle_append_rows.cc); host.Plugin's signature plus `.calls()`."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_append_rows.cc")]
    deps = ORACLE_DEPS + [os.path.join(STUB, f) for f in ("engine_oracle_threshold_rows.cc", "engine_oracle_selector_rows.cc")] + HOST_DEPS
    lib = _build("libkt_hostoracle_append_rows.so", srcs, deps, ORACLE_LINK)
    make = functools.partial(host.Plugin, library=lib)
    counted = _counting(lib, ("kt_test_threshold_calls", "kt_test_selector_calls", "kt_test_append_calls"))

    def calls():
        got = counted()
        got["update_selector_rows"] = lib.kt_test_selector_calls()
        got["append_throttle_rows"] = lib.kt_test_append_calls()
        return got

    make.calls = calls
    return make


@pytest.fixture(scope="module")
def host_on_oracle_whole_creations(oracle):
    """The same host layer on the engine double without kt_append_throttle_rows (engine_oracle_selector_rows.cc): every creation
    uploads the throttles whole."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_selector_rows.cc")]
    deps = ORACLE_DEPS + [os.path.join(STUB, "engine_oracle_threshold_rows.cc")] + HOST_DEPS
    lib = _build("libkt_hostoracle_selector_rows.so", srcs, deps, ORACLE_LINK)
    return functools.partial(host.Plugin, library=lib)


@pytest.fixture(scope="module")
def product_full_creations(kt):
    """kt_host.cc linked against the product library but built without its kt_append_throttle_rows reference
    (tests/host_stub/no_append_rows.h): the same device calls as host.Plugin, with every creation uploaded whole."""
    from kube_throttler_b200 import host

    pkg = os.path.join(ROOT, "kube_throttler_b200")
    srcs = [os.path.join(pkg, "csrc", "kt_host.cc")]
    deps = [os.path.join(STUB, "no_append_rows.h"), os.path.join(pkg, "libkt_b200.so")] + HOST_DEPS
    lib = _build("libkt_host_full_creations.so", srcs, deps,
                 ["-Dkt_append_throttle_rows=kt_append_throttle_rows_absent", "-include", os.path.join(STUB, "no_append_rows.h"),
                  "-L", pkg, "-lkt_b200", "-Wl,-rpath," + pkg])
    return functools.partial(host.Plugin, library=lib)


@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def plugins(request):
    """(the plugin on the column path, its twin on whole throttle uploads for creations)"""
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle_append_rows"), request.getfixturevalue("host_on_oracle_whole_creations")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin, request.getfixturevalue("product_full_creations")


def run_stream(key_oracle, new_plugin, full_plugin, seed, steps=90, n_ns=4, batched=False):
    rng = random.Random(seed)
    ref, dut, full = key_oracle(), new_plugin(THROTTLER, SCHED), full_plugin(THROTTLER, SCHED)
    w = SelectorTwin(ref, dut, full)
    cnt = Counter(new_plugin)
    nss = [f"ns{i}" for i in range(n_ns)]
    for n in nss:
        w.apply(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
    throttles = {}
    for i in range(6):
        throttles[i] = rand_throttle(rng, i, nss)
    w.apply(*throttles.values())
    live = {i: True for i in throttles}
    pods = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(40)]
    w.apply(*pods)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(30)]
    w.apply(*queue)
    reserved, seen = [], {"create": 0, "recreate": 0, "delete": 0, "delta": 0, "full": 0}

    def send(t):
        if batched:
            w.events([{"type": "ADDED", "object": t}])
        else:
            w.apply(t)

    for step in range(steps):
        op = rng.random()
        where = (seed, step)
        if op < 0.4:  # a creation of a new name, a re-creation or a deletion
            dead = [i for i in live if not live[i]]
            what = rng.choice(["create", "create", "recreate", "delete"] if dead else ["create", "create", "delete"])
            dut.prefilter_queue()
            full.prefilter_queue()
            cnt.mark()
            if what == "create":
                i = len(throttles)
                throttles[i] = rand_throttle(rng, i, nss)
                live[i] = True
                send(throttles[i])
            elif what == "recreate":
                i = rng.choice(dead)
                live[i] = True
                send(strip_status(throttles[i]))
            else:
                i = rng.choice([j for j in live if live[j]] or [0])
                if live[i]:
                    t = throttles[i]
                    w.delete(t["kind"], t["metadata"]["name"], t["metadata"].get("namespace", ""))
                    live[i] = False
            dut.prefilter_queue()
            c = cnt.since()
            seen[what] += 1
            if c is not None and what != "delete":
                assert c["append_throttle_rows"] <= 1 and c["upload_throttles"] <= 1, (where, c)
                seen["delta" if c["upload_throttles"] == 0 else "full"] += 1
        elif op < 0.46:  # a threshold edit of a live throttle
            i = rng.choice([j for j in live if live[j]] or [0])
            if live[i]:
                t = strip_status(throttles[i])
                t["spec"]["threshold"] = rand_amount(rng)
                throttles[i] = t
                send(t)
        elif op < 0.52:  # a Namespace relabel
            w.apply(namespace(rng.choice(nss), {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
        elif op < 0.64:  # reconcile(key) of a few throttles, then the informer echoes every status it wrote
            keys = [nn_of(t) for t in rng.sample(list(throttles.values()), rng.randint(1, 4))]
            got = w.reconcile(keys, rng.choice(TIMES))
            w.echo([k for k in got["changed"]])
        elif op < 0.76:  # PreFilter, and Reserve on Success
            p = rng.choice(queue)
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if dut.queue_row(*k) >= 0 and ref.prefilter(p)["code"] == "Success":
                assert ref.reserve(p)["code"] == dut.reserve_key(*k)["code"] == full.reserve_key(*k)["code"] == "Success", where
                reserved.append(p)
        elif op < 0.8:  # another writer's status, spec unchanged
            i = rng.choice(list(throttles))
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
def test_creation_stream(key_oracle, plugins, seed):
    seen = run_stream(key_oracle, *plugins, seed)
    assert seen["create"] >= 5 and seen["recreate"] + seen["delete"] >= 3, seen
    if getattr(plugins[0], "calls", None):
        assert seen["delta"] >= 3, seen


@pytest.mark.parametrize("seed", [10, 11])
def test_creation_stream_batched(key_oracle, plugins, seed):
    """The same kind of stream with every creation and edit through kth_apply_events."""
    seen = run_stream(key_oracle, *plugins, seed, batched=True)
    assert seen["create"] >= 5, seen


def test_creation_delta_voids_only_reachable_pods(key_oracle, host_on_oracle_append_rows):
    """Throttles in two namespaces, a queued pod in each: after one pass over the queue, creations that fill a hole of their
    group, append behind their group or start a new group make one kt_append_throttle_rows or column deltas and no upload; qb (in
    the other namespace) is answered from the cache, qa is checked again.  A creation whose group already has a word but neither
    a hole there nor room at the end, and one with a new label value, upload the throttles whole."""
    make = host_on_oracle_append_rows
    ref, dut = key_oracle(), make(THROTTLER, SCHED)
    w = Twin(ref, dut)
    cnt = Counter(make)
    x, y = {"app": "x"}, {"app": "y"}
    w.apply(namespace("na"), namespace("nb"), namespace("nc"))
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

    def delta(apply, n_append):
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
        assert c["append_throttle_rows"] == n_append and c["upload_throttles"] == 0, c
        assert c["upload_status"] == 0 and c["set_reserved"] == 0, c

    # in-group: a third Throttle of na, appended behind the group (the last word holds na's columns and has room)
    delta(lambda: w.apply(throttle("na", "a3", x, pod_cnt=2)), 1)
    assert dut.queue_stats()["throttleColumns"] == 5
    # a deletion leaves a hole; a re-creation of the same name in na fills it (a hole in a word of its group)
    delta(lambda: w.delete("Throttle", "a", "na"), 0)
    assert check(qa)["code"] == "Success"
    delta(lambda: w.apply(throttle("na", "a", x, pod_cnt=1)), 0)
    assert dut.queue_stats()["throttleColumns"] == 5
    # a new group: a Throttle of nc (no queued pod there: both verdicts stay cached)
    dut.prefilter_queue()
    cnt.mark()
    before = dut.queue_stats()
    w.apply(throttle("nc", "c", x, pod_cnt=1))
    check(qa)
    check(qb)
    assert dut.queue_stats()["passes"] == before["passes"] and dut.queue_stats()["hits"] == before["hits"] + 2
    w.reconcile(["nc/c"], NOW)  # (the cached verdicts sent nothing yet: the column goes with the next sync)
    c = cnt.since()
    assert c["append_throttle_rows"] == 1 and c["upload_throttles"] == 0, c
    # the whole path: a new label value; then a creation in na when na has words but no hole there and the last word is nb's
    cnt.mark()
    w.apply(throttle("na", "a4", {"app": "new"}, pod_cnt=5))
    check(qa)
    c = cnt.since()
    assert c["upload_throttles"] == 1 and c["append_throttle_rows"] == 0, c
    w.apply(*[throttle("nb", f"b{i}", y, pod_cnt=5) for i in range(3, 40)])  # the last word: nb's columns only
    check(qa)
    cnt.mark()
    w.apply(throttle("na", "a5", x, pod_cnt=3))  # na has words, but no hole there and the last word is not na's
    check(qa)
    c = cnt.since()
    assert c["upload_throttles"] == 1 and c["append_throttle_rows"] == 0, c
    w.compare([qa, qb], "end")
    dut.close()
    ref.close()
