"""The host layer's column moves: a creation that no hole or end column can take without growing a namespace's word list
(placement rule 4), and a deletion past the "at most half the columns are holes" rule, lay the columns out again through one
kt_move_throttle_columns instead of a whole throttle upload.

Random streams whose groups fill their 32-throttle words -- 70 throttles over two namespaces -- so that creations hit rule 4 and
deletion bursts pass the half-holes rule, mixed with re-creations, threshold edits, Namespace relabels, pod events, reconciles
with their echoes and PreFilter / Reserve by key, some streams through kth_apply_events.  Each stream runs on three plugins: the
move path, a twin on whole uploads for those events and the object oracle; after every step they must answer alike, result for
result, including kth_queue_stats' throttleColumns and wordsPerNamespaceX100.  On the counting engine double
(tests/host_stub/engine_oracle_move_columns.cc) the moves make no kt_upload_throttles, and a creation that brings a label key
the dictionaries lack still makes one."""
import functools
import os
import random

import pytest

from test_plugin_vs_oracle import VALS, rand_amount, rand_pod, rand_throttle
from test_reconcile_keys import TIMES, _build, key_oracle, nn_of  # noqa: F401 (fixtures)
from test_scenarios import SCHED, THROTTLER, namespace
from test_selector_rows_host import SelectorTwin, strip_status
from test_threshold_rows_host import HOST_DEPS, ORACLE_DEPS, ORACLE_LINK, ROOT, STUB, Counter, _counting

DOUBLES = ("engine_oracle_threshold_rows.cc", "engine_oracle_selector_rows.cc", "engine_oracle_append_rows.cc")


@pytest.fixture(scope="module")
def host_on_oracle_move_columns(oracle):
    """kt_host.cc linked against the oracle-backed engine double with the column moves and call counters; host.Plugin's
    signature plus `.calls()`."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_move_columns.cc")]
    deps = ORACLE_DEPS + [os.path.join(STUB, f) for f in DOUBLES] + HOST_DEPS
    lib = _build("libkt_hostoracle_move_columns.so", srcs, deps, ORACLE_LINK)
    make = functools.partial(host.Plugin, library=lib)
    counted = _counting(lib, ("kt_test_threshold_calls", "kt_test_selector_calls", "kt_test_append_calls", "kt_test_move_calls"))

    def calls():
        got = counted()
        got["append_throttle_rows"] = lib.kt_test_append_calls()
        got["move_throttle_columns"] = lib.kt_test_move_calls()
        return got

    make.calls = calls
    return make


@pytest.fixture(scope="module")
def host_on_oracle_whole_moves(oracle):
    """The same host layer on the engine double without kt_move_throttle_columns (engine_oracle_append_rows.cc): rule-4
    creations and compactions upload the throttles whole."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_append_rows.cc")]
    deps = ORACLE_DEPS + [os.path.join(STUB, f) for f in DOUBLES[:2]] + HOST_DEPS
    lib = _build("libkt_hostoracle_append_rows.so", srcs, deps, ORACLE_LINK)
    return functools.partial(host.Plugin, library=lib)


@pytest.fixture(scope="module")
def product_whole_moves(kt):
    """kt_host.cc linked against the product library but built without its kt_move_throttle_columns reference
    (tests/host_stub/no_move_columns.h)."""
    from kube_throttler_b200 import host

    pkg = os.path.join(ROOT, "kube_throttler_b200")
    deps = [os.path.join(STUB, "no_move_columns.h"), os.path.join(pkg, "libkt_b200.so")] + HOST_DEPS
    lib = _build("libkt_host_whole_moves.so", [os.path.join(pkg, "csrc", "kt_host.cc")], deps,
                 ["-Dkt_move_throttle_columns=kt_move_throttle_columns_absent", "-include", os.path.join(STUB, "no_move_columns.h"),
                  "-L", pkg, "-lkt_b200", "-Wl,-rpath," + pkg])
    return functools.partial(host.Plugin, library=lib)


@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def plugins(request):
    """(the plugin on the move path, its twin on whole throttle uploads for those events)"""
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle_move_columns"), request.getfixturevalue("host_on_oracle_whole_moves")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin, request.getfixturevalue("product_whole_moves")


def new_key_throttle(t, n):
    """The throttle with a podSelector on a label key nothing mentioned before."""
    t = strip_status(t)
    t["spec"]["selector"]["selectorTerms"] = [dict(t["spec"]["selector"]["selectorTerms"][0] if t["spec"]["selector"]["selectorTerms"] else {},
                                                   podSelector={"matchLabels": {f"fresh-{n}": "x"}})]
    return t


def run_stream(key_oracle, new_plugin, full_plugin, seed, steps=80, batched=False):
    rng = random.Random(seed)
    ref, dut, full = key_oracle(), new_plugin(THROTTLER, SCHED), full_plugin(THROTTLER, SCHED)
    w = SelectorTwin(ref, dut, full)
    cnt = Counter(new_plugin)
    nss = ["ns0", "ns1"]
    for n in nss:
        w.apply(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
    throttles = {i: rand_throttle(rng, i, nss) for i in range(70)}
    w.apply(*throttles.values())
    live = {i: True for i in throttles}
    pods = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(40)]
    w.apply(*pods)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(30)]
    w.apply(*queue)
    reserved, seen = [], {"create": 0, "move": 0, "compact": 0, "new_key": 0}

    def send(t):
        if batched:
            w.events([{"type": "ADDED", "object": t}])
        else:
            w.apply(t)

    for step in range(steps):
        op = rng.random()
        where = (seed, step)
        if op < 0.45:  # creations, a re-creation, a burst of deletions past half holes, or a creation with a new label key
            what = rng.choice(["create", "create", "create", "recreate", "burst", "new_key"])
            dut.prefilter_queue()
            full.prefilter_queue()
            cnt.mark()
            if what in ("create", "new_key"):
                i = len(throttles)
                throttles[i] = rand_throttle(rng, i, nss) if what == "create" else new_key_throttle(rand_throttle(rng, i, nss), i)
                live[i] = True
                send(throttles[i])
            elif what == "recreate":
                dead = [i for i in live if not live[i]]
                if dead:
                    i = rng.choice(dead)
                    live[i] = True
                    send(strip_status(throttles[i]))
            else:
                alive = [i for i in live if live[i]]
                for i in rng.sample(alive, max(0, min(len(alive) - 3, len(alive) // 2 + 2))):  # (some stay live)
                    t = throttles[i]
                    w.delete(t["kind"], t["metadata"]["name"], t["metadata"].get("namespace", ""))
                    live[i] = False
            dut.prefilter_queue()
            c = cnt.since()
            seen["create"] += what == "create"
            if c is not None:
                assert c["move_throttle_columns"] <= 1, (where, c)  # at most one move per sync
                if c["move_throttle_columns"]:
                    assert c["upload_throttles"] == 0, (where, c)
                    seen["compact" if what == "burst" else "move"] += 1
                if what == "new_key":
                    assert c["upload_throttles"] == 1, (where, c)
                    seen["new_key"] += 1
        elif op < 0.5:  # a threshold edit of a live throttle
            i = rng.choice([j for j in live if live[j]] or [0])
            if live[i]:
                t = strip_status(throttles[i])
                t["spec"]["threshold"] = rand_amount(rng)
                throttles[i] = t
                send(t)
        elif op < 0.56:  # a Namespace relabel
            w.apply(namespace(rng.choice(nss), {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
        elif op < 0.66:  # reconcile(key) of a few throttles, then the informer echoes every status it wrote
            keys = [nn_of(t) for t in rng.sample(list(throttles.values()), rng.randint(1, 4))]
            got = w.reconcile(keys, rng.choice(TIMES))
            w.echo([k for k in got["changed"]])
        elif op < 0.8:  # PreFilter, and Reserve on Success
            p = rng.choice(queue)
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if dut.queue_row(*k) >= 0 and ref.prefilter(p)["code"] == "Success":
                assert ref.reserve(p)["code"] == dut.reserve_key(*k)["code"] == full.reserve_key(*k)["code"] == "Success", where
                reserved.append(p)
        elif op < 0.88 and reserved:  # bind
            p = reserved.pop(rng.randrange(len(reserved)))
            if p not in queue:  # (reserved twice)
                continue
            queue.remove(p)
            p = dict(p, spec=dict(p["spec"], nodeName="node-2"), status={"phase": "Running"})
            pods.append(p)
            w.apply(p)
        else:
            p = rand_pod(rng, rng.choice(nss), f"n{step}", False)
            queue.append(p)
            w.apply(p)
        w.compare(queue, where)
        for key in ("throttleColumns", "wordsPerNamespaceX100"):
            assert dut.queue_stats()[key] == full.queue_stats()[key], (where, key)
    for x in (dut, full, ref):
        x.close()
    return seen


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_move_stream(key_oracle, plugins, seed):
    seen = run_stream(key_oracle, *plugins, seed)
    assert seen["create"] >= 5, seen
    if getattr(plugins[0], "calls", None):
        assert seen["move"] >= 1 and seen["compact"] >= 1 and seen["new_key"] >= 1, seen


@pytest.mark.parametrize("seed", [10])
def test_move_stream_batched(key_oracle, plugins, seed):
    """The same kind of stream with every creation and edit through kth_apply_events."""
    seen = run_stream(key_oracle, *plugins, seed, batched=True)
    assert seen["create"] >= 3, seen
