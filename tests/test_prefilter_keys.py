"""kth_pre_filter_keys: PreFilter by key for a list of pods, checked row by row on the device (kt_check_pending_rows), compared
entry by entry with kth_pre_filter_key and with the object-level oracle's PreFilter.

Random worlds and event streams (both kinds, reservations, relabels, binds, throttle edits with broken podSelectors, namespace
relabels and deletes) call it after every step for a random subset of queued keys plus a pod that is not queued, an unknown key
and a malformed key.  The call must leave the cached queue verdicts (queue_stats passes / hits), statuses, reservations and
affectedPods as they were.  Runs on the product (GPU) and on the product's host layer over an engine test double whose
kt_check_pending_rows is the columnar oracle (CPU)."""
import functools
import json
import os
import random

import pytest

from test_plugin_vs_oracle import VALS, norm_amount, norm_prefilter, norm_status, rand_labels, rand_pod, rand_throttle
from test_reconcile_keys import BROKEN, TIMES, _build
from test_scenarios import NOW, SCHED, THROTTLER, namespace, pod, throttle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUB = os.path.join(ROOT, "tests", "host_stub")


@pytest.fixture(scope="module")
def host_on_oracle_check_rows(oracle):
    """kt_host.cc linked against the oracle-backed engine test double plus its kt_check_pending_rows
    (tests/host_stub/engine_oracle_check_rows.cc); host.Plugin's signature.  CPU only; says nothing about the kernels."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_check_rows.cc")]
    deps = [os.path.join(STUB, "engine_oracle.cc"), os.path.join(ROOT, "oracle", "libkt_oracle.so")] + \
        [os.path.join(ROOT, "kube_throttler_b200", "csrc", f) for f in ("kt_json.h", "kt_quantity.h")] + \
        [os.path.join(ROOT, "include", f) for f in ("kt_b200.h", "kt_host.h")]
    lib = _build("libkt_hostoracle_check_rows.so", srcs, deps,
                 ["-L", os.path.join(ROOT, "oracle"), "-lkt_oracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    return functools.partial(host.Plugin, library=lib)


@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def new_plugin(request):
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle_check_rows")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin


def key_of(p):
    return p["metadata"]["namespace"] + "/" + p["metadata"]["name"]


def by_key(dut, key):
    """kth_pre_filter_key's answer, with its error text in place of an exception (the shape of a kth_pre_filter_keys entry)."""
    ns, _, name = key.partition("/")
    try:
        return dut.prefilter_key(ns, name)
    except RuntimeError as e:
        return {"error": str(e)}


def observe(dut, throttles):
    """Everything a PreFilter must not move: statuses, reservations, affectedPods (or its error) of every throttle."""
    out = []
    for t in throttles:
        md = t["metadata"]
        ns, nn = md.get("namespace", ""), md.get("namespace", "") + "/" + md["name"]
        try:
            st = norm_status(dut.status(md["name"], ns))
        except RuntimeError as e:
            st = str(e)
        try:
            aff = dut.affected_pods(md["name"], ns)
        except RuntimeError as e:
            aff = str(e)
        res = dut.reserved(t["kind"], nn)
        out.append((nn, st, aff, sorted(res["pods"]), norm_amount(res["amount"])))
    return out


def check_keys(ref, dut, keys, manifests, throttles, where):
    """kth_pre_filter_keys(keys) against kth_pre_filter_key key by key and, for queued pods, the oracle's PreFilter."""
    stats0 = dut.queue_stats()
    seen0 = observe(dut, throttles)
    stats1 = dut.queue_stats()  # (affectedPods may run a pass of its own; it touches no cached verdict)
    got = dut.prefilter_keys(keys)
    stats2 = dut.queue_stats()
    assert (stats2["passes"], stats2["hits"]) == (stats1["passes"], stats1["hits"]) == (stats0["passes"], stats0["hits"]), (where, stats0, stats2)
    assert observe(dut, throttles) == seen0, where
    assert len(got) == len(keys), (where, keys, got)
    for key, entry in zip(keys, got):
        ns, slash, name = key.partition("/")
        if not slash or not name or "/" in name:
            assert set(entry) == {"error"} and "unexpected key format" in entry["error"], (where, key, entry)
            continue
        assert entry == by_key(dut, key), (where, key, entry)
        if key in manifests and dut.queue_row(ns, name) >= 0:
            assert norm_prefilter(entry) == norm_prefilter(ref.prefilter(manifests[key])), (where, key, entry)
    return got


def run_stream(oracle, new_plugin, seed, steps=40, n_thr=10):
    rng = random.Random(seed)
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    nss = [f"ns{i}" for i in range(5)]
    both(*[namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}) for n in nss])
    throttles = [rand_throttle(rng, i, nss) for i in range(n_thr)]
    both(*throttles)
    running = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(40)]
    both(*running)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(30)]
    both(*queue)
    reserved, calls = [], 0
    for step in range(steps):
        op = rng.random()
        if op < 0.12:
            now = rng.choice(TIMES)
            try:
                ref.reconcile_all(now)
            except RuntimeError:
                pass
            dut.reconcile_all(now)
        elif op < 0.35 and queue:
            p = rng.choice(queue)
            a = ref.prefilter(p)
            if a["code"] == "Success" and dut.queue_row(*key_of(p).split("/")) >= 0:
                assert ref.reserve(p)["code"] == dut.reserve_key(*key_of(p).split("/"))["code"] == "Success", (seed, step)
                reserved.append(p)
        elif op < 0.45 and reserved:
            p = reserved.pop(rng.randrange(len(reserved)))
            if rng.random() < 0.5:
                queue.remove(p)
                p = dict(p, spec=dict(p["spec"], nodeName="node-9"), status={"phase": "Running"})
                running.append(p)
                both(p)
            else:
                ref.unreserve(p), dut.unreserve_key(*key_of(p).split("/"))
        elif op < 0.55 and queue:
            p = rng.choice(queue)
            p["metadata"]["labels"] = rand_labels(rng)
            both(p)
        elif op < 0.72:
            i = rng.randrange(len(throttles))
            t = rand_throttle(rng, i, nss)
            t["kind"], t["metadata"] = throttles[i]["kind"], throttles[i]["metadata"]
            if t["kind"] == "Throttle":
                for term in t["spec"]["selector"]["selectorTerms"]:
                    term.pop("namespaceSelector", None)
            if t["spec"]["selector"]["selectorTerms"] and rng.random() < 0.2:
                rng.choice(t["spec"]["selector"]["selectorTerms"])["podSelector"] = rng.choice(BROKEN)
            throttles[i] = t
            both(t)
        elif op < 0.8:
            n = rng.choice(nss)
            if rng.random() < 0.3:
                ref.delete("Namespace", n), dut.delete("Namespace", n)
            else:
                both(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
        elif op < 0.86 and len(queue) > 10:
            p = queue.pop(rng.randrange(len(queue)))
            if p in reserved:
                reserved.remove(p)
            ref.delete("Pod", p["metadata"]["name"], p["metadata"]["namespace"]), dut.delete("Pod", p["metadata"]["name"], p["metadata"]["namespace"])
        else:
            p = rand_pod(rng, rng.choice(nss), f"n{step}", False)
            queue.append(p)
            both(p)
        keys = [key_of(p) for p in rng.sample(queue, rng.randint(1, min(8, len(queue))))]
        if keys and rng.random() < 0.3:
            keys.append(rng.choice(keys))  # a duplicate
        keys += [key_of(rng.choice(running)), rng.choice(["ns0/nobody", "ns9/q1"]), rng.choice(["no-slash", "ns0/a/b", "ns0/"])]
        rng.shuffle(keys)
        manifests = {key_of(p): p for p in queue}
        check_keys(ref, dut, keys, manifests, throttles, (seed, step))
        calls += 1
    dut.close()
    ref.close()
    return calls


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_event_stream(oracle, new_plugin, seed):
    assert run_stream(oracle, new_plugin, seed) == 40


@pytest.mark.parametrize("seed", [5, 6])
def test_scheduling_cycle_by_keys(oracle, new_plugin, seed):
    """The scheduler's cycle over a sorted queue -- PreFilter by keys, then Reserve by key on Success -- gives the oracle's
    one-pod-per-cycle results, pod by pod, and the same reservations."""
    rng = random.Random(seed)
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    nss = [f"ns{i}" for i in range(3)]
    both(*[namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}) for n in nss])
    throttles = [rand_throttle(rng, i, nss) for i in range(8)]
    both(*throttles)
    both(*[rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(30)])
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(40)]
    both(*queue)
    admitted = 0
    for p in queue:
        ns, name = p["metadata"]["namespace"], p["metadata"]["name"]
        (got,) = dut.prefilter_keys([key_of(p)])
        if dut.queue_row(ns, name) < 0:
            continue  # another scheduler's pod
        want = ref.prefilter(p)
        assert norm_prefilter(got) == norm_prefilter(want), (seed, key_of(p), got, want)
        if got["code"] == "Success":
            assert ref.reserve(p)["code"] == dut.reserve_key(ns, name)["code"] == "Success"
            admitted += 1
    assert admitted > 0
    for t in throttles:
        k, nn = t["kind"], t["metadata"].get("namespace", "") + "/" + t["metadata"]["name"]
        a, b = ref.reserved(k, nn), dut.reserved(k, nn)
        assert sorted(a["pods"]) == sorted(b["pods"]) and norm_amount(a["amount"]) == norm_amount(b["amount"]), (seed, nn)
    dut.close()
    ref.close()


def test_error_entries(oracle, new_plugin):
    """A broken podSelector in the pod's way and a namespace the lister does not hold are PreFilter Error results, as by key; an
    unknown pod and malformed keys are {"error": ...} entries; an empty list is an empty list."""
    ref, dut = oracle.World(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    both = lambda *m: (ref.apply(*m), dut.apply(*m))
    lbl = {"app": "x"}
    broken = throttle("na", "broken", lbl, pod_cnt=5)
    broken["spec"]["selector"]["selectorTerms"][0]["podSelector"] = BROKEN[0]
    ct = {"kind": "ClusterThrottle", "metadata": {"name": "ct"},
          "spec": {"throttlerName": THROTTLER, "threshold": {"resourceCounts": {"pod": 1}},
                   "selector": {"selectorTerms": [{"podSelector": {"matchLabels": lbl}}]}}}
    both(namespace("na"), namespace("nb"), broken, ct, throttle("nb", "ok", lbl, pod_cnt=1, cpu="1"))
    qa, qb, qc = pod("na", "qa", "100m", lbl), pod("nb", "qb", "100m", lbl), pod("nc", "qc", "100m", lbl)  # nc: no such namespace
    both(qa, qb, qc, pod("nb", "run", "100m", lbl, node="n", phase="Running"))
    ref.reconcile_all(NOW), dut.reconcile_all(NOW)
    keys = ["na/qa", "nb/qb", "nc/qc", "nb/run", "nb/ghost", "bad", "nb/x/y", "nb/"]
    got = check_keys(ref, dut, keys, {key_of(p): p for p in (qa, qb, qc)}, [broken, ct], "errors")
    assert got[0]["code"] == "Error" and got[0]["reasons"] == norm_prefilter(ref.prefilter(qa))["reasons"]
    assert got[2]["code"] == "Error" and got[2]["reasons"] == ['namespace "nc" not found']
    assert got[1]["code"] == "UnschedulableAndUnresolvable"
    assert got[3]["code"] in ("Success", "UnschedulableAndUnresolvable")  # a running pod, checked like a manifest
    assert got[4] == {"error": "pod nb/ghost is not in the informer cache"}
    assert all(set(e) == {"error"} for e in got[5:])
    assert dut.prefilter_keys([]) == []
    assert "JSON array" in json.loads(dut._L.kth_pre_filter_keys(dut._h, b'{"na/qa": 1}').decode())["error"]
    dut.close()
    ref.close()
