"""kth_apply_events: a batch of informer watch events applied in order, with the reconcile keys the reference's handlers enqueue
for each one (throttle_controller.go:401-531, clusterthrottle_controller.go:429-563).

Random worlds and event streams, cut into batches of 1 to about 50 events (pod adds, binds, phase changes to finished, relabels,
deletes of bound and unbound pods, other schedulers' pods, throttle creations / edits / deletions with broken podSelectors and
other throttlers, namespace relabels and deletes, unknown objects).  For every event the keys must be the oracle's set at that
moment (tests/host_stub/oracle_events.cc), in creation order.  After every batch the plugin must be in the state a twin plugin
fed the same events one by one through kth_apply / kth_delete is in, and reconciling exactly the returned keys must leave the
plugin and the oracle's per-key reconcile agreeing.  On the engine test double (CPU), every run of pod events that needs the
affected throttles costs exactly one kt_match_pods and no kt_evaluate; a run of pods that are not counted costs nothing."""
import ctypes as C
import functools
import json
import os
import random

import pytest

from test_plugin_vs_oracle import CPUS, VALS, norm_amount, norm_status, rand_labels, rand_pod, rand_throttle
from test_reconcile_keys import BROKEN, TIMES, KeyWorld, _build, parse_metrics
from test_scenarios import SCHED, THROTTLER, namespace, pod, throttle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUB = os.path.join(ROOT, "tests", "host_stub")


@pytest.fixture(scope="module")
def host_on_oracle_match_pods(oracle):
    """kt_host.cc linked against the oracle-backed engine test double plus its kt_match_pods
    (tests/host_stub/engine_oracle_match_pods.cc); host.Plugin's signature plus the double's call counter."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_match_pods.cc")]
    deps = [os.path.join(STUB, f) for f in ("engine_oracle.cc", "engine_oracle_reconcile.cc")] + [os.path.join(ROOT, "oracle", "libkt_oracle.so")] + \
        [os.path.join(ROOT, "kube_throttler_b200", "csrc", f) for f in ("kt_json.h", "kt_quantity.h")] + \
        [os.path.join(ROOT, "include", f) for f in ("kt_b200.h", "kt_host.h")]
    lib = _build("libkt_hostoracle_match_pods.so", srcs, deps,
                 ["-L", os.path.join(ROOT, "oracle"), "-lkt_oracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    lib.kt_test_device_calls.argtypes = [C.POINTER(C.c_int64)]
    lib.kt_test_device_calls.restype = None

    def calls():
        out = (C.c_int64 * 2)()
        lib.kt_test_device_calls(out)
        return out[0], out[1]

    make = functools.partial(host.Plugin, library=lib)
    make.device_calls = calls
    return make


@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def new_plugin(request):
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle_match_pods")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin


class EventWorld(KeyWorld):
    """The object oracle with reconcile by key and the keys each watch event enqueues."""

    def event(self, e):
        return self._j(self.L.ko_world_event(self.h, json.dumps(e).encode()))["keys"]


@pytest.fixture(scope="module")
def events_oracle(oracle):
    srcs = [os.path.join(STUB, "oracle_events.cc")]
    deps = [os.path.join(STUB, "oracle_reconcile_key.cc")] + \
        [os.path.join(ROOT, "oracle", f) for f in ("ko_capi.cc", "ko_model.h", "ko_quantity.h", "ko_json.h", "ko_columnar.h")]
    L = _build("libko_events.so", srcs, deps, ["-pthread"])
    cp, vp = C.c_char_p, C.c_void_p
    L.ko_world_new.restype = vp
    L.ko_world_new.argtypes = [cp, cp]
    L.ko_world_free.argtypes = [vp]
    for name, args in (("ko_world_apply", [vp, cp]), ("ko_world_delete_pod", [vp, cp, cp]), ("ko_world_delete_namespace", [vp, cp]),
                       ("ko_world_delete_throttle", [vp, C.c_int, cp, cp]), ("ko_world_get_status", [vp, cp, cp]), ("ko_world_prefilter", [vp, cp]),
                       ("ko_world_reserve", [vp, cp]), ("ko_world_reserved", [vp, C.c_int, cp]), ("ko_world_reconcile_key", [vp, C.c_int, cp, cp, cp]),
                       ("ko_world_event", [vp, cp])):
        getattr(L, name).argtypes = args
        getattr(L, name).restype = cp
    return lambda: EventWorld(L)


def nn_of(m):
    return m["metadata"].get("namespace", "") + "/" + m["metadata"]["name"]


def counted(p):
    return p["spec"].get("schedulerName") == SCHED and bool(p["spec"].get("nodeName"))


def one_by_one(twin, e):
    """What kth_apply / kth_delete return for the event (an {"error": ...} entry in place of an exception)."""
    obj = e["object"]
    try:
        if e["type"] == "DELETED":
            md = obj["metadata"]
            twin.delete(obj["kind"], md["name"], md.get("namespace", ""))
            return {"ok": True}
        return twin.apply(obj)
    except RuntimeError as ex:
        return {"error": str(ex)}


class Model:
    """What the plugin holds, as far as the keys' order and the device calls of a batch depend on it."""

    def __init__(self):
        self.pods, self.thr_seq, self.seq = {}, {}, 0

    def runs_needing_match(self, batch):
        """The number of runs of pod events (cut at every Throttle / ClusterThrottle / Namespace event) that need the affected
        throttles of some pod version -- the number of kt_match_pods calls the batch makes (throttles exist throughout)."""
        runs, need = 0, False
        for e in batch:
            kind = e["object"]["kind"]
            if kind in ("Throttle", "ClusterThrottle", "Namespace"):
                runs, need = runs + need, False
                continue
            if kind != "Pod":
                continue
            key, old = nn_of(e["object"]), self.pods.get(nn_of(e["object"]))
            if e["type"] == "DELETED":
                need |= old is not None and counted(old)
                self.pods.pop(key, None)
            else:
                need |= counted(e["object"]) or (old is not None and counted(old))
                self.pods[key] = e["object"]
        return runs + need

    def note_throttle(self, e):
        key = (e["object"]["kind"], nn_of(e["object"]))
        if e["type"] == "DELETED":
            self.thr_seq.pop(key, None)
        elif key not in self.thr_seq:
            self.seq += 1
            self.thr_seq[key] = self.seq

    def creation_order(self, keys):
        def seq(k):
            kind = "ClusterThrottle" if k.startswith("/") else "Throttle"
            return self.thr_seq[(kind, k)]
        return sorted(keys, key=seq)


def compare(dut, twin, ref, throttles, queue, where, with_ref):
    """dut against the twin (statuses, reservations, PreFilter by key, affectedPods, metrics) and, after a reconcile of the same
    keys on all three, against the oracle (statuses, reservations, PreFilter by key)."""
    for t in throttles:
        md, nn = t["metadata"], nn_of(t)
        ns = md.get("namespace", "")
        try:
            a = norm_status(dut.status(md["name"], ns))
        except RuntimeError as e:
            a = str(e)
        try:
            b = norm_status(twin.status(md["name"], ns))
        except RuntimeError as e:
            b = str(e)
        assert a == b, (where, nn, a, b)
        ra, rb = dut.reserved(t["kind"], nn), twin.reserved(t["kind"], nn)
        assert sorted(ra["pods"]) == sorted(rb["pods"]) and norm_amount(ra["amount"]) == norm_amount(rb["amount"]), (where, nn, ra, rb)
        for w in (dut, twin):
            try:
                w._aff = w.affected_pods(md["name"], ns)
            except RuntimeError as e:
                w._aff = str(e)
        assert dut._aff == twin._aff, (where, nn)
        if with_ref and isinstance(a, dict):
            try:
                c = norm_status(ref.status(md["name"], ns))
            except RuntimeError:
                c = None
            if c is not None:
                assert a == c, (where, nn, a, c)
            rc = ref.reserved(t["kind"], nn)
            assert sorted(ra["pods"]) == sorted(rc["pods"]) and norm_amount(ra["amount"]) == norm_amount(rc["amount"]), (where, nn, ra, rc)
    for p in queue:
        k = (p["metadata"]["namespace"], p["metadata"]["name"])
        if dut.queue_row(*k) < 0:
            continue
        a, b = dut.prefilter_key(*k), twin.prefilter_key(*k)
        assert a == b, (where, k, a, b)
        if with_ref:
            c = ref.prefilter(p)
            assert (a["code"], a["reasons"]) == (c["code"], c["reasons"]), (where, k, a, c)
    assert parse_metrics(dut.metrics()) == parse_metrics(twin.metrics()), where


def random_event(rng, st, step):
    """One watch event of the stream; st holds the generator's view of the world."""
    nss, throttles, running, queue = st["nss"], st["throttles"], st["running"], st["queue"]
    op = rng.random()
    if op < 0.14:  # a new pod: queued, running, or another scheduler's
        p = rand_pod(rng, rng.choice(nss + ["nsx"]), f"n{step}", rng.random() < 0.5)
        (running if p["spec"]["nodeName"] else queue).append(p)
        return {"type": "ADDED", "object": p}
    if op < 0.26 and queue:  # bind
        p = queue.pop(rng.randrange(len(queue)))
        p = dict(p, spec=dict(p["spec"], nodeName="node-2"), status={"phase": "Running"})
        running.append(p)
        return {"type": "MODIFIED", "object": p}
    if op < 0.42 and running:  # relabel, maybe finish
        i = rng.randrange(len(running))
        p = json.loads(json.dumps(running[i]))
        if rng.random() < 0.8:
            p["metadata"]["labels"] = rand_labels(rng)
        if rng.random() < 0.3:
            p["status"] = {"phase": rng.choice(["Running", "Succeeded", "Failed"])}
        running[i] = p
        return {"type": "MODIFIED", "object": p}
    if op < 0.5 and queue:  # relabel of a queued pod
        i = rng.randrange(len(queue))
        p = json.loads(json.dumps(queue[i]))
        p["metadata"]["labels"] = rand_labels(rng)
        queue[i] = p
        return {"type": "MODIFIED", "object": p}
    if op < 0.6 and running:  # delete of a bound pod
        p = running.pop(rng.randrange(len(running)))
        return {"type": "DELETED", "object": p}
    if op < 0.64 and len(queue) > 5:  # delete of an unbound pod
        p = queue.pop(rng.randrange(len(queue)))
        return {"type": "DELETED", "object": p}
    if op < 0.76:  # throttle edit or (re)creation, sometimes a broken podSelector
        i = rng.randrange(len(throttles))
        t = rand_throttle(rng, i, nss)
        t["kind"], t["metadata"] = throttles[i]["kind"], throttles[i]["metadata"]
        if t["kind"] == "Throttle":
            for term in t["spec"]["selector"]["selectorTerms"]:
                term.pop("namespaceSelector", None)
        if t["spec"]["selector"]["selectorTerms"] and rng.random() < 0.25:
            rng.choice(t["spec"]["selector"]["selectorTerms"])["podSelector"] = rng.choice(BROKEN)
        throttles[i] = t
        return {"type": rng.choice(["ADDED", "MODIFIED"]), "object": t}
    if op < 0.8:  # throttle deletion (maybe of one that is gone already)
        return {"type": "DELETED", "object": rng.choice(throttles)}
    if op < 0.9:  # namespace relabel or delete
        n = rng.choice(nss)
        if rng.random() < 0.25:
            return {"type": "DELETED", "object": namespace(n)}
        return {"type": "MODIFIED", "object": namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)})}
    if op < 0.93:  # an unknown pod goes away
        return {"type": "DELETED", "object": pod(rng.choice(nss), "ghost")}
    p = rand_pod(rng, rng.choice(nss), f"c{step}", True)  # a counted pod with a new cpu request
    p["spec"]["containers"][0]["resources"]["requests"]["cpu"] = rng.choice(CPUS)
    running.append(p)
    return {"type": "ADDED", "object": p}


def run_stream(events_oracle, new_plugin, seed, batches=12, n_thr=12):
    rng = random.Random(seed)
    ref, dut, twin = events_oracle(), new_plugin(THROTTLER, SCHED), new_plugin(THROTTLER, SCHED)
    model = Model()
    nss = [f"ns{i}" for i in range(4)]
    st = {"nss": nss, "throttles": [rand_throttle(rng, i, nss) for i in range(n_thr)],
          "running": [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(50)],
          "queue": [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(25)]}
    initial = [{"type": "ADDED", "object": namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)})} for n in nss] + \
        [{"type": "ADDED", "object": t} for t in st["throttles"]] + \
        [{"type": "ADDED", "object": p} for p in st["running"] + st["queue"]]
    stats = {"events": 0, "keys": 0, "runs": 0}
    step = 0
    for b in range(batches + 1):
        if b == 0:
            batch = initial  # the informers' initial list: one batch
        else:
            batch = []
            for _ in range(rng.randint(1, 50)):
                batch.append(random_event(rng, st, step))
                step += 1
        want_runs = model.runs_needing_match(batch)
        calls0 = new_plugin.device_calls() if hasattr(new_plugin, "device_calls") else None
        got = dut.apply_events(batch)
        if calls0 is not None:
            calls1 = new_plugin.device_calls()
            assert (calls1[0] - calls0[0], calls1[1] - calls0[1]) == (want_runs, 0), (seed, b, calls0, calls1, want_runs)
        assert len(got["results"]) == len(batch), (seed, b)
        union = []
        for i, (e, entry) in enumerate(zip(batch, got["results"])):
            where = (seed, b, i, e["type"], e["object"]["kind"], nn_of(e["object"]))
            want_keys = ref.event(e)
            plain = one_by_one(twin, e)
            if e["object"]["kind"] in ("Throttle", "ClusterThrottle"):
                model.note_throttle(e)  # (a throttle event enqueues at most its own key: no order to check)
            if "error" in plain:
                assert set(entry) == {"error"}, (where, entry, plain)
                continue
            assert {k: v for k, v in entry.items() if k != "enqueue"} == plain, (where, entry, plain)
            assert sorted(entry["enqueue"]) == sorted(want_keys), (where, entry["enqueue"], want_keys)
            if len(entry["enqueue"]) > 1:
                assert entry["enqueue"] == model.creation_order(entry["enqueue"]), (where, entry["enqueue"])
            union += [k for k in entry["enqueue"] if k not in union]
        assert got["enqueue"] == union, (seed, b)
        stats["events"] += len(batch)
        stats["keys"] += len(union)
        stats["runs"] += want_runs
        where = (seed, b)
        compare(dut, twin, ref, st["throttles"], st["queue"], where, with_ref=False)
        now = rng.choice(TIMES)
        rd, rt = dut.reconcile(union, now), twin.reconcile(union, now)
        assert rd == rt, (where, rd, rt)
        for k in union:
            ns, _, name = k.partition("/")
            ref.reconcile_key("ClusterThrottle" if ns == "" else "Throttle", ns, name, now)
        compare(dut, twin, ref, st["throttles"], st["queue"], where, with_ref=True)
    dut.close(), twin.close(), ref.close()
    return stats


@pytest.mark.parametrize("seed", [0, 1, 2, 3, 4])
def test_event_stream(events_oracle, new_plugin, seed):
    stats = run_stream(events_oracle, new_plugin, seed)
    assert stats["keys"] > 20 and stats["runs"] > 5, stats


def test_device_calls_per_run(host_on_oracle_match_pods):
    """One kt_match_pods per run that needs matching, none for the queue's churn, none for throttle and namespace events."""
    make = host_on_oracle_match_pods
    dut = make(THROTTLER, SCHED)
    lbl = {"app": "x"}
    dut.apply_events([{"type": "ADDED", "object": o} for o in (namespace("na"), throttle("na", "t1", lbl, pod_cnt=5))])
    c0 = make.device_calls()
    queued = [pod("na", f"q{i}", "100m", lbl) for i in range(20)] + [pod("na", "other", "100m", lbl, node="n1", scheduler="other")]
    out = dut.apply_events([{"type": "ADDED", "object": p} for p in queued])
    assert make.device_calls() == c0 and out["enqueue"] == [], out
    bound = [dict(p, spec=dict(p["spec"], nodeName="n1"), status={"phase": "Running"}) for p in queued[:4]]
    ev = [{"type": "MODIFIED", "object": p} for p in bound[:2]] + [{"type": "ADDED", "object": namespace("nb")}] + \
        [{"type": "MODIFIED", "object": p} for p in bound[2:]] + [{"type": "DELETED", "object": bound[0]}]
    out = dut.apply_events(ev)
    c1 = make.device_calls()
    assert (c1[0] - c0[0], c1[1] - c0[1]) == (2, 0), (c0, c1)
    assert out["enqueue"] == ["na/t1"] and all(r.get("enqueue") in ([], ["na/t1"]) for r in out["results"]), out
    assert out["results"][2] == {"ok": True, "enqueue": []}
    dut.close()


def test_error_entries(events_oracle, new_plugin):
    """Malformed events, unsupported kinds and refused objects are {"error": ...} entries; the rest of the batch applies and
    enqueues its keys."""
    ref, dut = events_oracle(), new_plugin(THROTTLER, SCHED)
    lbl = {"app": "x"}
    t1 = throttle("na", "t1", lbl, pod_cnt=5)
    foreign = throttle("na", "f1", lbl, pod_cnt=5, throttler="foreign")
    broken = throttle("na", "broken", lbl, pod_cnt=5)
    broken["spec"]["selector"]["selectorTerms"][0]["podSelector"] = BROKEN[0]
    bad_qty = pod("na", "badq", "100m", lbl, node="n1", phase="Running")
    bad_qty["spec"]["containers"][0]["resources"]["requests"]["cpu"] = "12xyz"
    too_many = pod("na", "many", "100m", {f"k{i}": "v" for i in range(40)}, node="n1", phase="Running")
    run1 = pod("na", "run1", "100m", lbl, node="n1", phase="Running")
    run2 = pod("nc", "run2", "100m", lbl, node="n1", phase="Running")  # nc: no such namespace
    ct = {"kind": "ClusterThrottle", "metadata": {"name": "ct"},
          "spec": {"throttlerName": THROTTLER, "threshold": {"resourceCounts": {"pod": 1}},
                   "selector": {"selectorTerms": [{"podSelector": {"matchLabels": lbl}}]}}}
    batch = [{"type": "ADDED", "object": namespace("na")}, {"type": "ADDED", "object": t1}, {"type": "ADDED", "object": foreign},
             {"type": "ADDED", "object": ct}, "not an event", {"type": "BOOKMARK", "object": run1}, {"type": "ADDED"},
             {"type": "ADDED", "object": {"kind": "ConfigMap", "metadata": {"name": "x"}}}, {"type": "ADDED", "object": bad_qty},
             {"type": "ADDED", "object": too_many}, {"type": "ADDED", "object": run1}, {"type": "ADDED", "object": run2},
             {"type": "DELETED", "object": {"kind": "Secret", "metadata": {"name": "s"}}}, {"type": "ADDED", "object": broken},
             {"type": "MODIFIED", "object": dict(run1, metadata=dict(run1["metadata"], labels={"app": "y"}))},
             {"type": "DELETED", "object": foreign}, {"type": "DELETED", "object": t1}, {"type": "DELETED", "object": t1}]
    got = dut.apply_events(batch)
    res = got["results"]
    assert len(res) == len(batch)
    for i in (4, 5, 6, 7, 8, 9, 12):
        assert set(res[i]) == {"error"}, (i, res[i])
    assert "unsupported kind: ConfigMap" in res[7]["error"] and "unsupported kind: Secret" in res[12]["error"]
    assert res[1]["enqueue"] == ["na/t1"] and res[2]["enqueue"] == [] and res[3]["enqueue"] == ["/ct"]
    assert res[10]["enqueue"] == ["na/t1", "/ct"]   # both controllers
    assert res[11]["enqueue"] == []  # nc: no Throttle there, and the ClusterThrottle controller does not find the namespace
    for i, e in enumerate(batch):
        if isinstance(e, dict) and "object" in e and i not in (5, 7, 12) and "error" not in res[i]:
            assert sorted(res[i]["enqueue"]) == sorted(ref.event(e)), (i, res[i])
    assert res[14]["enqueue"] == ["/ct"]  # the Throttle controller hits the broken podSelector for the new version
    assert res[15]["enqueue"] == [] and res[16]["enqueue"] == ["na/t1"] and res[17]["enqueue"] == []
    assert res[13]["enqueue"] == ["na/broken"]
    assert got["enqueue"] == ["na/t1", "/ct", "na/broken"]
    assert dut.apply_events([]) == {"results": [], "enqueue": []}
    assert "JSON array" in json.loads(dut._L.kth_apply_events(dut._h, b'{"type": "ADDED"}').decode())["error"]
    dut.close(), ref.close()
