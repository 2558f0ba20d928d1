"""kth_reconcile: reconcile(key) for listed throttles only, compared key by key with the object-level oracle's own per-throttle
reconcile (World::reconcile, throttle_controller.go:84-211 / clusterthrottle_controller.go:87-214).

Random worlds and event streams (both kinds, finished pods, reservations, relabels, namespace moves, threshold and override edits,
broken podSelectors) interleave random key subsets -- duplicates, unknown keys, other throttlers' keys, malformed keys -- with
reconcile_all.  After every step every status, reservation, PreFilter by key, gauge and requeueAfterNanos must agree with the
oracle; gauges and requeues are modelled from the oracle's statuses and the specs (the oracle keeps neither).  Runs on the product
(GPU) and on the product's host layer over an engine test double whose kt_reconcile_throttles is the columnar oracle (CPU)."""
import ctypes as C
import datetime
import functools
import json
import math
import os
import random
import subprocess

import pytest

from test_oracle_kat import q
from test_plugin_vs_oracle import CPUS, VALS, norm_amount, norm_status, rand_labels, rand_pod, rand_throttle
from test_scenarios import NOW, SCHED, THROTTLER, namespace, pod, throttle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUB = os.path.join(ROOT, "tests", "host_stub")
TIMES = ["2026-01-01T00:00:00Z", "2026-01-15T12:00:00Z", "2026-03-01T12:00:00Z", "2025-12-31T23:59:59Z"]


def _build(out, srcs, deps, extra):
    out = os.path.join(ROOT, "tests", "_build", out)
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(f) for f in srcs + deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        tmp = out + f".{os.getpid()}.tmp"
        subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-Wl,-Bsymbolic", "-o", tmp] + srcs + extra, check=True)
        os.replace(tmp, out)
    return C.CDLL(out)


@pytest.fixture(scope="module")
def host_on_oracle_reconcile(oracle):
    """kt_host.cc linked against the oracle-backed engine test double plus its kt_reconcile_throttles
    (tests/host_stub/engine_oracle_reconcile.cc); host.Plugin's signature.  CPU only; says nothing about the kernels."""
    from kube_throttler_b200 import host

    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(STUB, "engine_oracle_reconcile.cc")]
    deps = [os.path.join(STUB, "engine_oracle.cc"), os.path.join(ROOT, "oracle", "libkt_oracle.so")] + \
        [os.path.join(ROOT, "kube_throttler_b200", "csrc", f) for f in ("kt_json.h", "kt_quantity.h")] + \
        [os.path.join(ROOT, "include", f) for f in ("kt_b200.h", "kt_host.h")]
    lib = _build("libkt_hostoracle_reconcile.so", srcs, deps,
                 ["-L", os.path.join(ROOT, "oracle"), "-lkt_oracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    return functools.partial(host.Plugin, library=lib)


class KeyWorld:
    """The object oracle (oracle/ko_capi.cc compiled with tests/host_stub/oracle_reconcile_key.cc) with reconcile by key."""

    def __init__(self, L):
        self.L = L
        self.h = L.ko_world_new(THROTTLER.encode(), SCHED.encode())

    def _j(self, raw):
        out = json.loads(raw.decode())
        if isinstance(out, dict) and set(out) == {"error"}:
            raise RuntimeError(out["error"])
        return out

    def apply(self, *ms):
        for m in ms:
            self._j(self.L.ko_world_apply(self.h, json.dumps(m).encode()))

    def delete(self, kind, name, ns=""):
        if kind == "Pod":
            return self._j(self.L.ko_world_delete_pod(self.h, ns.encode(), name.encode()))
        if kind == "Namespace":
            return self._j(self.L.ko_world_delete_namespace(self.h, name.encode()))
        return self._j(self.L.ko_world_delete_throttle(self.h, 0 if kind == "Throttle" else 1, ns.encode(), name.encode()))

    def status(self, name, ns=""):
        return self._j(self.L.ko_world_get_status(self.h, ns.encode(), name.encode()))

    def prefilter(self, p):
        return self._j(self.L.ko_world_prefilter(self.h, json.dumps(p).encode()))

    def reserve(self, p):
        return self._j(self.L.ko_world_reserve(self.h, json.dumps(p).encode()))

    def reserved(self, kind, nn):
        return self._j(self.L.ko_world_reserved(self.h, 0 if kind == "Throttle" else 1, nn.encode()))

    def reconcile_key(self, kind, ns, name, now):
        return self._j(self.L.ko_world_reconcile_key(self.h, 0 if kind == "Throttle" else 1, ns.encode(), name.encode(), now.encode()))

    def close(self):
        if self.h:
            self.L.ko_world_free(self.h)
            self.h = None


@pytest.fixture(scope="module")
def key_oracle(oracle):
    src = os.path.join(STUB, "oracle_reconcile_key.cc")
    deps = [os.path.join(ROOT, "oracle", f) for f in ("ko_capi.cc", "ko_model.h", "ko_quantity.h", "ko_json.h", "ko_columnar.h")]
    L = _build("libko_reconcile_key.so", [src], deps, ["-pthread"])
    cp, vp = C.c_char_p, C.c_void_p
    L.ko_world_new.restype = vp
    L.ko_world_new.argtypes = [cp, cp]
    L.ko_world_free.argtypes = [vp]
    for name, args in (("ko_world_apply", [vp, cp]), ("ko_world_delete_pod", [vp, cp, cp]), ("ko_world_delete_namespace", [vp, cp]),
                       ("ko_world_delete_throttle", [vp, C.c_int, cp, cp]), ("ko_world_get_status", [vp, cp, cp]), ("ko_world_prefilter", [vp, cp]),
                       ("ko_world_reserve", [vp, cp]), ("ko_world_reserved", [vp, C.c_int, cp]), ("ko_world_reconcile_key", [vp, C.c_int, cp, cp, cp])):
        getattr(L, name).argtypes = args
        getattr(L, name).restype = cp
    return lambda: KeyWorld(L)


@pytest.fixture(params=["host-on-oracle", pytest.param("b200", marks=pytest.mark.gpu)])
def new_plugin(request):
    if request.param == "host-on-oracle":
        return request.getfixturevalue("host_on_oracle_reconcile")
    from kube_throttler_b200 import host  # fails loudly without the CUDA library / a GPU

    return host.Plugin


def nn_of(t):
    return t["metadata"].get("namespace", "") + "/" + t["metadata"]["name"]


def _parse_time(s):
    try:
        return datetime.datetime.fromisoformat(s.replace("Z", "+00:00"))
    except ValueError:
        return None


def next_override_ns(t, now):
    """NextOverrideHappensIn (throttle_types.go:37-63) in ns, or None."""
    n, best = _parse_time(now), None
    for ov in t["spec"].get("temporaryThresholdOverrides", []):
        for field in ("begin", "end"):
            if not ov.get(field):
                continue
            at = _parse_time(ov[field])
            if at is None:
                break  # an unparsable Begin skips the override; an unparsable End only itself
            d = int((at - n).total_seconds()) * 10**9
            if d > 0 and (best is None or d < best):
                best = d
    return best


def gauges_of(t, st):
    """The series reconcile records for throttle manifest t with status st (throttle_metrics.go / clusterthrottle_metrics.go)."""
    cluster = t["kind"] == "ClusterThrottle"
    prefix = "clusterthrottle_" if cluster else "throttle_"
    md = t["metadata"]
    base = f'name="{md["name"]}"' + ("" if cluster else f',namespace="{md["namespace"]}"')

    def key(fam, res):
        return f'{prefix}{fam}{{{base},resource="{res}",uid="{md.get("uid", "")}"}}'

    out = {}

    def amount(fam, a):
        out[key(fam + "_resourceCounts", "pod")] = a["resourceCounts"]["pod"] if "resourceCounts" in a else 0
        for r, v in a.get("resourceRequests", {}).items():
            out[key(fam + "_resourceRequests", r)] = math.ceil(q(v) * (1000 if r == "cpu" else 1))

    amount("spec_threshold", t["spec"]["threshold"])
    out[key("status_throttled_resourceCounts", "pod")] = int(st["throttled"]["resourceCounts"]["pod"])
    for r, b in st["throttled"].get("resourceRequests", {}).items():
        out[key("status_throttled_resourceRequests", r)] = int(b)
    amount("status_used", st["used"])
    amount("status_calculated_threshold", st["calculatedThreshold"]["threshold"])
    return out


def parse_metrics(text):
    out = {}
    for line in text.splitlines():
        if line and not line.startswith("#"):
            k, v = line.rsplit(" ", 1)
            out[k] = float(v)
    return out


class Twin:
    """The oracle, the plugin and the models of what the oracle does not keep (gauges), driven by the same events."""

    def __init__(self, ref, dut):
        self.ref, self.dut, self.gauges, self.live = ref, dut, {}, {}

    def apply(self, *ms):
        for m in ms:
            self.ref.apply(m)
            self.dut.apply(m)
            if m["kind"] in ("Throttle", "ClusterThrottle"):
                self.live[(m["kind"], nn_of(m))] = m

    def delete(self, kind, name, ns=""):
        self.ref.delete(kind, name, ns)
        self.dut.delete(kind, name, ns)
        self.live.pop((kind, ns + "/" + name), None)

    def expect_key(self, key, now):
        """The oracle's reconcile of one key: (kind of outcome, detail); updates the gauge model."""
        ns, _, name = key.partition("/")
        kinds = ["ClusterThrottle"] if ns == "" else ["Throttle"]
        t = self.live.get((kinds[0], key))
        r = self.ref.reconcile_key(kinds[0], ns, name, now)
        if not r["found"]:
            return "notFound", None
        if not r["responsible"]:
            return "skipped", None
        if r["err"]:
            return "error", r["err"]
        self.gauges.update(gauges_of(t, self.ref.status(name, ns)))
        return "ok", (r["statusChanged"], next_override_ns(t, now))

    def reconcile(self, keys, now):
        got = self.dut.reconcile(keys, now)
        want = {"reconciled": 0, "changed": [], "requeueAfterNanos": {}, "errors": {}, "notFound": []}
        seen = set()
        for key in keys:
            if key in seen:
                continue
            seen.add(key)
            ns, slash, name = key.partition("/")
            if not slash or not name or "/" in name:  # malformed: the text is the plugin's
                want["errors"][key] = None
                continue
            what, detail = self.expect_key(key, now)
            if what == "notFound":
                want["notFound"].append(key)
            elif what == "error":
                want["errors"][key] = detail
            elif what == "ok":
                want["reconciled"] += 1
                if detail[0]:
                    want["changed"].append(key)
                if detail[1] is not None:
                    want["requeueAfterNanos"][key] = detail[1]
        assert set(got["errors"]) == set(want["errors"]), (keys, got, want)
        for k, text in want["errors"].items():
            if text is not None:
                assert got["errors"][k] == text, (k, got)
        for f in ("reconciled", "changed", "requeueAfterNanos", "notFound"):
            assert got[f] == want[f], (f, keys, got, want)
        return got

    def reconcile_all(self, now):
        keys = [nn_of(t) for t in self.live.values() if t["spec"]["throttlerName"] == THROTTLER]
        got = self.dut.reconcile_all(now)
        changed, requeue = [], {}
        for key in keys:
            what, detail = self.expect_key(key, now)
            if what == "ok":
                if detail[0]:
                    changed.append(key)
                if detail[1] is not None:
                    requeue[key] = detail[1]
        assert sorted(got["changed"]) == sorted(changed) and got["requeueAfterNanos"] == requeue, (got, changed, requeue)

    def compare(self, queue, where):
        for (kind, key), t in self.live.items():
            ns, _, name = key.partition("/")
            a, b = self.ref.status(name, ns), self.dut.status(name, ns)
            assert norm_status(a) == norm_status(b), (where, key, a, b)
        for (kind, key) in self.live:
            a, b = self.ref.reserved(kind, key), self.dut.reserved(kind, key)
            assert sorted(a["pods"]) == sorted(b["pods"]) and norm_amount(a["amount"]) == norm_amount(b["amount"]), (where, key, a, b)
        for p in queue:
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if self.dut.queue_row(*k) < 0:
                continue
            a, b = self.ref.prefilter(p), self.dut.prefilter_key(*k)
            assert (a["code"], a["reasons"]) == (b["code"], b["reasons"]), (where, k, a, b)
        assert parse_metrics(self.dut.metrics()) == {k: float(v) for k, v in self.gauges.items()}, where


BROKEN = [{"matchExpressions": [{"key": "team", "operator": "In", "values": []}]},
          {"matchExpressions": [{"key": "env", "operator": "Exists", "values": ["a"]}]}]


def random_keys(rng, throttles):
    keys = [nn_of(t) for t in rng.sample(throttles, rng.randint(0, min(6, len(throttles))))]
    if keys and rng.random() < 0.4:
        keys.append(rng.choice(keys))  # a duplicate
    if rng.random() < 0.3:
        keys.append(rng.choice(["ns0/nobody", "/nobody", "ns9/t1"]))  # unknown
    if rng.random() < 0.15:
        keys.append(rng.choice(["no-slash", "ns0/a/b", "ns0/"]))  # malformed
    rng.shuffle(keys)
    return keys


def run_stream(key_oracle, new_plugin, seed, steps=50, n_thr=14, n_ns=4):
    rng = random.Random(seed)
    ref, dut = key_oracle(), new_plugin(THROTTLER, SCHED)
    w = Twin(ref, dut)
    nss = [f"ns{i}" for i in range(n_ns)]
    for n in nss:
        w.apply(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
    throttles = [rand_throttle(rng, i, nss) for i in range(n_thr)]
    w.apply(*throttles)
    pods = [rand_pod(rng, rng.choice(nss), f"p{i}", True) for i in range(60)]
    w.apply(*pods)
    queue = [rand_pod(rng, rng.choice(nss), f"q{i}", False) for i in range(30)]
    w.apply(*queue)
    reserved, counts = [], {"keys": 0, "all": 0}
    for step in range(steps):
        op = rng.random()
        where = (seed, step)
        if op < 0.3:
            counts["keys"] += 1
            w.reconcile(random_keys(rng, throttles), rng.choice(TIMES))
        elif op < 0.36:
            counts["all"] += 1
            w.reconcile_all(rng.choice(TIMES))
        elif op < 0.5:
            p = rng.choice(queue)
            k = (p["metadata"]["namespace"], p["metadata"]["name"])
            if dut.queue_row(*k) >= 0 and ref.prefilter(p)["code"] == "Success":
                assert ref.reserve(p)["code"] == dut.reserve_key(*k)["code"] == "Success", where
                reserved.append(p)
        elif op < 0.56 and reserved:  # bind: the pod runs (or finishes at once) on a node
            p = reserved.pop(rng.randrange(len(reserved)))
            queue.remove(p)
            p = dict(p, spec=dict(p["spec"], nodeName="node-2"), status={"phase": rng.choice(["Running", "Running", "Succeeded"])})
            pods.append(p)
            w.apply(p)
        elif op < 0.68:
            p = rng.choice(pods)  # relabel, maybe finish
            p["metadata"]["labels"] = rand_labels(rng)
            if rng.random() < 0.3:
                p["status"] = {"phase": rng.choice(["Running", "Succeeded", "Failed"])}
            w.apply(p)
        elif op < 0.72:
            i = rng.randrange(len(pods))  # a pod deleted and re-created in another namespace
            old = pods[i]
            w.delete("Pod", old["metadata"]["name"], old["metadata"]["namespace"])
            pods[i] = rand_pod(rng, rng.choice(nss), old["metadata"]["name"], True)
            w.apply(pods[i])
        elif op < 0.84:
            i = rng.randrange(len(throttles))  # threshold / override / selector edit, sometimes a broken podSelector
            t = rand_throttle(rng, i, nss)
            t["kind"], t["metadata"] = throttles[i]["kind"], throttles[i]["metadata"]
            if t["kind"] == "Throttle":
                for term in t["spec"]["selector"]["selectorTerms"]:
                    term.pop("namespaceSelector", None)
            if t["spec"]["selector"]["selectorTerms"] and rng.random() < 0.2:
                rng.choice(t["spec"]["selector"]["selectorTerms"])["podSelector"] = rng.choice(BROKEN)
            throttles[i] = t
            w.apply(t)
        elif op < 0.9:
            n = rng.choice(nss)
            w.apply(namespace(n, {"team": rng.choice(VALS), "env": rng.choice(VALS)}))
        elif op < 0.93:
            i = rng.randrange(len(throttles))
            md = throttles[i]["metadata"]
            if (throttles[i]["kind"], nn_of(throttles[i])) in w.live:
                w.delete(throttles[i]["kind"], md["name"], md.get("namespace", ""))
        else:
            p = rand_pod(rng, rng.choice(nss), f"n{step}", True)
            p["spec"]["containers"][0]["resources"]["requests"]["cpu"] = rng.choice(CPUS)
            pods.append(p)
            w.apply(p)
        w.compare(queue, where)
    dut.close()
    ref.close()
    return counts


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_event_stream(key_oracle, new_plugin, seed):
    counts = run_stream(key_oracle, new_plugin, seed)
    assert counts["keys"] >= 8


def test_unlisted_throttles_are_untouched(key_oracle, new_plugin):
    """Two throttles of one namespace: reconciling one writes its status, un-reserves its observed pods and records its gauges;
    the other keeps its status, its reservation and has no gauges until it is reconciled itself."""
    ref, dut = key_oracle(), new_plugin(THROTTLER, SCHED)
    w = Twin(ref, dut)
    lbl = {"app": "x"}
    w.apply(namespace("default"), throttle("default", "a", lbl, pod_cnt=5, cpu="1"), throttle("default", "b", lbl, pod_cnt=5, cpu="2"))
    q0 = pod("default", "q0", "100m", lbl)
    w.apply(q0)
    assert ref.reserve(q0)["code"] == dut.reserve_key("default", "q0")["code"] == "Success"
    bound = pod("default", "q0", "100m", lbl, node="n", phase="Running")
    w.apply(bound, pod("default", "p1", "300m", lbl, node="n", phase="Running"))
    got = w.reconcile(["default/a", "default/a", "/nobody"], NOW)
    assert got["reconciled"] == 1 and got["changed"] == ["default/a"] and got["notFound"] == ["/nobody"]
    assert dut.reserved("Throttle", "default/a")["pods"] == [] and dut.reserved("Throttle", "default/b")["pods"] == ["default/q0"]
    assert dut.status("b", "default")["calculatedThreshold"]["calculatedAtSet"] is False
    assert not any('name="b"' in k for k in parse_metrics(dut.metrics()))
    w.compare([], "after a")
    w.reconcile(["default/b"], NOW)
    w.compare([], "after b")
    dut.close()
    ref.close()


def test_selector_error_is_per_key(key_oracle, new_plugin):
    """A ClusterThrottle whose broken term a counted pod reaches (through its namespaceSelector): its key is an error, its status
    and reservations stay, and the other key of the same call is reconciled."""
    ref, dut = key_oracle(), new_plugin(THROTTLER, SCHED)
    w = Twin(ref, dut)
    team_a = {"matchLabels": {"team": "a"}}
    ct = {"kind": "ClusterThrottle", "metadata": {"name": "ct"},
          "spec": {"throttlerName": THROTTLER, "threshold": {"resourceCounts": {"pod": 5}},
                   "selector": {"selectorTerms": [{"namespaceSelector": team_a, "podSelector": {"matchLabels": {"x": "1"}}},
                                                  {"namespaceSelector": team_a, "podSelector": BROKEN[0]}]}}}
    w.apply(namespace("na", {"team": "a"}), namespace("nb", {"team": "b"}), ct, throttle("nb", "t", {"y": "1"}, pod_cnt=1),
            throttle("nb", "foreign", {"y": "1"}, pod_cnt=1, throttler="other-throttler"))
    w.apply(pod("na", "p0", "100m", {"x": "1"}, node="n", phase="Running"), pod("nb", "p1", "100m", {"y": "1"}, node="n", phase="Running"))
    got = w.reconcile(["/ct", "nb/t", "nb/foreign"], NOW)  # nobody reaches the broken term yet
    assert got["reconciled"] == 2 and not got["errors"]
    w.apply(pod("na", "p2", "100m", {"y": "1"}, node="n", phase="Failed"))  # a counted pod of a team-a namespace reaches it
    got = w.reconcile(["/ct", "nb/t"], "2026-01-02T00:00:00Z")
    assert list(got["errors"]) == ["/ct"] and got["reconciled"] == 1
    w.compare([], "after the error")
    dut.close()
    ref.close()


def test_resource_count_active_by_key(new_plugin):
    """throttle_test.go: a pod-count threshold of 2 filled by two running pods; reconcile(["default/test-throttle"]) in place of
    reconcile_all, then the third pod waits, throttled [active]."""
    dut = new_plugin(THROTTLER, SCHED)
    lbl = {"throttle": "test-throttle"}
    dut.apply(namespace("default"), throttle("default", "test-throttle", lbl, pod_cnt=2, cpu="1"),
              pod("default", "pod-1", "100m", lbl, node="n", phase="Running"), pod("default", "pod-2", "100m", lbl, node="n", phase="Running"))
    got = dut.reconcile(["default/test-throttle"], NOW)
    assert got == {"reconciled": 1, "changed": ["default/test-throttle"], "requeueAfterNanos": {}, "errors": {}, "notFound": []}
    st = dut.status("test-throttle", "default")
    assert st["used"]["resourceCounts"] == {"pod": 2} and q(st["used"]["resourceRequests"]["cpu"]) == q("200m")
    assert st["throttled"]["resourceCounts"]["pod"] is True and st["throttled"]["resourceRequests"]["cpu"] is False
    dut.apply(pod("default", "pod-3", "100m", lbl))
    assert dut.prefilter_key("default", "pod-3")["reasons"] == ["throttle[active]=default/test-throttle"]
    assert dut.reconcile(["default/test-throttle"], NOW)["changed"] == []  # nothing moved: no status write
    dut.close()
