"""ctypes binding of include/kt_host.h: the kube-scheduler plugin surface above the device engine.

`Plugin` reads like the reference's plugin: `Plugin(name, target_scheduler_name)` is NewPlugin
(plugin.go:63), `pre_filter` / `reserve` / `unreserve` are PreFilter / Reserve / Unreserve (plugin.go:148-257),
`apply` / `delete` are the informer events and `reconcile_all` runs every throttle's reconcile(key)
(throttle_controller.go:84) as one device pass.  Manifests are plain dicts (Kubernetes JSON).
Nothing is computed here; every call crosses the C ABI.
"""
from __future__ import annotations

import ctypes as C
import json

from . import KtError, abi, lib


def _bind(L=None):
    """Declare the kt_host.h prototypes on a loaded library: the product's (default), or any other build of kt_host.cc that
    exports them (tests link the host layer against engine test doubles to check its bookkeeping without a device)."""
    L = L if L is not None else lib()
    if getattr(L, "_kth_bound", False):
        return L
    vp, cp = C.c_void_p, C.c_char_p
    L.kth_new_plugin.argtypes = [C.POINTER(vp), cp, C.c_int]
    L.kth_new_plugin_error.restype = cp
    L.kth_free.argtypes = [vp]
    L.kth_free.restype = None
    for name, args in (("kth_apply", [vp, cp]), ("kth_delete", [vp, cp, cp, cp]), ("kth_apply_events", [vp, cp]), ("kth_reconcile_all", [vp, cp]), ("kth_reconcile", [vp, cp, cp]),
                       ("kth_get_status", [vp, cp, cp]), ("kth_get_status_manifest", [vp, cp, cp]), ("kth_affected_pods", [vp, cp, cp]), ("kth_queue_report", [vp]), ("kth_pre_filter", [vp, cp]), ("kth_pre_filter_batch", [vp, cp]),
                       ("kth_admit_queue", [vp, cp]), ("kth_pre_filter_key", [vp, cp, cp]), ("kth_pre_filter_keys", [vp, cp]), ("kth_reserve_key", [vp, cp, cp]), ("kth_unreserve_key", [vp, cp, cp]),
                       ("kth_queue_stats", [vp]), ("kth_reserve", [vp, cp]), ("kth_unreserve", [vp, cp]), ("kth_reserved", [vp, C.c_int, cp]), ("kth_metrics", [vp]), ("kth_eval", [cp])):
        fn = getattr(L, name)
        fn.argtypes = args
        fn.restype = cp
    L.kth_pre_filter_queue.argtypes = [vp, C.c_void_p, C.c_int64]
    L.kth_pre_filter_queue.restype = C.c_int64
    L.kth_queue_row.argtypes = [vp, cp, cp]
    L.kth_queue_row.restype = C.c_int64
    L.kth_pod_row.argtypes = [vp, cp, cp]
    L.kth_pod_row.restype = C.c_int64
    L.kth_last_error.restype = cp
    L._kth_bound = True
    return L


HOST_EXPORTS = ["kth_new_plugin", "kth_new_plugin_error", "kth_free", "kth_apply", "kth_delete", "kth_reconcile_all", "kth_get_status", "kth_get_status_manifest",
                "kth_pre_filter", "kth_pre_filter_key", "kth_reserve_key", "kth_unreserve_key", "kth_pre_filter_queue", "kth_queue_row", "kth_pod_row", "kth_queue_stats", "kth_last_error", "kth_pre_filter_batch", "kth_admit_queue", "kth_reserve", "kth_unreserve", "kth_reserved", "kth_metrics", "kth_eval", "kth_affected_pods", "kth_reconcile", "kth_pre_filter_keys", "kth_apply_events", "kth_queue_report"]


def _result(raw):
    out = json.loads(raw.decode())
    if isinstance(out, dict) and set(out.keys()) == {"error"}:
        raise RuntimeError(out["error"])
    return out


def eval_host(fn: str, **kw):
    """Host-only packer helpers (kth_eval): no device involved."""
    return _result(_bind().kth_eval(json.dumps(dict(kw, fn=fn)).encode()))


class Plugin:
    """kubethrottler.NewPlugin(configuration, handle) -- fails without a GPU (there is no CPU path)."""

    def __init__(self, name="kube-throttler", target_scheduler_name="my-scheduler", device=0, library=None, **extra_args):
        self._L = _bind(library)
        self._h = C.c_void_p()
        args = dict(extra_args, name=name, targetSchedulerName=target_scheduler_name)
        rc = self._L.kth_new_plugin(C.byref(self._h), json.dumps(args).encode(), device)
        if rc != abi.OK:
            self._h = None
            raise KtError(rc, self._L.kth_new_plugin_error().decode())

    def close(self):
        if self._h:
            self._L.kth_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # informer events
    def apply(self, *manifests):
        out = None
        for m in manifests:
            out = _result(self._L.kth_apply(self._h, json.dumps(m).encode()))
        return out  # {"ok": true} -- plus "warning" when a stored pod update could not move its reservations

    def delete(self, kind, name, namespace=""):
        _result(self._L.kth_delete(self._h, kind.encode(), namespace.encode(), name.encode()))

    def apply_events(self, events):
        """A batch of watch events ({"type": "ADDED" | "MODIFIED" | "DELETED", "object": manifest}) applied in order:
        {"results": [per event what apply / delete return, plus "enqueue": [keys]], "enqueue": [the union of the keys]}.
        A refused or malformed event is an {"error": ...} entry (no exception for those); the rest of the batch applies."""
        return _result(self._L.kth_apply_events(self._h, json.dumps(list(events)).encode()))

    # controllers
    def reconcile_all(self, now="2026-01-01T00:00:00Z"):
        return _result(self._L.kth_reconcile_all(self._h, now.encode()))

    def reconcile(self, keys, now="2026-01-01T00:00:00Z"):
        """reconcile(key) for the listed keys only ("namespace/name" for a Throttle, "/name" for a ClusterThrottle):
        {"reconciled", "changed", "requeueAfterNanos", "errors", "notFound"}."""
        return _result(self._L.kth_reconcile(self._h, json.dumps(list(keys)).encode(), now.encode()))

    def status(self, name, namespace=""):
        return _result(self._L.kth_get_status(self._h, namespace.encode(), name.encode()))

    def status_manifest(self, name, namespace="") -> str:
        """The status subresource as the reference's UpdateStatus would send it (raw JSON text: key order and spellings matter)."""
        raw = self._L.kth_get_status_manifest(self._h, namespace.encode(), name.encode()).decode()
        _result(raw.encode())  # raises on {"error": ...}
        return raw

    def affected_pods(self, name, namespace=""):
        """affectedPods of a Throttle (namespace given) or ClusterThrottle: {"pods": [...], "terminatedPods": [...],
        "queued": [{"pod": "ns/name", "status": ...}, ...]}, each sorted by namespace, then name."""
        return _result(self._L.kth_affected_pods(self._h, namespace.encode(), name.encode()))

    def queue_report(self):
        """The scheduling queue per throttle: {"queued", "success", "unschedulable", "error", "throttles": [{"key", "kind",
        "active", "insufficient", "podRequestsExceedsThreshold", "onlyBlocker", "heldBack"}, ...]} for every throttle of this
        plugin, in creation order -- one device call (plus at most one pass) instead of affected_pods for every throttle."""
        return _result(self._L.kth_queue_report(self._h))

    # plugin
    def prefilter(self, pod):
        return _result(self._L.kth_pre_filter(self._h, json.dumps(pod).encode()))

    # the same for pods the informer already delivered (kth_apply), addressed by key: the resident scheduling queue
    def prefilter_key(self, namespace, name):
        return _result(self._L.kth_pre_filter_key(self._h, namespace.encode(), name.encode()))

    def prefilter_keys(self, keys):
        """PreFilter by key for the listed "namespace/name" keys, checked on the device row by row: one entry per key, in order --
        what prefilter_key returns, or {"error": ...} for an unknown pod or a malformed key (no exception for those)."""
        return _result(self._L.kth_pre_filter_keys(self._h, json.dumps(list(keys)).encode()))

    def reserve_key(self, namespace, name):
        return _result(self._L.kth_reserve_key(self._h, namespace.encode(), name.encode()))

    def unreserve_key(self, namespace, name):
        return _result(self._L.kth_unreserve_key(self._h, namespace.encode(), name.encode()))

    def prefilter_queue(self):
        """One verdict byte per queue row (0 free, 1 Success, 2 UnschedulableAndUnresolvable, 3 Error) in at most one device pass."""
        import numpy as np

        n = self._L.kth_pre_filter_queue(self._h, None, 0)
        if n < 0:
            _result(self._L.kth_last_error())
        out = np.zeros(max(n, 1), np.uint8)
        n = self._L.kth_pre_filter_queue(self._h, out.ctypes.data, out.shape[0])
        if n < 0:
            _result(self._L.kth_last_error())
        return out[:n]

    def queue_row(self, namespace, name) -> int:
        return int(self._L.kth_queue_row(self._h, namespace.encode(), name.encode()))

    def pod_row(self, namespace, name) -> int:
        return int(self._L.kth_pod_row(self._h, namespace.encode(), name.encode()))

    def queue_stats(self):
        return _result(self._L.kth_queue_stats(self._h))

    def prefilter_batch(self, pods):
        return _result(self._L.kth_pre_filter_batch(self._h, json.dumps(list(pods)).encode()))

    def admit_queue(self, pods):
        """PreFilter -> Reserve for a sorted queue with the one-pod-per-cycle semantics, in few device passes."""
        return _result(self._L.kth_admit_queue(self._h, json.dumps(list(pods)).encode()))

    def reserve(self, pod):
        return _result(self._L.kth_reserve(self._h, json.dumps(pod).encode()))

    def unreserve(self, pod):
        return _result(self._L.kth_unreserve(self._h, json.dumps(pod).encode()))

    def metrics(self) -> str:
        """The controllers' gauges as Prometheus text exposition (throttle_metrics.go, clusterthrottle_metrics.go)."""
        text = self._L.kth_metrics(self._h).decode()
        if text.startswith('{"error"'):
            raise RuntimeError(json.loads(text)["error"])
        return text

    def reserved(self, kind: str, thr_nn: str):
        return _result(self._L.kth_reserved(self._h, 0 if kind == "Throttle" else 1, thr_nn.encode()))
