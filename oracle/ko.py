"""ctypes wrapper of the ORACLE (oracle/libkt_oracle.so).

TEST INFRASTRUCTURE ONLY.  Importers allowed: tests/, __graft_entry__.smoke(), bench.py's
cpu_baseline / --impl reference leg.  The product package (kube_throttler_b200/) never imports this.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess
from typing import Optional

import numpy as np

from kube_throttler_b200 import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libkt_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    """Compile the oracle (gcc only; no GPU, no reference sources needed)."""
    srcs = ["ko_capi.cc", "ko_model.h", "ko_quantity.h", "ko_json.h", "ko_columnar.h"]
    newest = max(os.path.getmtime(os.path.join(_HERE, s)) for s in srcs)
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < newest:
        subprocess.run(["make", "-C", _HERE, "-s", "-B"], check=True)
    return _LIB_PATH


class ColumnarArgs(C.Structure):
    _fields_ = [
        ("lim", abi.Limits),
        ("n_running", C.c_int64), ("run_labels", C.c_void_p), ("run_req", C.c_void_p), ("run_present", C.c_void_p),
        ("run_flags", C.c_void_p), ("run_ns", C.c_void_p),
        ("n_pending", C.c_int64), ("pend_labels", C.c_void_p), ("pend_req", C.c_void_p), ("pend_present", C.c_void_p),
        ("pend_flags", C.c_void_p), ("pend_ns", C.c_void_p),
        ("n_ns", C.c_int32), ("ns_labels", C.c_void_p),
        ("m", C.c_int32),
        ("thr", C.POINTER(abi.ThrottleCols)), ("sel", C.POINTER(abi.SelectorTable)), ("status", C.POINTER(abi.StatusCols)),
        ("reserved", C.c_void_p), ("reserved_present", C.c_void_p), ("reserved_cnt", C.c_void_p),
        ("now", C.c_int64), ("flags", C.c_uint32), ("words_per_row", C.c_int32),
        ("rec", abi.ReconcileOut),
        ("run_bitmap", C.c_void_p), ("pend_bitmap", C.c_void_p), ("codes", C.c_void_p), ("admit", C.c_void_p),
    ]


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        for name in ("ko_eval", "ko_world_apply", "ko_world_reconcile_all", "ko_world_prefilter", "ko_world_reserve",
                     "ko_world_unreserve"):
            getattr(L, name).restype = C.c_char_p
        L.ko_eval.argtypes = [C.c_char_p]
        L.ko_world_new.restype = C.c_void_p
        L.ko_world_new.argtypes = [C.c_char_p, C.c_char_p]
        L.ko_world_free.argtypes = [C.c_void_p]
        L.ko_world_apply.argtypes = [C.c_void_p, C.c_char_p]
        L.ko_world_delete_pod.restype = C.c_char_p
        L.ko_world_delete_pod.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
        L.ko_world_delete_namespace.restype = C.c_char_p
        L.ko_world_delete_namespace.argtypes = [C.c_void_p, C.c_char_p]
        L.ko_world_delete_throttle.restype = C.c_char_p
        L.ko_world_delete_throttle.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p]
        L.ko_world_reconcile_all.argtypes = [C.c_void_p, C.c_char_p]
        L.ko_world_get_status.restype = C.c_char_p
        L.ko_world_get_status.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
        L.ko_world_prefilter.argtypes = [C.c_void_p, C.c_char_p]
        L.ko_world_reserve.argtypes = [C.c_void_p, C.c_char_p]
        L.ko_world_unreserve.argtypes = [C.c_void_p, C.c_char_p]
        L.ko_world_reserved.restype = C.c_char_p
        L.ko_world_reserved.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
        L.ko_columnar_evaluate.restype = C.c_int
        L.ko_columnar_evaluate.argtypes = [C.POINTER(ColumnarArgs)]
        L.ko_columnar_admit_queue.restype = C.c_int
        L.ko_columnar_admit_queue.argtypes = [C.POINTER(ColumnarArgs), C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.POINTER(C.c_int64)]
        L.ko_world_from_columns.restype = C.c_void_p
        L.ko_world_from_columns.argtypes = [C.POINTER(ColumnarArgs)]
        L.ko_world_run_columns.restype = C.c_double
        L.ko_world_run_columns.argtypes = [C.c_void_p, C.POINTER(ColumnarArgs), C.c_int, C.c_int64, C.c_int32,
                                           C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.ko_hardware_threads.restype = C.c_int
        _lib = L
    return _lib


def call(fn: str, **kw):
    """Unit-level oracle call: returns the decoded JSON result (raises on {"error":...})."""
    out = json.loads(lib().ko_eval(json.dumps(dict(fn=fn, **kw)).encode()).decode())
    if isinstance(out, dict) and set(out.keys()) == {"error"}:
        raise RuntimeError(out["error"])
    return out


class World:
    """Object-level oracle world (informer caches + both controllers + plugin)."""

    def __init__(self, throttler_name="kube-throttler", target_scheduler_name="my-scheduler", handle=None):
        self._h = handle if handle is not None else lib().ko_world_new(throttler_name.encode(), target_scheduler_name.encode())

    def close(self):
        if self._h:
            lib().ko_world_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _json(self, raw):
        out = json.loads(raw.decode())
        if isinstance(out, dict) and set(out.keys()) == {"error"}:
            raise RuntimeError(out["error"])
        return out

    def apply(self, *manifests):
        for m in manifests:
            self._json(lib().ko_world_apply(self._h, json.dumps(m).encode()))

    def delete(self, kind, name, namespace=""):
        """Informer Delete event of a Pod, Throttle or ClusterThrottle (host.Plugin.delete has the same signature)."""
        if kind == "Pod":
            return self._json(lib().ko_world_delete_pod(self._h, namespace.encode(), name.encode()))
        if kind in ("Throttle", "ClusterThrottle"):
            return self._json(lib().ko_world_delete_throttle(self._h, 0 if kind == "Throttle" else 1, namespace.encode(), name.encode()))
        if kind == "Namespace":
            return self._json(lib().ko_world_delete_namespace(self._h, name.encode()))
        raise NotImplementedError("the oracle does not model deletes of " + kind)

    def reconcile_all(self, now="2026-01-01T00:00:00Z"):
        return self._json(lib().ko_world_reconcile_all(self._h, now.encode()))

    def status(self, name, namespace=""):
        return self._json(lib().ko_world_get_status(self._h, namespace.encode(), name.encode()))

    def prefilter(self, pod):
        return self._json(lib().ko_world_prefilter(self._h, json.dumps(pod).encode()))

    def reserve(self, pod):
        return self._json(lib().ko_world_reserve(self._h, json.dumps(pod).encode()))

    def unreserve(self, pod):
        return self._json(lib().ko_world_unreserve(self._h, json.dumps(pod).encode()))

    def reserved(self, kind: str, thr_nn: str):
        return self._json(lib().ko_world_reserved(self._h, 0 if kind == "Throttle" else 1, thr_nn.encode()))


def _args(snap: abi.Snapshot, flags: int, out: Optional[abi.PassResult], keep: list) -> ColumnarArgs:
    thr, sel, st = snap.throttle_cols(), snap.selector_table(), snap.status_cols()
    keep += [thr, sel, st, snap, out]
    a = ColumnarArgs()
    a.lim = snap.limits()
    r, p = snap.running, snap.pending
    a.n_running, a.run_labels, a.run_req, a.run_present, a.run_flags, a.run_ns = (
        r.n, abi.ptr(r.labels), abi.ptr(r.req), abi.ptr(r.present), abi.ptr(r.flags), abi.ptr(r.ns_id))
    a.n_pending, a.pend_labels, a.pend_req, a.pend_present, a.pend_flags, a.pend_ns = (
        p.n, abi.ptr(p.labels), abi.ptr(p.req), abi.ptr(p.present), abi.ptr(p.flags), abi.ptr(p.ns_id))
    a.n_ns, a.ns_labels = snap.n_ns, abi.ptr(snap.ns_labels)
    a.m = snap.m
    a.thr = C.pointer(thr)
    a.sel = C.pointer(sel)
    a.status = C.pointer(st) if st is not None else None
    a.reserved, a.reserved_present, a.reserved_cnt = abi.ptr(snap.reserved), abi.ptr(snap.reserved_present), abi.ptr(snap.reserved_cnt)
    a.now, a.flags = snap.now, flags
    if out is not None:
        a.words_per_row = out.words_per_row
        a.rec = out.reconcile_out()
        a.run_bitmap, a.pend_bitmap, a.codes, a.admit = abi.ptr(out.run_bitmap), abi.ptr(out.pend_bitmap), abi.ptr(out.codes), abi.ptr(out.admit)
    else:
        a.words_per_row = abi.default_words_per_row(snap.m)
    return a


def columnar_evaluate(snap: abi.Snapshot, flags: int = abi.EVAL_FRESH_STATUS, words_per_row: Optional[int] = None) -> abi.PassResult:
    """The columnar oracle: plain loops over the engine's own columns."""
    snap.normalize()
    out = abi.PassResult.alloc(snap, words_per_row or abi.default_words_per_row(snap.m))
    keep: list = []
    a = _args(snap, flags, out, keep)
    rc = lib().ko_columnar_evaluate(C.byref(a))
    if rc != 0:
        raise RuntimeError("ko_columnar_evaluate failed")
    return out


def columnar_admit_queue(snap: abi.Snapshot, first: int, count: int, flags: int = 0, words_per_row: Optional[int] = None):
    """Queue-ordered greedy admission of the pending rows [first, first + count), one pod per cycle, against snap.status and
    snap.reserved (flags: KT_EVAL_ON_EQUAL or 0).  Returns (PassResult with pend_bitmap / codes / admit filled, admitted count,
    (reserved, reserved_present, reserved_cnt) after the queue)."""
    snap.normalize()
    if snap.status is None:
        raise ValueError("columnar_admit_queue checks against the observed status: snap.status is required")
    out = abi.PassResult.alloc(snap, words_per_row or abi.default_words_per_row(snap.m))
    keep: list = []
    a = _args(snap, flags, out, keep)
    res = np.zeros((snap.R, snap.m), np.int64)
    res_present = np.zeros(snap.m, np.uint32)
    res_cnt = np.zeros(snap.m, np.int64)
    admitted = C.c_int64(0)
    rc = lib().ko_columnar_admit_queue(C.byref(a), first, count, abi.ptr(res), abi.ptr(res_present), abi.ptr(res_cnt), C.byref(admitted))
    if rc != 0:
        raise RuntimeError("ko_columnar_admit_queue failed")
    return out, admitted.value, (res, res_present, res_cnt)


def object_evaluate(snap: abi.Snapshot, flags: int = abi.EVAL_FRESH_STATUS, threads: int = 1, max_pending: int = 0,
                    max_reconcile: int = 0, words_per_row: Optional[int] = None):
    """Reference-shaped path: build string/map objects from the columns, reconcile + PreFilter every pending pod.

    Returns (PassResult, timings dict).  run_bitmap is not produced by this path (left zero)."""
    snap.normalize()
    out = abi.PassResult.alloc(snap, words_per_row or abi.default_words_per_row(snap.m))
    keep: list = []
    a = _args(snap, flags, out, keep)
    h = lib().ko_world_from_columns(C.byref(a))
    rs, cs = C.c_double(0), C.c_double(0)
    try:
        total = lib().ko_world_run_columns(h, C.byref(a), threads, max_pending, max_reconcile, C.byref(rs), C.byref(cs))
    finally:
        lib().ko_world_free(h)
    return out, dict(total_s=abs(total), reconcile_s=rs.value, check_s=cs.value, had_error=total < 0)


def hardware_threads() -> int:
    return lib().ko_hardware_threads()
