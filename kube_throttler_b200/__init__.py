"""kube_throttler_b200 -- H100-native throttle-admission hot path of everpeace/kube-throttler.

The product is the C-ABI shared library `libkt_b200.so` (include/kt_b200.h; CUDA kernels in csrc/).
This Python module is a thin ctypes binding used by the tests and bench.py -- the same calls a Go
plugin would make through cgo (INTEGRATION.md).  There is no CPU fallback anywhere in this package:
if the library or a GPU is missing, `Engine(...)` raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Optional

import numpy as np

from . import abi
from .abi import PassResult, PodCols, Snapshot  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("KT_B200_LIB") or os.path.join(_HERE, "libkt_b200.so")  # override: kernel-variant experiments only
_lib = None


class KtError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"kt error {code}: {msg}")
        self.code = code


def build(force: bool = False) -> str:
    """Compile csrc/ for sm_90a in-tree (nvcc cross-compiles without a GPU)."""
    srcs = [os.path.join(_HERE, "csrc", f) for f in ("kt_engine.cu", "kt_tables.cc", "kt_host.cc", "kt_kernels.cuh", "kt_admit.cuh", "kt_keyed.cuh", "kt_nsrows.cuh", "kt_order.cuh", "kt_tables.h", "kt_json.h", "kt_quantity.h")]
    srcs.append(os.path.join(_HERE, "..", "include", "kt_b200.h"))
    srcs.append(os.path.join(_HERE, "..", "include", "kt_host.h"))
    newest = max(os.path.getmtime(s) for s in srcs)
    if force or not os.path.exists(LIB_PATH) or os.path.getmtime(LIB_PATH) < newest:
        subprocess.run(["make", "-C", os.path.join(_HERE, "csrc"), "-s", "-B", "NVCCFLAGS_EXTRA="], check=True,
                       stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
    return LIB_PATH


EXPORTS = [
    "kt_create", "kt_destroy", "kt_last_error", "kt_version", "kt_set_stream", "kt_sync", "kt_enable_timing",
    "kt_enable_trace", "kt_get_trace", "kt_host_alloc", "kt_host_alloc_upload", "kt_host_free", "kt_upload_pods", "kt_upload_pods_compact", "kt_upload_pods_packed", "kt_set_async_uploads", "kt_update_pod_rows", "kt_upload_namespaces", "kt_update_namespace_rows",
    "kt_upload_throttles", "kt_upload_status", "kt_set_reserved", "kt_update_status_rows", "kt_update_reserved_rows", "kt_update_threshold_rows", "kt_update_selector_rows", "kt_append_throttle_rows", "kt_move_throttle_columns", "kt_evaluate", "kt_get_reconcile",
    "kt_match_words", "kt_get_match_bitmap", "kt_get_match_rows", "kt_get_match_columns", "kt_get_check_summary", "kt_reconcile_throttles", "kt_get_check", "kt_set_sparse_check", "kt_get_check_sparse", "kt_get_check_rows", "kt_check_pending_rows", "kt_match_pods", "kt_check_pods", "kt_get_changed", "kt_get_reconcile_rows", "kt_step_submit", "kt_step_wait", "kt_admit_queue", "kt_get_timing", "kt_comm_unique_id",
    "kt_comm_init", "kt_comm_destroy", "kt_debug_compile_tables", "kt_debug_set_pass_plan", "kt_debug_get_pass_plan", "kt_debug_get_ns_tables",
    "kt_debug_set_row_order", "kt_debug_get_row_order",
]


def lib():
    """Load libkt_b200.so (must have been built: `python -c 'import __graft_entry__ as g; g.build()'`)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise KtError(abi.ERR_STATE, f"{LIB_PATH} is missing -- build it first (there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        vp = C.c_void_p
        L.kt_create.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(abi.Limits)]
        L.kt_destroy.argtypes = [vp]
        L.kt_destroy.restype = None
        L.kt_last_error.argtypes = [vp]
        L.kt_last_error.restype = C.c_char_p
        L.kt_version.restype = C.c_char_p
        L.kt_set_stream.argtypes = [vp, vp]
        L.kt_sync.argtypes = [vp]
        L.kt_enable_timing.argtypes = [vp, C.c_int]
        L.kt_enable_trace.argtypes = [vp, C.c_int]
        L.kt_get_trace.argtypes = [vp, vp, C.c_int64, vp]
        L.kt_get_trace.restype = C.c_int64
        L.kt_host_alloc.argtypes = [C.c_size_t]
        L.kt_host_alloc.restype = vp
        L.kt_host_alloc_upload.argtypes = [C.c_size_t]
        L.kt_host_alloc_upload.restype = vp
        L.kt_host_free.argtypes = [vp]
        L.kt_host_free.restype = None
        L.kt_upload_pods.argtypes = [vp, C.c_int, C.c_int64, vp, vp, vp, vp, vp]
        L.kt_set_async_uploads.argtypes = [vp, C.c_int]
        L.kt_upload_pods_compact.argtypes = [vp, C.c_int, C.c_int64, C.c_int32, vp, vp, vp, vp, vp]
        L.kt_upload_pods_packed.argtypes = [vp, C.c_int, C.c_int64, C.POINTER(abi.PackedPodsStruct)]
        L.kt_set_sparse_check.argtypes = [vp, C.c_int64]
        L.kt_get_check_sparse.argtypes = [vp, vp, vp, C.c_int64, C.POINTER(C.c_int64)]
        L.kt_step_submit.argtypes = [vp, C.c_int64, C.POINTER(abi.PackedPodsStruct), C.c_int64, C.POINTER(abi.PackedPodsStruct), C.c_int64, C.c_uint32]
        L.kt_step_wait.argtypes = [vp, C.POINTER(abi.StepResult)]
        L.kt_admit_queue.argtypes = [vp, C.c_int64, C.c_int64, C.c_uint32, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]
        L.kt_get_check_rows.argtypes = [vp, C.c_int64, vp, vp, vp]
        L.kt_get_match_rows.argtypes = [vp, C.c_int, C.c_int64, vp, vp]
        L.kt_check_pending_rows.argtypes = [vp, C.c_uint32, C.c_int64, vp, vp, vp, vp]
        L.kt_match_pods.argtypes = [vp, C.c_int64, vp, vp, vp]
        L.kt_check_pods.argtypes = [vp, C.c_uint32, C.c_int64, vp, vp, vp, vp, vp, vp, vp]
        L.kt_get_changed.argtypes = [vp, vp, C.c_int64, C.POINTER(C.c_int64), vp]
        L.kt_get_reconcile_rows.argtypes = [vp, C.c_int64, vp, C.POINTER(abi.ReconcileOut)]
        L.kt_update_pod_rows.argtypes = [vp, C.c_int, C.c_int64, vp, vp, vp, vp, vp, vp]
        L.kt_upload_namespaces.argtypes = [vp, C.c_int32, vp]
        L.kt_update_namespace_rows.argtypes = [vp, C.c_int32, C.c_int64, vp, vp]
        L.kt_upload_throttles.argtypes = [vp, C.c_int32, C.POINTER(abi.ThrottleCols), C.POINTER(abi.SelectorTable)]
        L.kt_upload_status.argtypes = [vp, C.POINTER(abi.StatusCols)]
        L.kt_set_reserved.argtypes = [vp, vp, vp, vp]
        L.kt_update_status_rows.argtypes = [vp, C.c_int64, vp, C.POINTER(abi.StatusCols)]
        L.kt_update_reserved_rows.argtypes = [vp, C.c_int64, vp, vp, vp, vp]
        L.kt_update_threshold_rows.argtypes = [vp, C.c_int64, vp, C.POINTER(abi.ThrottleCols)]
        L.kt_update_selector_rows.argtypes = [vp, C.c_int64, vp, C.POINTER(abi.ThrottleCols), C.POINTER(abi.SelectorTable), vp]
        L.kt_append_throttle_rows.argtypes = [vp, C.c_int64, C.POINTER(abi.ThrottleCols), C.POINTER(abi.SelectorTable), vp]
        L.kt_move_throttle_columns.argtypes = [vp, C.c_int32, vp]
        L.kt_evaluate.argtypes = [vp, C.c_int64, C.c_uint32]
        L.kt_get_reconcile.argtypes = [vp, C.POINTER(abi.ReconcileOut)]
        L.kt_match_words.argtypes = [vp]
        L.kt_match_words.restype = C.c_int32
        L.kt_get_match_bitmap.argtypes = [vp, C.c_int, vp]
        L.kt_get_match_columns.argtypes = [vp, C.c_int, C.c_int64, vp, vp, vp, vp, C.c_int64]
        L.kt_reconcile_throttles.argtypes = [vp, C.c_int64, C.c_int64, vp, C.POINTER(abi.ReconcileOut), vp, vp, C.c_int64]
        L.kt_get_check.argtypes = [vp, vp, vp]
        L.kt_get_check_summary.argtypes = [vp, C.c_int64, C.c_int64, vp, C.POINTER(abi.CheckSummary)]
        L.kt_get_timing.argtypes = [vp, C.POINTER(abi.Timing)]
        L.kt_comm_unique_id.argtypes = [vp]
        L.kt_comm_init.argtypes = [vp, vp, C.c_int, C.c_int]
        L.kt_comm_destroy.argtypes = [vp]
        L.kt_debug_compile_tables.argtypes = [C.POINTER(abi.Limits), C.c_int32, C.POINTER(abi.ThrottleCols), C.POINTER(abi.SelectorTable), C.c_int32, vp,
                                              vp, vp, vp, vp, vp, vp, vp, vp, vp]
        L.kt_debug_set_pass_plan.argtypes = [vp, C.POINTER(abi.PassPlan)]
        L.kt_debug_get_pass_plan.argtypes = [vp, C.POINTER(abi.PassPlan)]
        L.kt_debug_get_ns_tables.argtypes = [vp, vp, vp, vp, vp]
        L.kt_debug_set_row_order.argtypes = [vp, C.c_int, C.c_int]
        L.kt_debug_get_row_order.argtypes = [vp, C.c_int, vp, C.POINTER(C.c_int32)]
        _lib = L
    return _lib


class Pinned:
    """Pinned (cudaHostAlloc) host buffer exposed as a numpy array: `.array`.  Keep the object alive
    while the array is in use."""

    def __init__(self, shape, dtype, upload_only: bool = False):
        dtype = np.dtype(dtype)
        count = int(np.prod(shape))
        nbytes = max(count * dtype.itemsize, 1)
        self._ptr = (lib().kt_host_alloc_upload if upload_only else lib().kt_host_alloc)(nbytes)  # upload_only: write-combined
        if not self._ptr:
            raise KtError(abi.ERR_CUDA, "kt_host_alloc failed")
        self._buf = (C.c_char * nbytes).from_address(self._ptr)
        self.array = np.frombuffer(self._buf, dtype=dtype, count=count).reshape(shape)

    def __del__(self):
        try:
            if self._ptr:
                lib().kt_host_free(self._ptr)
                self._ptr = None
        except Exception:
            pass


class Engine:
    """One context == one GPU (one row shard in a multi-GPU run)."""

    def __init__(self, R: int, L: int, LN: int, device: int = 0):
        self._L = lib()
        self._h = C.c_void_p()
        self.R, self.Lslots, self.LN = R, L, LN
        lim = abi.Limits(abi.ABI_VERSION, R, L, LN)
        rc = self._L.kt_create(C.byref(self._h), device, C.byref(lim))
        if rc != 0:
            self._h = C.c_void_p()
            raise KtError(rc, "kt_create failed (no CUDA device? bad limits?) -- there is no CPU fallback")
        self.m = 0
        self.n = [0, 0]
        self._keep = []

    # -- plumbing -----------------------------------------------------------------------------
    def _ck(self, rc: int):
        if rc != 0:
            raise KtError(rc, self._L.kt_last_error(self._h).decode())

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._L.kt_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream: Optional[int]):
        self._ck(self._L.kt_set_stream(self._h, cuda_stream))

    def enable_timing(self, on: bool = True):
        self._ck(self._L.kt_enable_timing(self._h, int(on)))

    def enable_trace(self, on: bool = True):
        self._ck(self._L.kt_enable_trace(self._h, int(on)))

    def trace(self):
        """(rows[n][32] = ticket, sm, start_ns, end_ns, 12 stage stamps (4.. per role, see kt_kernels.cuh), 12 cycle counts, CTA, CTA exit_ns;
        roles[4] = match tiles, reconcile tiles, status tiles, CTAs launched) of the last fused pass: one row per match / reconcile / status tile."""
        roles = np.zeros(4, np.uint32)
        n = self._L.kt_get_trace(self._h, None, 0, roles.ctypes.data)
        rows = np.zeros((int(roles.sum()), 32), np.uint64)
        n = self._L.kt_get_trace(self._h, rows.ctypes.data, rows.shape[0], roles.ctypes.data)
        if n < 0:
            self._ck(int(n))
        return rows[: int(n)], roles

    def sync(self):
        self._ck(self._L.kt_sync(self._h))

    def set_pass_plan(self, threads: int = 0, decide: int = 0, max_ctas: int = 0):
        """Test seam: force the fused pass's build (512 / 768 threads per SM), decide mode (abi.PLAN_DECIDE_*) and a cap on its
        grid; all zero restores the automatic choices.  Diagnostic only (kt_debug_set_pass_plan)."""
        plan = abi.PassPlan(threads_per_sm=threads, decide=decide, max_ctas=max_ctas)
        self._ck(self._L.kt_debug_set_pass_plan(self._h, C.byref(plan)))

    def pass_plan(self) -> abi.PassPlan:
        """What the last fused pass ran: build, decide mode, grid, capacity, kernel variant, pieces per role."""
        plan = abi.PassPlan()
        self._ck(self._L.kt_debug_get_pass_plan(self._h, C.byref(plan)))
        return plan

    def set_row_order(self, kind: int, mode: int):
        """Test seam: store the rows of `kind` as given (abi.ROW_ORDER_AS_GIVEN), by namespace (abi.ROW_ORDER_BY_NAMESPACE) or as
        the engine chooses from the rows (abi.ROW_ORDER_AUTO, the default), from the next full upload on (kt_debug_set_row_order)."""
        self._ck(self._L.kt_debug_set_row_order(self._h, kind, mode))

    def row_order(self, kind: int):
        """(clustered, dev_row[n]) of the resident rows of `kind`: whether they are laid out by namespace, and the device row of
        every caller row (kt_debug_get_row_order)."""
        n = self.n[kind] if kind in (abi.PODS_RUNNING, abi.PODS_PENDING) else 0
        dev_row = np.zeros(max(n, 1), np.int64)
        clustered = C.c_int32(0)
        self._ck(self._L.kt_debug_get_row_order(self._h, kind, abi.ptr(dev_row), C.byref(clustered)))
        return bool(clustered.value), dev_row[:n]

    # -- uploads ------------------------------------------------------------------------------
    def upload_pods(self, kind: int, pods: PodCols):
        self._ck(self._L.kt_upload_pods(self._h, kind, pods.n, abi.ptr(pods.labels), abi.ptr(pods.req), abi.ptr(pods.present),
                                        abi.ptr(pods.flags), abi.ptr(pods.ns_id)))
        self.n[kind] = pods.n

    def set_async_uploads(self, on: bool = True):
        """Uploads return once queued; the host buffers must stay untouched until sync() / a getter returns."""
        self._ck(self._L.kt_set_async_uploads(self._h, int(on)))

    def upload_pods_compact(self, kind: int, cp: "abi.CompactPodCols"):
        """kt_upload_pods_compact: 56 instead of 108 bytes per row over the host link; expanded to the same int64 columns on the device."""
        self._ck(self._L.kt_upload_pods_compact(self._h, kind, cp.n, cp.val_bits, abi.ptr(cp.labels32), abi.ptr(cp.req32), abi.ptr(cp.req_shift),
                                                abi.ptr(cp.present), abi.ptr(cp.meta)))
        self.n[kind] = cp.n

    def upload_pods_packed(self, kind: int, pk: "abi.PackedPodCols"):
        """kt_upload_pods_packed: 36 bytes per row (L=8, R=4): 16-bit label-pair indices, presence inside the meta word."""
        st = pk.struct()
        self._ck(self._L.kt_upload_pods_packed(self._h, kind, pk.n, C.byref(st)))
        self.n[kind] = pk.n

    def update_pod_rows(self, kind: int, rows: np.ndarray, pods: PodCols):
        rows = np.ascontiguousarray(rows, np.int64)
        self._ck(self._L.kt_update_pod_rows(self._h, kind, rows.shape[0], abi.ptr(rows), abi.ptr(pods.labels), abi.ptr(pods.req),
                                            abi.ptr(pods.present), abi.ptr(pods.flags), abi.ptr(pods.ns_id)))

    def upload_namespaces(self, ns_labels: np.ndarray):
        self._ck(self._L.kt_upload_namespaces(self._h, ns_labels.shape[1], abi.ptr(ns_labels)))

    def ns_tables(self):
        """Test seam: the resident namespace masks and word lists, {NS, nsmask[NS][W][TPpad], nsw_off[NS+1], nsw_idx, max_ns_words}."""
        dims = np.zeros(5, np.int32)
        self._ck(self._L.kt_debug_get_ns_tables(self._h, abi.ptr(dims), None, None, None))
        NS, nnsw, mx, W, TPpad = (int(x) for x in dims)
        mask, off, idx = np.zeros((NS, W, TPpad), np.uint32), np.zeros(NS + 1, np.int32), np.zeros(max(nnsw, 1), np.int32)
        self._ck(self._L.kt_debug_get_ns_tables(self._h, abi.ptr(dims), abi.ptr(mask), abi.ptr(off), abi.ptr(idx)))
        return dict(NS=NS, nsmask=mask, nsw_off=off, nsw_idx=idx[:nnsw], max_ns_words=mx)

    def update_namespace_rows(self, n_ns: int, idx: np.ndarray, labels: np.ndarray):
        """kt_update_namespace_rows: the rows of the listed namespaces replaced by labels[LN][k], the count grown to n_ns (rows
        it grows by that are not listed are label-less); the tables' namespace masks and word lists are rebuilt on the device."""
        idx = np.ascontiguousarray(idx, np.int32)
        labels = abi._arr(labels, np.int64, (self.LN, idx.shape[0]))
        self._ck(self._L.kt_update_namespace_rows(self._h, int(n_ns), idx.shape[0], abi.ptr(idx), abi.ptr(labels)))

    def upload_throttles(self, snap: Snapshot):
        cols, sel = snap.throttle_cols(), snap.selector_table()
        self._ck(self._L.kt_upload_throttles(self._h, snap.m, C.byref(cols), C.byref(sel)))
        self.m = snap.m

    def upload_status(self, snap: Snapshot):
        st = snap.status_cols()
        self._ck(self._L.kt_upload_status(self._h, C.byref(st)))

    def set_reserved(self, snap: Snapshot):
        self._ck(self._L.kt_set_reserved(self._h, abi.ptr(snap.reserved), abi.ptr(snap.reserved_present), abi.ptr(snap.reserved_cnt)))

    def update_status_rows(self, idx: np.ndarray, status: dict):
        """kt_update_status_rows: the observed status of the listed throttle columns, replaced in place.  `status` holds the k
        listed columns, named and shaped like Snapshot.status ([R][k] / [k]); idx entries distinct and in [0, m)."""
        idx = np.ascontiguousarray(idx, np.int32)
        k, R = idx.shape[0], self.R
        cols = dict(calculated=abi._arr(status["calculated"], np.uint8), calc_thr=abi._arr(status["calc_thr"], np.int64, (R, k)),
                    calc_present=abi._arr(status["calc_present"], np.uint32), calc_cnt=abi._arr(status["calc_cnt"], np.int64),
                    used=abi._arr(status["used"], np.int64, (R, k)), used_present=abi._arr(status["used_present"], np.uint32),
                    used_cnt=abi._arr(status["used_cnt"], np.int64), throttled=abi._arr(status["throttled"], np.uint32))
        st = abi.StatusCols(*(abi.ptr(cols[f]) for f in ("calculated", "calc_thr", "calc_present", "calc_cnt", "used", "used_present", "used_cnt", "throttled")))
        self._ck(self._L.kt_update_status_rows(self._h, k, abi.ptr(idx), C.byref(st)))

    def update_threshold_rows(self, idx: np.ndarray, cols: dict):
        """kt_update_threshold_rows: spec.threshold and the temporaryThresholdOverrides of the listed throttle columns, replaced
        without recompiling the tables.  `cols` holds the k listed columns, named and shaped like the Snapshot fields: thr[R][k],
        thr_present[k], thr_cnt[k], ovr_off[k+1], and ovr_begin / ovr_end / ovr_flags / ovr_present / ovr_cnt [n_ovr] and
        ovr_thr[R][n_ovr] with n_ovr = ovr_off[k]; idx entries distinct and in [0, m)."""
        idx = np.ascontiguousarray(idx, np.int32)
        k, R = idx.shape[0], self.R
        off = abi._arr(cols["ovr_off"], np.int32)
        n = int(off[-1]) if off.shape[0] else 0
        a = dict(thr=abi._arr(cols["thr"], np.int64, (R, k)), thr_present=abi._arr(cols["thr_present"], np.uint32),
                 thr_cnt=abi._arr(cols["thr_cnt"], np.int64), ovr_off=off, ovr_begin=abi._arr(cols["ovr_begin"], np.int64),
                 ovr_end=abi._arr(cols["ovr_end"], np.int64), ovr_flags=abi._arr(cols["ovr_flags"], np.uint8),
                 ovr_thr=abi._arr(cols["ovr_thr"], np.int64, (R, n)), ovr_present=abi._arr(cols["ovr_present"], np.uint32),
                 ovr_cnt=abi._arr(cols["ovr_cnt"], np.int64))
        tc = abi.ThrottleCols(None, None, None, abi.ptr(a["thr"]), abi.ptr(a["thr_present"]), abi.ptr(a["thr_cnt"]), abi.ptr(off), n,
                              abi.ptr(a["ovr_begin"]), abi.ptr(a["ovr_end"]), abi.ptr(a["ovr_flags"]), abi.ptr(a["ovr_thr"]),
                              abi.ptr(a["ovr_present"]), abi.ptr(a["ovr_cnt"]))
        self._ck(self._L.kt_update_threshold_rows(self._h, k, abi.ptr(idx), C.byref(tc)))

    def update_selector_rows(self, idx: np.ndarray, cols: dict) -> bool:
        """kt_update_selector_rows: kind, ns_id, flags and the selector terms of the listed throttle columns replaced (a deletion is
        zero terms and flags 0).  `cols` holds the k listed columns: kind[k], thr_ns[k], thr_flags[k], and a CSR over them in idx
        order named like the Snapshot fields -- term_off[k+1], term_flags, pod_req_off, ns_req_off, req_key, req_op, req_val_off,
        req_vals.  Returns whether the engine compiled the tables again (a column did not fit the resident tables)."""
        idx = np.ascontiguousarray(idx, np.int32)
        k = idx.shape[0]
        a = dict(kind=abi._arr(cols["kind"], np.uint8), ns=abi._arr(cols["thr_ns"], np.int32), flags=abi._arr(cols["thr_flags"], np.uint8),
                 term_off=abi._arr(cols["term_off"], np.int32), term_flags=abi._arr(cols["term_flags"], np.uint8),
                 pod_req_off=abi._arr(cols["pod_req_off"], np.int32), ns_req_off=abi._arr(cols["ns_req_off"], np.int32),
                 req_key=abi._arr(cols["req_key"], np.uint32), req_op=abi._arr(cols["req_op"], np.uint8),
                 req_val_off=abi._arr(cols["req_val_off"], np.int32), req_vals=abi._arr(cols["req_vals"], np.uint32))
        tc = abi.ThrottleCols(abi.ptr(a["kind"]), abi.ptr(a["ns"]), abi.ptr(a["flags"]), None, None, None, None, 0, None, None, None, None,
                              None, None)
        st = abi.SelectorTable(int(a["term_off"][-1]) if a["term_off"].shape[0] else 0, int(a["req_key"].shape[0]), int(a["req_vals"].shape[0]),
                               *(abi.ptr(a[f]) for f in ("term_off", "term_flags", "pod_req_off", "ns_req_off", "req_key", "req_op", "req_val_off", "req_vals")))
        out = np.zeros(1, np.int32)
        self._ck(self._L.kt_update_selector_rows(self._h, k, abi.ptr(idx), C.byref(tc), C.byref(st), abi.ptr(out)))
        return bool(out[0])

    def append_throttle_rows(self, cols: dict) -> bool:
        """kt_append_throttle_rows: k new throttle columns appended at [m, m+k), their status and reservations zero.  `cols` holds
        the k new columns named and shaped like the Snapshot fields: kind, thr_ns, thr_flags, thr[R][k], thr_present, thr_cnt,
        ovr_off[k+1] and the override columns, and the selector CSR (term_off[k+1], term_flags, pod_req_off, ns_req_off, req_key,
        req_op, req_val_off, req_vals).  Returns whether the engine compiled the tables again (a column did not fit them)."""
        k, R = int(np.asarray(cols["kind"]).shape[0]), self.R
        off = abi._arr(cols["ovr_off"], np.int32)
        n = int(off[-1]) if off.shape[0] else 0
        a = dict(kind=abi._arr(cols["kind"], np.uint8), ns=abi._arr(cols["thr_ns"], np.int32), flags=abi._arr(cols["thr_flags"], np.uint8),
                 thr=abi._arr(cols["thr"], np.int64, (R, k)), thr_present=abi._arr(cols["thr_present"], np.uint32),
                 thr_cnt=abi._arr(cols["thr_cnt"], np.int64), ovr_off=off, ovr_begin=abi._arr(cols["ovr_begin"], np.int64),
                 ovr_end=abi._arr(cols["ovr_end"], np.int64), ovr_flags=abi._arr(cols["ovr_flags"], np.uint8),
                 ovr_thr=abi._arr(cols["ovr_thr"], np.int64, (R, n)), ovr_present=abi._arr(cols["ovr_present"], np.uint32),
                 ovr_cnt=abi._arr(cols["ovr_cnt"], np.int64),
                 term_off=abi._arr(cols["term_off"], np.int32), term_flags=abi._arr(cols["term_flags"], np.uint8),
                 pod_req_off=abi._arr(cols["pod_req_off"], np.int32), ns_req_off=abi._arr(cols["ns_req_off"], np.int32),
                 req_key=abi._arr(cols["req_key"], np.uint32), req_op=abi._arr(cols["req_op"], np.uint8),
                 req_val_off=abi._arr(cols["req_val_off"], np.int32), req_vals=abi._arr(cols["req_vals"], np.uint32))
        tc = abi.ThrottleCols(*(abi.ptr(a[f]) for f in ("kind", "ns", "flags", "thr", "thr_present", "thr_cnt", "ovr_off")), n,
                              *(abi.ptr(a[f]) for f in ("ovr_begin", "ovr_end", "ovr_flags", "ovr_thr", "ovr_present", "ovr_cnt")))
        st = abi.SelectorTable(int(a["term_off"][-1]) if a["term_off"].shape[0] else 0, int(a["req_key"].shape[0]), int(a["req_vals"].shape[0]),
                               *(abi.ptr(a[f]) for f in ("term_off", "term_flags", "pod_req_off", "ns_req_off", "req_key", "req_op", "req_val_off", "req_vals")))
        out = np.zeros(1, np.int32)
        self._ck(self._L.kt_append_throttle_rows(self._h, k, C.byref(tc), C.byref(st), abi.ptr(out)))
        self.m += k
        return bool(out[0])

    def move_throttle_columns(self, src) -> None:
        """kt_move_throttle_columns: the throttle columns laid out again, column j taking previous column src[j] (spec, thresholds,
        overrides, status and reservations), or an empty column for -1; previous columns src does not name are dropped."""
        a = abi._arr(src, np.int32)
        self._ck(self._L.kt_move_throttle_columns(self._h, int(a.shape[0]), abi.ptr(a)))
        self.m = int(a.shape[0])

    def update_reserved_rows(self, idx: np.ndarray, reserved: np.ndarray, present: np.ndarray, cnt: np.ndarray):
        """kt_update_reserved_rows: reserved[R][k], present[k], cnt[k] of the listed throttle columns, replaced in place (the
        columns never set since the last set_reserved(None) / upload_throttles count as nothing reserved)."""
        idx = np.ascontiguousarray(idx, np.int32)
        k = idx.shape[0]
        reserved = abi._arr(reserved, np.int64, (self.R, k))
        present, cnt = abi._arr(present, np.uint32), abi._arr(cnt, np.int64)
        self._ck(self._L.kt_update_reserved_rows(self._h, k, abi.ptr(idx), abi.ptr(reserved), abi.ptr(present), abi.ptr(cnt)))

    def upload_snapshot(self, snap: Snapshot):
        """Everything a pass needs, in dependency order."""
        snap.normalize()
        self.upload_namespaces(snap.ns_labels)
        self.upload_throttles(snap)
        if snap.reserved is not None:
            self.set_reserved(snap)
        if snap.status is not None:
            self.upload_status(snap)
        self.upload_pods(abi.PODS_RUNNING, snap.running)
        self.upload_pods(abi.PODS_PENDING, snap.pending)

    # -- the pass -------------------------------------------------------------------------------
    def evaluate(self, now: int, flags: int = abi.EVAL_FRESH_STATUS):
        self._ck(self._L.kt_evaluate(self._h, now, flags))

    @property
    def words_per_row(self) -> int:
        return int(self._L.kt_match_words(self._h))

    def timing(self) -> abi.Timing:
        t = abi.Timing()
        self._ck(self._L.kt_get_timing(self._h, C.byref(t)))
        return t

    # -- downloads ------------------------------------------------------------------------------
    def download(self, out: Optional[PassResult] = None, bitmaps: bool = True) -> PassResult:
        W = self.words_per_row
        if out is None:
            z = np.zeros
            m, R = self.m, self.R
            N, P = self.n
            out = PassResult(W, z((R, m), np.int64), z(m, np.uint32), z(m, np.int64), z(m, np.uint32), z((R, m), np.int64),
                             z(m, np.uint32), z(m, np.int64), z(m, np.uint8), z((N if bitmaps else 0, W), np.uint32),
                             z((P if bitmaps else 0, W), np.uint32), z((P, 2 * W), np.uint32), z(P, np.uint8))
        rec = out.reconcile_out()
        self._ck(self._L.kt_get_reconcile(self._h, C.byref(rec)))
        if bitmaps:
            if self.n[0]:
                self._ck(self._L.kt_get_match_bitmap(self._h, abi.PODS_RUNNING, abi.ptr(out.run_bitmap)))
            if self.n[1]:
                self._ck(self._L.kt_get_match_bitmap(self._h, abi.PODS_PENDING, abi.ptr(out.pend_bitmap)))
        self._ck(self._L.kt_get_check(self._h, abi.ptr(out.codes), abi.ptr(out.admit)))
        return out

    def get_check(self, codes: Optional[np.ndarray], admit: Optional[np.ndarray]):
        self._ck(self._L.kt_get_check(self._h, abi.ptr(codes), abi.ptr(admit)))

    def check_summary(self, first: int, count: int, row_class: Optional[np.ndarray] = None):
        """The pending rows [first, first + count) of the last checking pass summarised per throttle: (status_cnt[3][m] by code
        ACTIVE / INSUFFICIENT / POD_REQUESTS_EXCEEDS_THRESHOLD, sole_cnt[m], held[R][m], held_present[m]).  row_class[count]
        (None: all 1) is 0 skip, 1 count, 2 count but never as the only blocker (kt_get_check_summary)."""
        m, R, z = self.m, self.R, np.zeros
        status_cnt, sole_cnt, held, held_present = z((3, m), np.int64), z(m, np.int64), z((R, m), np.int64), z(m, np.uint32)
        cls = None if row_class is None else np.ascontiguousarray(row_class, np.uint8)
        if cls is not None and cls.shape[0] != count:
            raise ValueError(f"row_class has {cls.shape[0]} entries, count is {count}")
        out = abi.CheckSummary(abi.ptr(status_cnt), abi.ptr(sole_cnt), abi.ptr(held), abi.ptr(held_present))
        self._ck(self._L.kt_get_check_summary(self._h, first, count, abi.ptr(cls), C.byref(out)))
        return status_cnt, sole_cnt, held, held_present

    def set_sparse_check(self, cap_entries: int):
        """Later passes also append every non-zero code word to a device list (0: off)."""
        self._ck(self._L.kt_set_sparse_check(self._h, cap_entries))

    def get_check_sparse(self, admit: Optional[np.ndarray], entries: np.ndarray) -> int:
        """admit[p] and the non-zero code words as rows {pending row, word index, codes}; returns their total number
        (more than entries.shape[0]: read the dense rows with get_check instead)."""
        n = C.c_int64(0)
        self._ck(self._L.kt_get_check_sparse(self._h, abi.ptr(admit), abi.ptr(entries), entries.shape[0], C.byref(n)))
        return int(n.value)

    # -- one end-to-end step in one call ----------------------------------------------------------
    def step_submit(self, running, pending, now: int, flags: int = abi.EVAL_FRESH_STATUS):
        """Queue packed uploads (abi.PackedPodCols or a prepared (n, struct) pair; None keeps the resident rows) + the pass + the
        result copies; returns at once.  The host columns must stay untouched until step_wait()."""
        def prep(x):
            if x is None:
                return 0, None
            if isinstance(x, tuple):
                return x
            return x.n, x.struct()
        (nr, sr), (np_, sp) = prep(running), prep(pending)
        self._ck(self._L.kt_step_submit(self._h, nr, C.byref(sr) if sr is not None else None, np_, C.byref(sp) if sp is not None else None, now, flags))
        if running is not None:
            self.n[abi.PODS_RUNNING] = nr
        if pending is not None:
            self.n[abi.PODS_PENDING] = np_

    def step_wait(self) -> "abi.StepResult":
        """Block until the submitted step's results have landed; the returned struct points into the library's pinned block
        (valid until the next step_submit): .admit [n_pending] u8, .entries [n_sparse][3] u32, .status columns."""
        res = abi.StepResult()
        self._ck(self._L.kt_step_wait(self._h, C.byref(res)))
        return res

    def admit_queue(self, first: int, count: int, flags: int = 0):
        """Queue-ordered greedy admission of the pending rows [first, first + count) on the device: (rounds, admitted)."""
        rounds, admitted = C.c_int32(0), C.c_int64(0)
        self._ck(self._L.kt_admit_queue(self._h, first, count, flags, C.byref(rounds), C.byref(admitted)))
        return int(rounds.value), int(admitted.value)

    def get_check_rows(self, rows: np.ndarray):
        """(codes[k][2W], admit[k]) of the listed pending rows."""
        rows = np.ascontiguousarray(rows, np.int64)
        codes = np.zeros((rows.shape[0], 2 * self.words_per_row), np.uint32)
        admit = np.zeros(rows.shape[0], np.uint8)
        self._ck(self._L.kt_get_check_rows(self._h, rows.shape[0], abi.ptr(rows), abi.ptr(codes), abi.ptr(admit)))
        return codes, admit

    def check_pending_rows(self, rows, on_equal: bool = False):
        """PreFilter of the listed pending rows as they are now, without a pass over the pending table: (words[k][W], codes[k][2W],
        admit[k]) -- what a GIVEN_STATUS | SKIP_RECONCILE pass followed by match_rows(PENDING) / get_check_rows would return."""
        rows = np.ascontiguousarray(rows, np.int64)
        k, W = rows.shape[0], self.words_per_row
        words, codes, admit = np.zeros((k, W), np.uint32), np.zeros((k, 2 * W), np.uint32), np.zeros(k, np.uint8)
        flags = abi.EVAL_ON_EQUAL if on_equal else 0
        self._ck(self._L.kt_check_pending_rows(self._h, flags, k, abi.ptr(rows), abi.ptr(words), abi.ptr(codes), abi.ptr(admit)))
        return words, codes, admit

    def match_pods(self, labels, ns_id) -> np.ndarray:
        """affectedThrottles of k pods given by value (label codes [L][k], namespace ids [k]), matched against the tables as they
        are now: words[k][W], what match_rows(PENDING) returns for pending rows holding the same labels and namespaces."""
        labels = np.ascontiguousarray(labels, np.int64).reshape(self.Lslots, -1)
        ns_id = np.ascontiguousarray(ns_id, np.int32)
        k = ns_id.shape[0]
        if labels.shape[1] != k:
            raise ValueError(f"labels has {labels.shape[1]} pods, ns_id {k}")
        words = np.zeros((k, self.words_per_row), np.uint32)
        self._ck(self._L.kt_match_pods(self._h, k, abi.ptr(labels), abi.ptr(ns_id), abi.ptr(words)))
        return words

    def check_pods(self, labels, req, present, ns_id, on_equal: bool = False):
        """PreFilter of k pods given by value (label codes [L][k], requests [R][k], presence bits [k], namespace ids [k]: the
        columns of upload_pods without the flags, which the pass never reads for a pending row), checked against the tables,
        observed status and reservations as they are now, with no pending row read: (words[k][W], codes[k][2W], admit[k]) --
        what check_pending_rows returns for pending rows holding the same values."""
        labels = np.ascontiguousarray(labels, np.int64).reshape(self.Lslots, -1)
        ns_id = np.ascontiguousarray(ns_id, np.int32)
        k = ns_id.shape[0]
        req = np.ascontiguousarray(req, np.int64).reshape(self.R, -1)
        present = np.ascontiguousarray(present, np.uint32)
        if labels.shape[1] != k or req.shape[1] != k or present.shape[0] != k:
            raise ValueError(f"column lengths differ: labels {labels.shape[1]}, req {req.shape[1]}, present {present.shape[0]}, ns_id {k}")
        W = self.words_per_row
        words, codes, admit = np.zeros((k, W), np.uint32), np.zeros((k, 2 * W), np.uint32), np.zeros(k, np.uint8)
        flags = abi.EVAL_ON_EQUAL if on_equal else 0
        self._ck(self._L.kt_check_pods(self._h, flags, k, abi.ptr(labels), abi.ptr(req), abi.ptr(present), abi.ptr(ns_id),
                                       abi.ptr(words), abi.ptr(codes), abi.ptr(admit)))
        return words, codes, admit

    def match_rows(self, kind: int, rows: np.ndarray) -> np.ndarray:
        """words[k][words_per_row]: the match bitmap rows of the listed rows of a kind, gathered on the device."""
        rows = np.ascontiguousarray(rows, np.int64)
        words = np.zeros((rows.shape[0], self.words_per_row), np.uint32)
        self._ck(self._L.kt_get_match_rows(self._h, kind, rows.shape[0], abi.ptr(rows), abi.ptr(words)))
        return words

    def match_columns(self, kind: int, idx, cap: Optional[int] = None):
        """affectedPods from the throttles' side: (off[k+1], rows, codes) with throttle idx[j]'s rows, ascending, in
        rows[off[j]:off[j+1]]; codes (PENDING only, else None) the 2-bit check code of each (row, idx[j]).  `cap` sizes the
        first attempt (default: the rows of the kind); a larger relation is fetched again with the exact room."""
        idx = np.ascontiguousarray(idx, np.int32)
        k = idx.shape[0]
        off = np.zeros(k + 1, np.int64)
        cap = self.n[kind] if cap is None else cap
        while True:
            rows = np.zeros(max(cap, 1), np.int64)
            codes = np.zeros(max(cap, 1), np.uint8) if kind == abi.PODS_PENDING else None
            self._ck(self._L.kt_get_match_columns(self._h, kind, k, abi.ptr(idx), abi.ptr(off), abi.ptr(rows), abi.ptr(codes), cap))
            total = int(off[k])
            if total <= cap:
                return off, rows[:total], (codes[:total] if codes is not None else None)
            cap = total

    def reconcile_throttles(self, now: int, idx, cap: Optional[int] = None):
        """reconcile(key) of the listed throttles at `now` on the running rows as they are: (status columns shaped for len(idx)
        throttles as get_reconcile_rows returns them, off[k+1], rows) with throttle idx[j]'s matched rows, ascending, in
        rows[off[j]:off[j+1]].  `cap` sizes the first attempt (default: the running rows)."""
        idx = np.ascontiguousarray(idx, np.int32)
        k, R, z = idx.shape[0], self.R, np.zeros
        out = PassResult(self.words_per_row, z((R, k), np.int64), z(k, np.uint32), z(k, np.int64), z(k, np.uint32), z((R, k), np.int64), z(k, np.uint32),
                         z(k, np.int64), z(k, np.uint8), z((0, 1), np.uint32), z((0, 1), np.uint32), z((0, 1), np.uint32), z(0, np.uint8))
        rec = out.reconcile_out()
        off = np.zeros(k + 1, np.int64)
        cap = self.n[abi.PODS_RUNNING] if cap is None else cap
        while True:
            rows = np.zeros(max(cap, 1), np.int64)
            self._ck(self._L.kt_reconcile_throttles(self._h, now, k, abi.ptr(idx), C.byref(rec), abi.ptr(off), abi.ptr(rows), cap))
            total = int(off[k])
            if total <= cap:
                return out, off, rows[:total]
            cap = total

    def get_changed(self):
        """(sorted indices of the throttles whose status this pass changes, flags[m]) -- the device-side diff against kt_upload_status."""
        idx = np.zeros(max(self.m, 1), np.int32)
        flags = np.zeros(max(self.m, 1), np.uint8)
        n = C.c_int64(0)
        self._ck(self._L.kt_get_changed(self._h, abi.ptr(idx), idx.shape[0], C.byref(n), abi.ptr(flags)))
        return np.sort(idx[: int(n.value)]), flags[: self.m]

    def get_reconcile_rows(self, idx: np.ndarray) -> PassResult:
        """Status columns of the listed throttles only (shaped for len(idx) throttles)."""
        idx = np.ascontiguousarray(idx, np.int32)
        k, R, z = idx.shape[0], self.R, np.zeros
        out = PassResult(self.words_per_row, z((R, k), np.int64), z(k, np.uint32), z(k, np.int64), z(k, np.uint32), z((R, k), np.int64), z(k, np.uint32),
                         z(k, np.int64), z(k, np.uint8), z((0, 1), np.uint32), z((0, 1), np.uint32), z((0, 1), np.uint32), z(0, np.uint8))
        rec = out.reconcile_out()
        self._ck(self._L.kt_get_reconcile_rows(self._h, k, abi.ptr(idx), C.byref(rec)))
        return out

    def get_reconcile(self, out: PassResult):
        rec = out.reconcile_out()
        self._ck(self._L.kt_get_reconcile(self._h, C.byref(rec)))

    # -- multi-GPU --------------------------------------------------------------------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        rc = lib().kt_comm_unique_id(buf)
        if rc != 0:
            raise KtError(rc, "kt_comm_unique_id failed (libnccl.so.2 missing?)")
        return bytes(buf)

    def comm_init(self, uid: bytes, nranks: int, rank: int):
        buf = (C.c_uint8 * 128).from_buffer_copy(uid)
        self._ck(self._L.kt_comm_init(self._h, buf, nranks, rank))

    def comm_destroy(self):
        self._ck(self._L.kt_comm_destroy(self._h))


def evaluate_snapshot(snap: Snapshot, flags: int = abi.EVAL_FRESH_STATUS, device: int = 0) -> PassResult:
    """Convenience: upload + one pass + download on one GPU."""
    eng = Engine(snap.R, snap.L, snap.LN, device)
    try:
        eng.upload_snapshot(snap)
        eng.evaluate(snap.now, flags)
        return eng.download()
    finally:
        eng.close()
