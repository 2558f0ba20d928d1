"""ctypes mirror of include/kt_b200.h (the C ABI of the engine) plus the columnar Snapshot
container that both the engine wrapper and the test-side oracle wrapper consume.

Nothing here computes anything: it only describes memory.  Field order and types must match
include/kt_b200.h exactly (tests/test_abi.py checks sizes against the compiled library).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

ABI_VERSION = 1
MAX_RESOURCES = 31
COUNT_BIT = 0x80000000
MAX_LABEL_SLOTS = 32
LABEL_EMPTY = -1
TIME_OPEN_BEGIN = -(2**63)
TIME_OPEN_END = 2**63 - 1

OK, ERR_INVALID, ERR_CUDA, ERR_STATE, ERR_LIMIT, ERR_NCCL = 0, -1, -2, -3, -4, -5
PODS_RUNNING, PODS_PENDING = 0, 1
POD_SCHEDULER_MATCH, POD_SCHEDULED, POD_NOT_FINISHED = 1, 2, 4
THR_RESPONSIBLE, THR_SELECTOR_ERROR = 1, 2
KIND_THROTTLE, KIND_CLUSTERTHROTTLE = 0, 1
OP_IN, OP_NOTIN, OP_EXISTS, OP_DOESNOTEXIST = 0, 1, 2, 3
TERM_NS_INVALID, TERM_POD_INVALID = 1, 2
OVR_PARSE_ERROR = 1
CHECK_NOT_THROTTLED, CHECK_ACTIVE, CHECK_INSUFFICIENT, CHECK_POD_REQUESTS_EXCEEDS_THRESHOLD = 0, 1, 2, 3
CHECK_NAMES = ("not-throttled", "active", "insufficient", "pod-requests-exceeds-threshold")
EVAL_FRESH_STATUS, EVAL_GIVEN_STATUS, EVAL_ON_EQUAL, EVAL_SKIP_RECONCILE, EVAL_SKIP_CHECK = 0, 1, 2, 4, 8

_p = C.POINTER


class Limits(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("n_resources", C.c_int32), ("label_slots", C.c_int32),
                ("ns_label_slots", C.c_int32)]


class SelectorTable(C.Structure):
    _fields_ = [("n_terms", C.c_int32), ("n_reqs", C.c_int32), ("n_vals", C.c_int32),
                ("term_off", C.c_void_p), ("term_flags", C.c_void_p), ("pod_req_off", C.c_void_p),
                ("ns_req_off", C.c_void_p), ("req_key", C.c_void_p), ("req_op", C.c_void_p),
                ("req_val_off", C.c_void_p), ("req_vals", C.c_void_p)]


class ThrottleCols(C.Structure):
    _fields_ = [("kind", C.c_void_p), ("ns_id", C.c_void_p), ("flags", C.c_void_p), ("thr", C.c_void_p),
                ("thr_present", C.c_void_p), ("thr_cnt", C.c_void_p), ("ovr_off", C.c_void_p),
                ("n_ovr", C.c_int32), ("ovr_begin", C.c_void_p), ("ovr_end", C.c_void_p),
                ("ovr_flags", C.c_void_p), ("ovr_thr", C.c_void_p), ("ovr_present", C.c_void_p),
                ("ovr_cnt", C.c_void_p)]


class StatusCols(C.Structure):
    _fields_ = [("calculated", C.c_void_p), ("calc_thr", C.c_void_p), ("calc_present", C.c_void_p),
                ("calc_cnt", C.c_void_p), ("used", C.c_void_p), ("used_present", C.c_void_p),
                ("used_cnt", C.c_void_p), ("throttled", C.c_void_p)]


class ReconcileOut(C.Structure):
    _fields_ = [("used", C.c_void_p), ("used_present", C.c_void_p), ("used_cnt", C.c_void_p),
                ("throttled", C.c_void_p), ("calc_thr", C.c_void_p), ("calc_present", C.c_void_p),
                ("calc_cnt", C.c_void_p), ("override_active", C.c_void_p)]


class CheckSummary(C.Structure):  # kt_check_summary
    _fields_ = [("status_cnt", C.c_void_p), ("sole_cnt", C.c_void_p), ("held", C.c_void_p), ("held_present", C.c_void_p)]


class StepResult(C.Structure):  # kt_step_result
    _fields_ = [("n_pending", C.c_int64), ("n_sparse", C.c_int64), ("admit", C.c_void_p), ("entries", C.c_void_p), ("status", ReconcileOut)]


class Timing(C.Structure):
    _fields_ = [("reconcile_ms", C.c_float), ("allreduce_ms", C.c_float), ("finalize_ms", C.c_float),
                ("check_ms", C.c_float), ("total_ms", C.c_float), ("launches", C.c_int32)]


PLAN_DECIDE_QUAD, PLAN_DECIDE_PER_POD = 1, 2
ROW_ORDER_AUTO, ROW_ORDER_AS_GIVEN, ROW_ORDER_BY_NAMESPACE = 0, 1, 2  # kt_debug_set_row_order (test seam of the row layout)


class PassPlan(C.Structure):  # kt_pass_plan (test seam of the fused pass: kt_debug_set_pass_plan / kt_debug_get_pass_plan)
    _fields_ = [("threads_per_sm", C.c_int32), ("decide", C.c_int32), ("max_ctas", C.c_uint32), ("grid", C.c_uint32),
                ("capacity", C.c_uint32), ("tile", C.c_int32), ("tpc", C.c_int32), ("b", C.c_int32), ("rt", C.c_int32),
                ("n_chk", C.c_uint32), ("n_rec", C.c_uint32), ("n_fin", C.c_uint32), ("n_sub", C.c_uint32)]


def ptr(a: Optional[np.ndarray]) -> Optional[int]:
    """Raw address of a C-contiguous numpy array (None -> NULL)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"], "columns must be C-contiguous"
    return a.ctypes.data


def _arr(x, dtype, shape=None) -> np.ndarray:
    a = np.ascontiguousarray(x, dtype=dtype)
    if shape is not None:
        a = a.reshape(shape)
    return a


@dataclass
class PodCols:
    """One pod kind: labels[L][n] int64, req[R][n] int64, present[n] u32, flags[n] u32, ns_id[n] i32."""
    labels: np.ndarray
    req: np.ndarray
    present: np.ndarray
    flags: np.ndarray
    ns_id: np.ndarray

    @property
    def n(self) -> int:
        return int(self.present.shape[0])

    def normalized(self, L: int, R: int) -> "PodCols":
        n = self.n
        return PodCols(_arr(self.labels, np.int64, (L, n)), _arr(self.req, np.int64, (R, n)),
                       _arr(self.present, np.uint32, (n,)), _arr(self.flags, np.uint32, (n,)),
                       _arr(self.ns_id, np.int32, (n,)))

    def rows(self, sl) -> "PodCols":
        return PodCols(np.ascontiguousarray(self.labels[:, sl]), np.ascontiguousarray(self.req[:, sl]),
                       np.ascontiguousarray(self.present[sl]), np.ascontiguousarray(self.flags[sl]),
                       np.ascontiguousarray(self.ns_id[sl]))


@dataclass
class CompactPodCols:
    """The compact transfer format of kt_upload_pods_compact (include/kt_b200.h).  Built by a packer that knows its
    dictionaries; `compact_pods` below derives it from wide columns and REFUSES anything that would not expand exactly."""
    val_bits: int
    labels32: np.ndarray   # [L][n] u32
    req32: np.ndarray      # [R][n] i32
    req_shift: np.ndarray  # [R] i32
    present: np.ndarray    # [n] u32
    meta: np.ndarray       # [n] u32 = ns_id | flags << 29

    @property
    def n(self) -> int:
        return int(self.present.shape[0])

    @property
    def nbytes(self) -> int:
        return sum(a.nbytes for a in (self.labels32, self.req32, self.req_shift, self.present, self.meta))


def compact_pods(pods: PodCols, val_bits: int = 20) -> CompactPodCols:
    """Wide int64 pod columns -> compact transfer columns, exactly (raises ValueError when a value does not fit:
    key/value ids beyond the bit split, requests that are not multiples of a power of two small enough for int32,
    namespace ids >= 2^29).  Pure repacking; nothing is evaluated."""
    lab = pods.labels
    empty = lab == LABEL_EMPTY
    key, val = (lab >> 32) & 0xFFFFFFFF, lab & 0xFFFFFFFF
    if ((~empty) & ((key >> (32 - val_bits) != 0) | (val >> val_bits != 0))).any():
        raise ValueError(f"label ids do not fit a {32 - val_bits}+{val_bits} bit split")
    lab32 = np.where(empty, 0xFFFFFFFF, (key << val_bits) | val).astype(np.uint32)
    if ((~empty) & (lab32 == 0xFFFFFFFF)).any():
        raise ValueError("a label collides with the empty-slot code")
    R = pods.req.shape[0]
    shift = np.zeros(R, np.int32)
    req32 = np.zeros(pods.req.shape, np.int32)
    for r in range(R):
        col = pods.req[r]
        nz = col[col != 0]
        sh = 0
        if nz.size:
            low = int(np.bitwise_or.reduce(nz))           # common trailing zero bits of the column
            sh = min((low & -low).bit_length() - 1, 32)
            if np.abs(nz >> sh).max() >= 2**31:
                raise ValueError(f"resource column {r} does not fit int32 even after dropping {sh} common zero bits")
        shift[r] = sh
        req32[r] = (col >> sh).astype(np.int32)
    if pods.n and (int(pods.ns_id.max()) >= 1 << 29 or int(pods.ns_id.min()) < 0 or int(pods.flags.max()) > 7):
        raise ValueError("namespace id / flags do not fit the packed meta word")
    meta = (pods.ns_id.astype(np.uint32) | (pods.flags.astype(np.uint32) << np.uint32(29))).astype(np.uint32)
    return CompactPodCols(val_bits, np.ascontiguousarray(lab32), np.ascontiguousarray(req32), shift, np.ascontiguousarray(pods.present, np.uint32), meta)


class PackedPodsStruct(C.Structure):
    """kt_packed_pods (include/kt_b200.h)"""
    _fields_ = [("n_pairs", C.c_int32), ("ns_bits", C.c_int32), ("pairs", C.c_void_p), ("labels16", C.c_void_p), ("req32", C.c_void_p),
                ("req_shift", C.c_void_p), ("meta", C.c_void_p), ("req_dict", C.c_void_p), ("req_dict_off", C.c_void_p),
                ("req_code_bytes", C.c_void_p), ("req_codes", C.c_void_p)]


@dataclass
class PackedPodCols:
    """The packed transfer format of kt_upload_pods_packed: 16-bit indices into a dictionary of label pairs, presence in meta."""
    ns_bits: int
    pairs: np.ndarray      # [n_pairs] i64
    labels16: np.ndarray   # [L][n] u16
    req32: Optional[np.ndarray]      # [R][n] i32            } either these two ...
    req_shift: Optional[np.ndarray]  # [R] i32               }
    meta: np.ndarray       # [n] u32 = ns_id | flags << ns_bits | present << (ns_bits + 3)
    req_dict: Optional[np.ndarray] = None        # i64, the columns' distinct values one after another   } ... or these four
    req_dict_off: Optional[np.ndarray] = None    # [R+1] i32                                                }
    req_code_bytes: Optional[np.ndarray] = None  # [R] u8: 1 or 2                                           }
    req_codes: Optional[np.ndarray] = None       # u8 buffer: the code columns, each padded to 4 bytes      }

    @property
    def n(self) -> int:
        return int(self.meta.shape[0])

    @property
    def coded(self) -> bool:
        return self.req_codes is not None

    @property
    def nbytes(self) -> int:
        cols = (self.pairs, self.labels16, self.meta) + ((self.req_dict, self.req_dict_off, self.req_code_bytes, self.req_codes) if self.coded
                                                         else (self.req32, self.req_shift))
        return sum(a.nbytes for a in cols)

    def struct(self) -> PackedPodsStruct:
        if self.coded:
            return PackedPodsStruct(int(self.pairs.shape[0]), self.ns_bits, ptr(self.pairs), ptr(self.labels16), None, None, ptr(self.meta),
                                    ptr(self.req_dict), ptr(self.req_dict_off), ptr(self.req_code_bytes), ptr(self.req_codes))
        return PackedPodsStruct(int(self.pairs.shape[0]), self.ns_bits, ptr(self.pairs), ptr(self.labels16), ptr(self.req32), ptr(self.req_shift), ptr(self.meta),
                                None, None, None, None)

    def unpack(self, Lpad: int | None = None) -> "PodCols":
        """What k_unpack_packed writes into HBM, in numpy (test-side mirror of the device expansion)."""
        L, n = self.labels16.shape
        idx = self.labels16.astype(np.int64)
        lab = np.where(idx == 0xFFFF, LABEL_EMPTY, self.pairs[np.minimum(idx, max(len(self.pairs) - 1, 0))] if len(self.pairs) else LABEL_EMPTY)
        if self.coded:
            R = int(self.req_code_bytes.shape[0])
            req = np.zeros((R, n), np.int64)
            off = 0
            for r in range(R):
                b = int(self.req_code_bytes[r])
                codes = np.frombuffer(self.req_codes.tobytes()[off:off + n * b], dtype=np.uint8 if b == 1 else "<u2").astype(np.int64)
                d = self.req_dict[int(self.req_dict_off[r]):int(self.req_dict_off[r + 1])]
                req[r] = d[codes] if n else 0
                off += (n * b + 3) // 4 * 4
        else:
            R = self.req32.shape[0]
            req = self.req32.astype(np.int64) << self.req_shift.astype(np.int64)[:, None]
        m = self.meta.astype(np.uint64)
        ns = (m & np.uint64((1 << self.ns_bits) - 1)).astype(np.int32)
        flags = ((m >> np.uint64(self.ns_bits)) & np.uint64(7)).astype(np.uint32)
        present = ((m >> np.uint64(self.ns_bits + 3)) & np.uint64((1 << R) - 1)).astype(np.uint32)
        return PodCols(np.ascontiguousarray(lab, np.int64).reshape(L, n), np.ascontiguousarray(req), present, flags, ns)


def packed_pods(pods: PodCols, code_requests: bool = False) -> PackedPodCols:
    """Wide int64 pod columns -> packed transfer columns, exactly (raises ValueError when the snapshot uses more than 65535
    distinct label pairs, a request column does not fit int32 in any power-of-two unit, or namespace / flags / presence do
    not fit one meta word).  code_requests: dictionary-code the request columns (1 or 2 bytes per value; ValueError when a column
    has more than 65536 distinct values).  Pure repacking; nothing is evaluated."""
    lab = pods.labels
    empty = lab == LABEL_EMPTY
    pairs, inv = np.unique(lab[~empty], return_inverse=True)
    if pairs.shape[0] > 65535:
        raise ValueError(f"{pairs.shape[0]} distinct label pairs do not fit 16-bit indices")
    lab16 = np.full(lab.shape, 0xFFFF, np.uint16)
    lab16[~empty] = inv.astype(np.uint16)
    R = pods.req.shape[0]
    shift = np.zeros(R, np.int32)
    req32 = np.zeros(pods.req.shape, np.int32)
    coded = None
    if code_requests:
        dicts, offs, widths, chunks = [], [0], [], []
        for r in range(R):
            vals, inv = np.unique(pods.req[r], return_inverse=True)
            if vals.shape[0] > 65536:
                raise ValueError(f"resource column {r} has {vals.shape[0]} distinct values: no 16-bit codes")
            b = 1 if vals.shape[0] <= 256 else 2
            raw = inv.astype(np.uint8 if b == 1 else "<u2").tobytes()
            chunks.append(raw + b"\0" * (-len(raw) % 4))
            dicts.append(vals.astype(np.int64))
            offs.append(offs[-1] + vals.shape[0])
            widths.append(b)
        coded = (np.ascontiguousarray(np.concatenate(dicts) if dicts else np.zeros(0, np.int64)), np.asarray(offs, np.int32), np.asarray(widths, np.uint8),
                 np.frombuffer(b"".join(chunks), dtype=np.uint8).copy())
    else:
        for r in range(R):
            col = pods.req[r]
            nz = col[col != 0]
            sh = 0
            if nz.size:
                low = int(np.bitwise_or.reduce(nz))
                sh = min((low & -low).bit_length() - 1, 32)
                if np.abs(nz >> sh).max() >= 2**31:
                    raise ValueError(f"resource column {r} does not fit int32 even after dropping {sh} common zero bits")
            shift[r] = sh
            req32[r] = (col >> sh).astype(np.int32)
    ns_bits = 32 - 3 - R
    if ns_bits < 1:
        raise ValueError(f"R={R}: presence does not fit the meta word")
    if pods.n and (int(pods.ns_id.max()) >= 1 << ns_bits or int(pods.ns_id.min()) < 0 or int(pods.flags.max()) > 7 or int(pods.present.max()) >> R):
        raise ValueError("namespace id / flags / presence do not fit the packed meta word")
    meta = (pods.ns_id.astype(np.uint32) | (pods.flags.astype(np.uint32) << np.uint32(ns_bits)) |
            (pods.present.astype(np.uint32) << np.uint32(ns_bits + 3))).astype(np.uint32)
    if coded:
        return PackedPodCols(ns_bits, np.ascontiguousarray(pairs, np.int64), np.ascontiguousarray(lab16), None, None, meta, *coded)
    return PackedPodCols(ns_bits, np.ascontiguousarray(pairs, np.int64), np.ascontiguousarray(lab16), np.ascontiguousarray(req32), shift, meta)


@dataclass
class Snapshot:
    """Everything one pass consumes, as the int64/u32 columns of include/kt_b200.h."""
    R: int
    L: int
    LN: int
    running: PodCols
    pending: PodCols
    ns_labels: np.ndarray  # [LN][n_ns] int64
    # throttles
    kind: np.ndarray       # [m] u8
    thr_ns: np.ndarray     # [m] i32
    thr_flags: np.ndarray  # [m] u8
    thr: np.ndarray        # [R][m] i64
    thr_present: np.ndarray  # [m] u32
    thr_cnt: np.ndarray    # [m] i64
    ovr_off: np.ndarray    # [m+1] i32
    ovr_begin: np.ndarray
    ovr_end: np.ndarray
    ovr_flags: np.ndarray
    ovr_thr: np.ndarray    # [R][n_ovr]
    ovr_present: np.ndarray
    ovr_cnt: np.ndarray
    # selector CSR
    term_off: np.ndarray
    term_flags: np.ndarray
    pod_req_off: np.ndarray
    ns_req_off: np.ndarray
    req_key: np.ndarray
    req_op: np.ndarray
    req_val_off: np.ndarray
    req_vals: np.ndarray
    # reservation cache totals (optional)
    reserved: Optional[np.ndarray] = None
    reserved_present: Optional[np.ndarray] = None
    reserved_cnt: Optional[np.ndarray] = None
    # observed status for GIVEN_STATUS (optional dict of arrays named like kt_status_cols)
    status: Optional[dict] = None
    now: int = 0
    meta: dict = field(default_factory=dict)

    @property
    def m(self) -> int:
        return int(self.kind.shape[0])

    @property
    def n_ns(self) -> int:
        return int(self.ns_labels.shape[1])

    def normalize(self) -> "Snapshot":
        m, R = self.m, self.R
        self.running = self.running.normalized(self.L, R)
        self.pending = self.pending.normalized(self.L, R)
        self.ns_labels = _arr(self.ns_labels, np.int64, (self.LN, -1))
        self.kind = _arr(self.kind, np.uint8)
        self.thr_ns = _arr(self.thr_ns, np.int32)
        self.thr_flags = _arr(self.thr_flags, np.uint8)
        self.thr = _arr(self.thr, np.int64, (R, m))
        self.thr_present = _arr(self.thr_present, np.uint32)
        self.thr_cnt = _arr(self.thr_cnt, np.int64)
        self.ovr_off = _arr(self.ovr_off, np.int32)
        n_ovr = int(self.ovr_off[-1])
        self.ovr_begin = _arr(self.ovr_begin, np.int64)
        self.ovr_end = _arr(self.ovr_end, np.int64)
        self.ovr_flags = _arr(self.ovr_flags, np.uint8)
        self.ovr_thr = _arr(self.ovr_thr, np.int64, (R, n_ovr))
        self.ovr_present = _arr(self.ovr_present, np.uint32)
        self.ovr_cnt = _arr(self.ovr_cnt, np.int64)
        self.term_off = _arr(self.term_off, np.int32)
        self.term_flags = _arr(self.term_flags, np.uint8)
        self.pod_req_off = _arr(self.pod_req_off, np.int32)
        self.ns_req_off = _arr(self.ns_req_off, np.int32)
        self.req_key = _arr(self.req_key, np.uint32)
        self.req_op = _arr(self.req_op, np.uint8)
        self.req_val_off = _arr(self.req_val_off, np.int32)
        self.req_vals = _arr(self.req_vals, np.uint32)
        if self.reserved is not None:
            self.reserved = _arr(self.reserved, np.int64, (R, m))
            self.reserved_present = _arr(self.reserved_present, np.uint32)
            self.reserved_cnt = _arr(self.reserved_cnt, np.int64)
        if self.status is not None:
            s = self.status
            self.status = dict(
                calculated=_arr(s["calculated"], np.uint8), calc_thr=_arr(s["calc_thr"], np.int64, (R, m)),
                calc_present=_arr(s["calc_present"], np.uint32), calc_cnt=_arr(s["calc_cnt"], np.int64),
                used=_arr(s["used"], np.int64, (R, m)), used_present=_arr(s["used_present"], np.uint32),
                used_cnt=_arr(s["used_cnt"], np.int64), throttled=_arr(s["throttled"], np.uint32))
        return self

    # ---- ctypes views (the returned structs borrow the numpy memory: keep `self` alive) ----
    def limits(self) -> Limits:
        return Limits(ABI_VERSION, self.R, self.L, self.LN)

    def selector_table(self) -> SelectorTable:
        return SelectorTable(int(self.term_off[-1]), int(self.req_key.shape[0]), int(self.req_vals.shape[0]),
                             ptr(self.term_off), ptr(self.term_flags), ptr(self.pod_req_off), ptr(self.ns_req_off),
                             ptr(self.req_key), ptr(self.req_op), ptr(self.req_val_off), ptr(self.req_vals))

    def throttle_cols(self) -> ThrottleCols:
        return ThrottleCols(ptr(self.kind), ptr(self.thr_ns), ptr(self.thr_flags), ptr(self.thr), ptr(self.thr_present),
                            ptr(self.thr_cnt), ptr(self.ovr_off), int(self.ovr_off[-1]), ptr(self.ovr_begin),
                            ptr(self.ovr_end), ptr(self.ovr_flags), ptr(self.ovr_thr), ptr(self.ovr_present),
                            ptr(self.ovr_cnt))

    def status_cols(self) -> Optional[StatusCols]:
        if self.status is None:
            return None
        s = self.status
        return StatusCols(ptr(s["calculated"]), ptr(s["calc_thr"]), ptr(s["calc_present"]), ptr(s["calc_cnt"]),
                          ptr(s["used"]), ptr(s["used_present"]), ptr(s["used_cnt"]), ptr(s["throttled"]))

    def shard(self, rank: int, world: int) -> "Snapshot":
        """Row shard for rank `rank` of `world`: contiguous row ranges of both pod kinds, throttles replicated
        (SURVEY section 8e)."""
        import copy

        def cut(n):
            lo = (n * rank) // world
            hi = (n * (rank + 1)) // world
            return slice(lo, hi)

        s = copy.copy(self)
        s.running = self.running.rows(cut(self.running.n))
        s.pending = self.pending.rows(cut(self.pending.n))
        s.meta = dict(self.meta, rank=rank, world=world)
        return s


@dataclass
class PassResult:
    """Host copies of every output of one pass (same layout for engine and oracle)."""
    words_per_row: int
    used: np.ndarray          # [R][m] i64
    used_present: np.ndarray  # [m] u32
    used_cnt: np.ndarray      # [m] i64
    throttled: np.ndarray     # [m] u32
    calc_thr: np.ndarray      # [R][m]
    calc_present: np.ndarray
    calc_cnt: np.ndarray
    override_active: np.ndarray
    run_bitmap: np.ndarray    # [N][W] u32
    pend_bitmap: np.ndarray   # [P][W] u32
    codes: np.ndarray         # [P][2W] u32
    admit: np.ndarray         # [P] u8

    @staticmethod
    def alloc(snap: Snapshot, words_per_row: int) -> "PassResult":
        m, R, W = snap.m, snap.R, words_per_row
        N, P = snap.running.n, snap.pending.n
        z = np.zeros
        return PassResult(W, z((R, m), np.int64), z(m, np.uint32), z(m, np.int64), z(m, np.uint32), z((R, m), np.int64),
                          z(m, np.uint32), z(m, np.int64), z(m, np.uint8), z((N, W), np.uint32), z((P, W), np.uint32),
                          z((P, 2 * W), np.uint32), z(P, np.uint8))

    def reconcile_out(self) -> ReconcileOut:
        return ReconcileOut(ptr(self.used), ptr(self.used_present), ptr(self.used_cnt), ptr(self.throttled),
                            ptr(self.calc_thr), ptr(self.calc_present), ptr(self.calc_cnt), ptr(self.override_active))

    def code_matrix(self, m: int) -> np.ndarray:
        """[P][m] uint8 of 2-bit check codes."""
        P = self.codes.shape[0]
        t = np.arange(m)
        return ((self.codes[:, t >> 4] >> (2 * (t & 15)).astype(np.uint32)) & 3).astype(np.uint8).reshape(P, m)

    def match_matrix(self, which: str, m: int) -> np.ndarray:
        bm = self.run_bitmap if which == "running" else self.pend_bitmap
        t = np.arange(m)
        return ((bm[:, t >> 5] >> (t & 31).astype(np.uint32)) & 1).astype(np.uint8)


def default_words_per_row(m: int) -> int:
    """ceil(m/32) rounded up to a multiple of 4 words (16-byte rows) -- must equal kt_match_words()."""
    w = (m + 31) // 32
    return max(4, (w + 3) // 4 * 4)
