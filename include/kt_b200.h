/*
 * kt_b200.h -- C ABI of the H100-native throttle-admission engine.
 *
 * This is the drop-in boundary for the ONE hot path of everpeace/kube-throttler:
 * the per-pod PreFilter/Reserve check (pkg/scheduler_plugin/plugin.go:148-238) plus
 * the controllers' used-resource reconcile (pkg/controllers/throttle_controller.go:84-269,
 * 349-397; clusterthrottle_controller.go:87-298, 378-425) recast as one batched pass.
 *
 * The reference has NO FFI (Makefile:3 sets CGO_ENABLED=0), so every entry point below
 * is new; each one names the reference Go code it replaces.  The Go plugin would bind
 * these through cgo (see INTEGRATION.md for the stub).  Plain pointers and sizes only;
 * no C++/torch types.  All functions return KT_OK (0) or a negative kt_status; the
 * message is available from kt_last_error().  The caller owns every host buffer; the
 * library owns all device memory.  Re-entrant from arbitrary OS threads (cgo calls hop
 * threads): every call takes the context mutex and does cudaSetDevice itself.
 *
 * There is deliberately NO CPU fallback: on a machine without a usable sm_90 GPU
 * kt_create() fails with KT_ERR_CUDA.
 *
 * Data model (all integers; exact decimal arithmetic is the packer's job, see
 * include/kt_host.h and DESIGN.md "Quantity columns"):
 *   - label keys / values are dictionary ids chosen by the packer (uint32 each);
 *     a label slot is int64  (keyId << 32) | valId ;  KT_LABEL_EMPTY marks an unused slot.
 *   - resource.Quantity values are int64 at a per-resource-column scale chosen by the
 *     packer (default 10^-3); presence (Go map "has key") is a bitmask per row.
 *   - matrices are column-major by attribute ("SoA"): labels[L][n], req[R][n], thr[R][m].
 */
#ifndef KT_B200_H_
#define KT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KT_ABI_VERSION 1
#define KT_MAX_RESOURCES 31      /* bit 31 of every resource mask is the pod-count bit */
#define KT_COUNT_BIT 0x80000000u
#define KT_MAX_LABEL_SLOTS 32
#define KT_LABEL_EMPTY ((int64_t)-1)
#define KT_TIME_OPEN_BEGIN INT64_MIN /* override.begin == ""  (temporary_threshold_override.go:33-44) */
#define KT_TIME_OPEN_END INT64_MAX   /* override.end == "" or zero time (:64-69) */

typedef enum kt_status {
  KT_OK = 0,
  KT_ERR_INVALID = -1, /* bad argument / inconsistent columns */
  KT_ERR_CUDA = -2,    /* CUDA runtime error (no device, launch failure, ...) */
  KT_ERR_STATE = -3,   /* call order: e.g. evaluate before upload */
  KT_ERR_LIMIT = -4,   /* exceeds kt_limits */
  KT_ERR_NCCL = -5
} kt_status;

typedef enum kt_pod_kind {
  KT_PODS_RUNNING = 0, /* rows the reconcile sums over (podInformer cache) */
  KT_PODS_PENDING = 1  /* rows PreFilter is asked about (scheduling queue) */
} kt_pod_kind;

/* pod row flags -- pkg/controllers/throttle_controller.go:217-219, pod_util.go:22-28 */
#define KT_POD_SCHEDULER_MATCH 1u /* spec.schedulerName == targetSchedulerName */
#define KT_POD_SCHEDULED 2u       /* spec.nodeName != ""            (isScheduled) */
#define KT_POD_NOT_FINISHED 4u    /* phase not in {Succeeded,Failed} (isNotFinished) */

/* throttle flags */
#define KT_THR_RESPONSIBLE 1u    /* spec.throttlerName == ours (throttle_controller.go:213-215) */
#define KT_THR_SELECTOR_ERROR 2u /* pod selector failed metav1.LabelSelectorAsSelector; never matches
                                    on device, the host turns it into framework.Error (plugin.go:154) */
#define KT_KIND_THROTTLE 0
#define KT_KIND_CLUSTERTHROTTLE 1

/* selector requirement operators (metav1.LabelSelectorRequirement; matchLabels k=v is IN{v}) */
#define KT_OP_IN 0
#define KT_OP_NOTIN 1
#define KT_OP_EXISTS 2
#define KT_OP_DOESNOTEXIST 3

/* term flags */
#define KT_TERM_NS_INVALID 1u /* namespaceSelector conversion error => term is false (Q9,
                                 clusterthrottle_selector.go:63-77) */
#define KT_TERM_POD_INVALID 2u /* podSelector conversion error: the term matches no pod, and for the pods that
                                  reach it (Throttle: its namespace; ClusterThrottle: the namespaces its
                                  namespaceSelector matches) no later term is looked at either -- MatchesToPod
                                  returned the error (throttle_selector.go:30-42, clusterthrottle_selector.go:45-87);
                                  the host turns "reached it" into framework.Error (plugin.go:154-156) */

/* override flags */
#define KT_OVR_PARSE_ERROR 1u /* begin/end failed time.Parse: entry skipped (throttle_types.go:80-84) */

/* CheckThrottleStatus codes, 2 bits each (throttle_types.go:121-126) */
#define KT_CHECK_NOT_THROTTLED 0u /* also "throttle does not affect this pod" (see match bitmap) */
#define KT_CHECK_ACTIVE 1u
#define KT_CHECK_INSUFFICIENT 2u
#define KT_CHECK_POD_REQUESTS_EXCEEDS_THRESHOLD 3u

/* kt_evaluate flags */
#define KT_EVAL_FRESH_STATUS 0u  /* status.{used,throttled,calculatedThreshold} come from this pass's
                                    reconcile (every throttle reconciled at `now`) */
#define KT_EVAL_GIVEN_STATUS 1u  /* PreFilter sees the informer copy of status uploaded with
                                    kt_upload_status (throttle_types.go:128-132) */
#define KT_EVAL_ON_EQUAL 2u      /* isThrottledOnEqual argument of CheckThrottled (PreFilter passes false) */
#define KT_EVAL_SKIP_RECONCILE 4u /* only the pending check (needs GIVEN_STATUS) */
#define KT_EVAL_SKIP_CHECK 8u    /* only the reconcile */

typedef struct kt_ctx kt_ctx;

typedef struct kt_limits {
  int32_t abi_version;     /* KT_ABI_VERSION */
  int32_t n_resources;     /* R: resource columns, 1..KT_MAX_RESOURCES */
  int32_t label_slots;     /* L: label slots per pod row, 1..KT_MAX_LABEL_SLOTS */
  int32_t ns_label_slots;  /* label slots per namespace row */
} kt_limits;

/* Selector table: CSR over throttles -> terms -> requirements -> values.
 * Replaces metav1.LabelSelectorAsSelector + labels.Selector.Matches as called from
 * v1alpha1/throttle_selector.go:30-54 and clusterthrottle_selector.go:30-87. */
typedef struct kt_selector_table {
  int32_t n_terms;
  int32_t n_reqs;
  int32_t n_vals;
  const int32_t* term_off;    /* [m+1]      throttle -> terms (0 terms => matches nothing) */
  const uint8_t* term_flags;  /* [n_terms]  KT_TERM_* */
  const int32_t* pod_req_off; /* [n_terms+1] term -> podSelector requirements (none => Everything) */
  const int32_t* ns_req_off;  /* [n_terms+1] term -> namespaceSelector requirements (ClusterThrottle) */
  const uint32_t* req_key;    /* [n_reqs] keyId */
  const uint8_t* req_op;      /* [n_reqs] KT_OP_* */
  const int32_t* req_val_off; /* [n_reqs+1] */
  const uint32_t* req_vals;   /* [n_vals] valIds */
} kt_selector_table;

/* Throttle / ClusterThrottle spec columns (v1alpha1/throttle_types.go:29-36,
 * temporary_threshold_override.go:25-31). */
typedef struct kt_throttle_cols {
  const uint8_t* kind;            /* [m] KT_KIND_* */
  const int32_t* ns_id;           /* [m] namespace id (Throttle); ignored for ClusterThrottle */
  const uint8_t* flags;           /* [m] KT_THR_* */
  const int64_t* thr;             /* [R][m] spec.threshold.resourceRequests */
  const uint32_t* thr_present;    /* [m]    bit r: threshold has resource r; KT_COUNT_BIT: resourceCounts != nil */
  const int64_t* thr_cnt;         /* [m]    spec.threshold.resourceCounts.pod */
  const int32_t* ovr_off;         /* [m+1]  CSR into temporaryThresholdOverrides (in spec order) */
  int32_t n_ovr;
  const int64_t* ovr_begin;       /* [n_ovr] unix ns, KT_TIME_OPEN_BEGIN if empty */
  const int64_t* ovr_end;         /* [n_ovr] unix ns, KT_TIME_OPEN_END if empty */
  const uint8_t* ovr_flags;       /* [n_ovr] KT_OVR_* */
  const int64_t* ovr_thr;         /* [R][n_ovr] */
  const uint32_t* ovr_present;    /* [n_ovr] as thr_present */
  const int64_t* ovr_cnt;         /* [n_ovr] */
} kt_throttle_cols;

/* Observed status columns for KT_EVAL_GIVEN_STATUS (v1alpha1/throttle_types.go:113-117). */
typedef struct kt_status_cols {
  const uint8_t* calculated;       /* [m] status.calculatedThreshold.calculatedAt != zero time */
  const int64_t* calc_thr;         /* [R][m] status.calculatedThreshold.threshold */
  const uint32_t* calc_present;    /* [m] */
  const int64_t* calc_cnt;         /* [m] */
  const int64_t* used;             /* [R][m] status.used.resourceRequests */
  const uint32_t* used_present;    /* [m] bit r; KT_COUNT_BIT: status.used.resourceCounts != nil */
  const int64_t* used_cnt;         /* [m] */
  const uint32_t* throttled;       /* [m] bit r: status.throttled.resourceRequests[r]==true; KT_COUNT_BIT: .resourceCounts.pod */
} kt_status_cols;

/* Per-throttle results of the reconcile half (what UpdateStatus would write,
 * throttle_controller.go:116-133).  Any pointer may be NULL to skip that column. */
typedef struct kt_reconcile_out {
  int64_t* used;            /* [R][m] */
  uint32_t* used_present;   /* [m] bit r: some counted pod has the key; KT_COUNT_BIT: >=1 pod counted */
  int64_t* used_cnt;        /* [m] */
  uint32_t* throttled;      /* [m] threshold.IsThrottled(used, true): bit r / KT_COUNT_BIT */
  int64_t* calc_thr;        /* [R][m] CalculateThreshold(now).threshold */
  uint32_t* calc_present;   /* [m] */
  int64_t* calc_cnt;        /* [m] */
  uint8_t* override_active; /* [m] 1 if >=1 override active at `now` */
} kt_reconcile_out;

typedef struct kt_timing {
  float reconcile_ms;   /* match-running + segmented sums */
  float allreduce_ms;   /* NCCL all-reduce of the partials (0 when single GPU) */
  float finalize_ms;    /* threshold/override/compare per throttle */
  float check_ms;       /* match-pending + 4-step check */
  float total_ms;       /* first launch -> last kernel end (device clock) */
  int32_t launches;     /* kernels of this library launched by the last kt_evaluate */
} kt_timing;

/* ---- lifecycle ------------------------------------------------------------------ */
/* Replaces the controller construction in NewPlugin (plugin.go:100-113). */
int kt_create(kt_ctx** out, int device, const kt_limits* limits);
void kt_destroy(kt_ctx* ctx);
const char* kt_last_error(const kt_ctx* ctx); /* valid until the next call on ctx */
const char* kt_version(void);
/* Run on a caller-owned CUDA stream (cudaStream_t as void*); NULL restores the private stream.  A switch keeps queued work
 * ordered: everything queued on the old stream before the switch (async uploads, passes) runs before anything the context
 * queues on the new one, and kt_sync, which waits on the new stream, also covers the work queued before the switch.
 * A whole pass queued right behind another whole pass of this library on the same stream (of any context; of the same one
 * unless either pass zero-fills after new rows or tables) starts its match and reconcile tiles while the pass ahead still
 * decides.  Copies, plain kernels and uploads queued between two passes are waited for in full as before.  A caller's own
 * kernel launched with programmatic stream serialization right behind a pass may start before that pass has finished (as
 * before: the pass lets its successor start early); it must wait for it (cudaGridDependencySynchronize) before reading or
 * writing anything the pass touches. */
int kt_set_stream(kt_ctx* ctx, void* cuda_stream);
int kt_sync(kt_ctx* ctx);
/* Record CUDA events around each kernel of kt_evaluate so kt_get_timing reports device times. */
int kt_enable_timing(kt_ctx* ctx, int on);
/* Tracing of the fused pass: with tracing on, every pending-match, reconcile and status tile of the next kt_evaluate records a
 * row of 32 uint64: [0] ticket, [1] SM id, [2] start, [3] end, [4..15] up to 12 stage stamps whose meaning depends on the tile's
 * role -- see the tile functions in csrc/kt_kernels.cuh -- (global timer, ns), [16..27] 12 SM-cycle counts of a shared decide
 * sub-tile's steps, [28] the CTA that ran the tile, [29] that CTA's exit time.  Rows: pending-match tiles, reconcile tiles, then
 * status tiles; roles[] = {match tiles, reconcile tiles, status tiles, CTAs launched}.  The CTAs draw tiles until none is left,
 * then the status tiles and decide work from the same queue; a CTA's last match / reconcile row carries the stamps of its first
 * decide sub-tile and its exit time.  kt_get_trace copies up to cap rows and returns the row count (or a negative kt_status).
 * Diagnostic only; off by default. */
int kt_enable_trace(kt_ctx* ctx, int on);
int64_t kt_get_trace(kt_ctx* ctx, uint64_t* rows /*[cap][32]*/, int64_t cap, uint32_t roles[4]);
/* Pinned host memory for zero-staging H2D/D2H (cudaHostAlloc / cudaFreeHost).  The columns of a packed upload carved out of
 * ONE such block cross the host link as one transfer. */
void* kt_host_alloc(size_t bytes);
/* The same, write-combined (cudaHostAllocWriteCombined): for buffers the CPU only ever WRITES, front to back, and the device
 * reads (upload columns).  The device's reads need no cache snooping on the host, which some platforms reward with a faster
 * host-to-device link; CPU reads of such memory are very slow.  Freed with kt_host_free. */
void* kt_host_alloc_upload(size_t bytes);
void kt_host_free(void* p);

/* ---- snapshot upload (host -> HBM) --------------------------------------------- */
/* Pod rows: replaces podInformer.Lister().Pods(ns).List() + ResourceAmountOfPod per pod
 * (throttle_controller.go:221-246, resource_amount.go:71-76). Replaces the whole kind. */
int kt_upload_pods(kt_ctx* ctx, int kind, int64_t n,
                   const int64_t* labels /*[L][n]*/, const int64_t* req /*[R][n]*/,
                   const uint32_t* present /*[n]*/, const uint32_t* flags /*[n]*/,
                   const int32_t* ns_id /*[n]*/);
/* The same rows in a COMPACT transfer format: the host link, not the device, bounds an end-to-end pass (11.9 MB of int64
 * columns per C2 snapshot), so a packer that knows its dictionaries are small can send 56 instead of 108 bytes per row;
 * a device kernel expands them into the very int64 columns above (the HBM layout and every result are unchanged).
 *   labels32[L][n]  (keyId << val_bits) | valId, 0xFFFFFFFF = empty slot; needs keyId < 2^(32-val_bits), valId < 2^val_bits
 *                   and (keyId, valId) != (all ones)
 *   req32[R][n]     value >> req_shift[r], as int32: exact only if the low req_shift[r] bits of every value are zero and the
 *                   quotient fits (the packer checks; e.g. shift 20 for byte quantities that are multiples of 1Mi)
 *   present[n]      as above
 *   meta[n]         ns_id | flags << 29   (ns_id < 2^29)
 * Returns KT_ERR_INVALID for val_bits outside 1..31 or a shift outside 0..32. */
int kt_upload_pods_compact(kt_ctx* ctx, int kind, int64_t n, int32_t val_bits, const uint32_t* labels32 /*[L][n]*/,
                           const int32_t* req32 /*[R][n]*/, const int32_t* req_shift /*[R]*/,
                           const uint32_t* present /*[n]*/, const uint32_t* meta /*[n]*/);
/* The same rows, smaller still (36 bytes per row at L=8, R=4): labels as 16-bit indices into a dictionary of the distinct
 * (key, value) PAIRS the snapshot uses, presence folded into the meta word.  A packer that interns label pairs (the informer
 * cache of a real cluster has a few thousand distinct pairs) sends 2 bytes per label slot.
 *   pairs[n_pairs]   keyId << 32 | valId, n_pairs <= 65535
 *   labels16[L][n]   index into pairs, 0xFFFF = empty slot
 *   req32, req_shift as in kt_upload_pods_compact
 *   meta[n]          ns_id | flags << ns_bits | present << (ns_bits + 3);  ns_bits + 3 + R <= 32, ns_id < 2^ns_bits
 * Expanded on the device into the int64 columns of kt_upload_pods: HBM layout and results unchanged. */
typedef struct {
  int32_t n_pairs;
  int32_t ns_bits;
  const int64_t* pairs;      /* [n_pairs] */
  const uint16_t* labels16;  /* [L][n] */
  const int32_t* req32;      /* [R][n] */
  const int32_t* req_shift;  /* [R] */
  const uint32_t* meta;      /* [n] */
  /* Optional, instead of req32 / req_shift (both may then be NULL): dictionary-coded request columns.  Pods come from a few
   * templates, so a column of 10^5 requests holds a few dozen distinct values: 1 byte per value instead of 4.
   *   req_dict[...]          the distinct values, column after column (exact int64, the engine's own unit)
   *   req_dict_off[R+1]      column r's values are req_dict[req_dict_off[r] .. req_dict_off[r+1])
   *   req_code_bytes[R]      1 or 2: width of column r's codes (at most 256 / 65536 distinct values)
   *   req_codes              the code columns one after another, column r = n little-endian codes of req_code_bytes[r] bytes,
   *                          each column padded to a multiple of 4 bytes */
  const int64_t* req_dict;
  const int32_t* req_dict_off;
  const uint8_t* req_code_bytes;
  const uint8_t* req_codes;
} kt_packed_pods;
int kt_upload_pods_packed(kt_ctx* ctx, int kind, int64_t n, const kt_packed_pods* rows);
/* With async uploads on, kt_upload_pods / kt_upload_pods_compact return as soon as the copies are QUEUED: the caller must
 * keep the host buffers alive and unchanged until kt_sync or any kt_get_* has returned.  Saves one stream
 * synchronisation per upload on the latency-sensitive end-to-end path.  Off by default. */
int kt_set_async_uploads(kt_ctx* ctx, int on);
/* Row-level delta (pod informer Add/Update/Delete, throttle_controller.go:431-532):
 * columns are compact [L][k] / [R][k] / [k]; rows[i] < current n.  A deleted pod is a row
 * with flags == 0 (never counted) and all label slots empty. */
int kt_update_pod_rows(kt_ctx* ctx, int kind, int64_t k, const int64_t* rows,
                       const int64_t* labels, const int64_t* req, const uint32_t* present,
                       const uint32_t* flags, const int32_t* ns_id);
/* Namespace rows (namespaceInformer, clusterthrottle_controller.go:224-247). */
int kt_upload_namespaces(kt_ctx* ctx, int32_t n_ns, const int64_t* labels /*[LN][n_ns]*/);
/* Row deltas of the namespace rows, for a caller that keeps the snapshot resident: a Namespace created, relabelled or deleted
 * changes its own row, and only the namespace masks and word lists of the tables depend on it (the pod-label tables do not).
 * Afterwards every call answers exactly as after a kt_upload_namespaces(ctx, n_ns, all_rows), where all_rows holds the previous
 * rows with the k listed ones replaced by labels[.][i] ([LN][k]); rows between the previous count and n_ns that are not listed
 * are label-less.  n_ns never shrinks; idx entries distinct and in [0, n_ns); k >= 0; no null idx, and no null labels when
 * LN > 0, with k > 0 (KT_ERR_INVALID otherwise); k = 0 with an unchanged n_ns is a no-op.  Before kt_upload_throttles only the
 * stored rows change, as with the full call.  Otherwise the listed rows (and the rows n_ns grew by) are evaluated against every
 * term on the device and the word lists are rebuilt there; no table compile, no re-upload of the pod-label tables, one staged
 * copy and one synchronisation.  The state flags move as the full call moves them: kt_evaluate is needed again before the
 * getters that read a pass.  Multi-GPU: the tables are replicated, so the call is local -- every rank applies the same updates. */
int kt_update_namespace_rows(kt_ctx* ctx, int32_t n_ns, int64_t k, const int32_t* idx, const int64_t* labels /*[LN][k]*/);
/* Throttle + ClusterThrottle specs; compiles the selectors into the bit-sliced match tables. */
int kt_upload_throttles(kt_ctx* ctx, int32_t m, const kt_throttle_cols* cols,
                        const kt_selector_table* sel);
/* Informer copy of .status for KT_EVAL_GIVEN_STATUS. */
int kt_upload_status(kt_ctx* ctx, const kt_status_cols* st);
/* reservedResourceAmounts.reservedResourceAmount(nn) for every throttle
 * (reserved_resource_amounts.go:113-126): sums, presence, pod count (KT_COUNT_BIT set
 * in present[t] iff >=1 pod is reserved on t).  NULL pointers mean "nothing reserved". */
int kt_set_reserved(kt_ctx* ctx, const int64_t* reserved /*[R][m]*/,
                    const uint32_t* present /*[m]*/, const int64_t* cnt /*[m]*/);
/* Column deltas of the throttle-side state, for a caller that keeps the snapshot resident: a status echoed back by the informer,
 * or one Reserve / Unreserve, changes a few columns, and the selector tables do not depend on either.
 * kt_update_status_rows: the observed status of k listed throttle columns, shaped as kt_get_reconcile_rows fills them ([R][k] /
 * [k]).  Afterwards every call answers exactly as after a kt_upload_status whose columns equal the previous ones with these k
 * replaced.  KT_ERR_STATE before kt_upload_status (a partial status over no status has no meaning).
 * kt_update_reserved_rows: reserved[R][k], present[k], cnt[k] of k listed columns; as kt_set_reserved with those k replaced.
 * Before any kt_set_reserved (or after kt_set_reserved(NULL, ...)) the other columns are "nothing reserved".
 * Both: idx entries distinct and in [0, M), k >= 0, no null column when k > 0 (KT_ERR_INVALID otherwise); KT_ERR_STATE before
 * kt_upload_throttles; k = 0 is a no-op.  One staged copy of the k columns, one scatter launch, one synchronisation (the caller
 * may reuse its buffers on return); no table compile, no re-upload of the other columns.  The state flags move as the full
 * calls move them.  Multi-GPU: the throttle columns are replicated, so the call is local, not collective -- every rank must
 * apply the same updates. */
int kt_update_status_rows(kt_ctx* ctx, int64_t k, const int32_t* idx, const kt_status_cols* st);
int kt_update_reserved_rows(kt_ctx* ctx, int64_t k, const int32_t* idx, const int64_t* reserved /*[R][k]*/,
                            const uint32_t* present /*[k]*/, const int64_t* cnt /*[k]*/);
/* Column deltas of the spec's thresholds: an edit of spec.threshold or spec.temporaryThresholdOverrides changes a few columns, and
 * no compiled table reads either.  cols is shaped for the k listed columns: thr[R][k], thr_present[k], thr_cnt[k]; ovr_off[k+1]
 * with n_ovr == ovr_off[k], and that many ovr_begin / ovr_end / ovr_flags / ovr_present / ovr_cnt entries and ovr_thr[R][n_ovr],
 * in spec order.  kind, ns_id and flags feed the tables and must be NULL.  Afterwards every call answers exactly as after a
 * kt_upload_throttles whose spec columns are the previous ones with these k replaced, followed by re-uploading the status and
 * the reservations held before the call (when they were held): both are kept, and so are the pod rows' table offsets.  The
 * state flags move as kt_upload_throttles moves them (a pass is needed again before the getters that read one).
 * KT_ERR_INVALID: k < 0; a null idx or column with k > 0; a non-null kind, ns_id or flags; an index out of [0, M) or listed
 * twice; an ovr_off that does not span [0, n_ovr] monotonically.  KT_ERR_STATE before kt_upload_throttles; k = 0 is a no-op.
 * One staged copy and one synchronisation (the caller may reuse its buffers on return); no table compile and no re-upload of
 * the other columns.  When no listed column changes its number of overrides the columns are scattered in place and the copy
 * carries O(k) data; otherwise every override entry moves (n_ovr and the stride of ovr_thr change): the new offsets, derived on
 * the host, travel with the copy (O(M) bytes) and the override columns are rebuilt on the device.  Multi-GPU: the call is
 * local, not collective -- every rank must apply the same updates. */
int kt_update_threshold_rows(kt_ctx* ctx, int64_t k, const int32_t* idx, const kt_throttle_cols* cols);
/* Column deltas of the compiled side of the spec: a deletion (zero terms, flags 0), a podSelector / namespaceSelector edit or a
 * throttlerName change (KT_THR_RESPONSIBLE) of a few columns, with M and every column's position kept.  cols carries kind[k],
 * ns_id[k] and flags[k] of the k listed columns; its threshold and override pointers belong to kt_update_threshold_rows and must
 * be NULL.  sel is a CSR over the k listed columns, in idx order, shaped as for kt_upload_throttles.  Afterwards every call
 * answers exactly as after a kt_upload_throttles whose spec is the previous one with the listed columns' kind, ns_id, flags and
 * selector terms replaced (threshold and override columns kept), followed by re-uploading the status and the reservations held
 * before the call (when they were held).  The state flags move as kt_upload_throttles moves them (a pass is needed again before
 * the getters that read one, and the next pass zero-fills its bitmap rows).  *recompiled (may be NULL) is 1 when the call
 * compiled the tables again, 0 when it patched them in place.
 * KT_ERR_INVALID: k < 0; a null idx, kind, ns_id, flags, sel or term_off with k > 0; a non-null threshold or override pointer;
 * an index out of [0, M) or listed twice; a malformed CSR.  KT_ERR_STATE before kt_upload_throttles; k = 0 is a no-op.
 * In place when every listed column fits the resident tables -- its podSelector keys and (key, value) pairs have table rows,
 * its term count fits TPpad, its need fits the counter planes, a Throttle's namespace is below the resident namespace count --:
 * the listed columns' table and need bits are recompiled on the host (the code compile_tables uses for one column) and only
 * their 32-throttle word slices cross, in one staged copy; the namespace masks of those words are evaluated again for every
 * namespace on the device and the word lists rebuilt; the pod rows keep their table offsets.  Otherwise the tables are
 * compiled again from the patched spec, as kt_upload_namespaces does.  One synchronisation; the caller may reuse its buffers on
 * return.  Multi-GPU: the call is local, not collective -- every rank must apply the same updates. */
int kt_update_selector_rows(kt_ctx* ctx, int64_t k, const int32_t* idx, const kt_throttle_cols* cols,
                            const kt_selector_table* sel, int32_t* recompiled);
/* k new throttle columns appended at [M, M+k): a Throttle or ClusterThrottle creation without recompiling the selector tables.
 * cols and sel are shaped exactly as for kt_upload_throttles(ctx, k, cols, sel): kind, ns_id, flags, thresholds, the override
 * CSR and the selector CSR of the k new columns.  Afterwards every call answers exactly as after a kt_upload_throttles of the
 * previous spec with these k columns appended, followed by re-uploading the status and the reservations held before the call,
 * each widened by k columns of zeros (no calculatedAt, nothing used, nothing reserved); status or reservations not held before
 * the call are still not held.  The state flags move as kt_update_selector_rows moves them; *recompiled (may be NULL) is as
 * there.
 * KT_ERR_INVALID: k < 0; a null column with k > 0; a malformed CSR or ovr_off.  KT_ERR_STATE before kt_upload_throttles;
 * k = 0 is a no-op.
 * In place when every new column fits the resident tables (the test of kt_update_selector_rows): the new columns are compiled on
 * the host into the partly filled last 32-throttle word and the words appended after it, and only those word slices cross, in
 * one staged copy; the resident per-throttle columns are widened on the device (the override columns rebuilt), the namespace
 * masks restrided when the word count grows and evaluated for the touched words, the word lists rebuilt; the pod rows keep their
 * table offsets.  Otherwise the tables are compiled again from the grown spec.  One synchronisation; the caller may reuse its
 * buffers on return.  Multi-GPU: the call is local, not collective -- every rank must apply the same appends. */
int kt_append_throttle_rows(kt_ctx* ctx, int64_t k, const kt_throttle_cols* cols, const kt_selector_table* sel,
                            int32_t* recompiled);
/* The throttle columns laid out again: column j of the new layout is previous column src[j], for j in [0, m).  Afterwards every
 * call answers exactly as after a kt_upload_throttles(ctx, m, spec') whose column j is previous column src[j] -- kind, ns_id,
 * flags, selector terms, threshold and overrides --, followed by re-uploading the status and the reservations held before the
 * call, gathered the same way.  src[j] == -1 makes an empty column: kind ClusterThrottle, ns_id -1, flags 0, no terms, no
 * threshold, no overrides, zero status and nothing reserved; it matches nothing and adds no word to any namespace's list.
 * Previous columns src does not name are dropped; m may be smaller than, equal to or larger than M.  Status or reservations not
 * held before the call are still not held.  The state flags move as kt_update_selector_rows moves them (a pass is needed again
 * before the getters that read one); kt_match_words may change.
 * KT_ERR_INVALID: m < 0; a null src with m > 0; an entry outside [-1, M); a non-negative entry listed twice.  KT_ERR_STATE
 * before kt_upload_throttles.
 * Always in place, never a table compile: every per-column thing the device holds is column-local, so the move is a gather.  The
 * table-row dictionary, TPpad, the counter planes and the namespace count are kept, and the pod rows keep their table offsets.
 * The table, need and namespace-mask bits are gathered by column on the device, the per-throttle columns restrided and the
 * override columns rebuilt through the column map, the word lists rebuilt.  One staged copy (src and the new override offsets)
 * and one synchronisation; the caller may reuse src on return.  Multi-GPU: the call is local, not collective -- every rank must
 * apply the same move. */
int kt_move_throttle_columns(kt_ctx* ctx, int32_t m, const int32_t* src /*[m]*/);

/* ---- the pass ------------------------------------------------------------------- */
/* One batched pass: reconcile every throttle (throttle_controller.go:84-133) and check
 * every pending pod against every throttle (CheckThrottled, :349-397).  Asynchronous on
 * the context stream unless a getter is called; kt_sync() waits.
 * Value domain: quantities are signed.  Every request, threshold, used and reserved value,
 * and for every resource column the sum of |v| over the running and pending requests, the
 * reservations and the status, must stay below 2^62 (the host layer, kt_host.cc, checks
 * the pod columns' sums before it uploads).  Sums are then exact in int64. */
int kt_evaluate(kt_ctx* ctx, int64_t now_unix_ns, uint32_t flags);

/* ---- queue-ordered greedy admission ------------------------------------------------ */
/* The scheduler admits one pod per cycle: PreFilter, then -- on Success -- Reserve, so that every admitted pod raises the
 * reservations the next one is checked against (plugin.go:148-238, reserved_resource_amounts.go:66-136).  kt_admit_queue runs
 * that sequence for the pending rows [first, first + count) taken IN ROW ORDER as one sorted queue, entirely on the device:
 * per-throttle prefix sums over the requests of the admitted pods before each pod, iterated to the fixpoint (see
 * csrc/kt_admit.cuh; a handful of rounds, each costing the host one 8-byte read).  PreFilter's view applies: the observed status
 * (kt_upload_status) + the uploaded reservations (kt_set_reserved), isThrottledOnEqual from `flags` (KT_EVAL_ON_EQUAL or 0).
 * Afterwards admit[row] says which rows were admitted and codes[row] holds the 2-bit codes each REJECTED row saw at its turn
 * (kt_get_check / kt_get_check_rows); the pending match rows (kt_get_match_rows) name the throttles an admitted pod must be
 * reserved on by the caller's reservation cache; the rows outside the queue keep the codes and admit bits of a
 * KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE pass.  Requests may be negative; the value domain is kt_evaluate's. */
int kt_admit_queue(kt_ctx* ctx, int64_t first, int64_t count, uint32_t flags, int32_t* rounds, int64_t* admitted);

/* ---- one end-to-end step in one call --------------------------------------------- */
/* A caller that hands over a fresh snapshot every pass (host buffers in, results out) pays for every boundary crossing and
 * every stream synchronisation.  kt_step_submit queues ONE whole step on the context's stream -- the packed pod rows of
 * either kind (NULL: keep the resident rows), the pass, the results into one library-owned pinned block: per-throttle status
 * columns, admit bits, the non-zero check-code words (needs kt_set_sparse_check) -- and returns; kt_step_wait blocks until
 * the block has landed and points `out` into it (valid until the next kt_step_submit on this context).  One synchronisation
 * per step; two contexts submitting alternately overlap one step's upload with the other's pass and download.
 * The host buffers of a submitted step must stay untouched until its kt_step_wait has returned. */
typedef struct kt_step_result {
  int64_t n_pending;        /* rows of admit[] */
  int64_t n_sparse;         /* non-zero code words of the pass; entries holds min(n_sparse, cap of kt_set_sparse_check) of them */
  const uint8_t* admit;     /* [n_pending] */
  const uint32_t* entries;  /* [..][3] {pending row, code word index, codes} as kt_get_check_sparse */
  kt_reconcile_out status;  /* pointers into the block, shaped as kt_get_reconcile fills them */
} kt_step_result;
int kt_step_submit(kt_ctx* ctx, int64_t n_running, const kt_packed_pods* running, int64_t n_pending, const kt_packed_pods* pending,
                   int64_t now_unix_ns, uint32_t flags);
int kt_step_wait(kt_ctx* ctx, kt_step_result* out);

/* ---- results (HBM -> host) ------------------------------------------------------ */
int kt_get_reconcile(kt_ctx* ctx, const kt_reconcile_out* out);
/* words_per_row = kt_match_words(ctx); bitmap rows are pod-major: bit (t&31) of
 * words[p*words_per_row + (t>>5)] == throttle t affects pod p.
 * RUNNING: affectedPods relation (shouldCountIn && selector match, finished pods included);
 * PENDING: affectedThrottles relation (responsible && namespace && selector match). */
int32_t kt_match_words(const kt_ctx* ctx);
int kt_get_match_bitmap(kt_ctx* ctx, int kind, uint32_t* words /*[n][words_per_row]*/);
/* The same for k selected rows only (gathered on the device): words[i] = bitmap row rows[i].  This is how the
 * host finds which reserved pods a reconcile has observed (unreserveAffectedPods, throttle_controller.go:135-155)
 * without downloading the whole relation. */
int kt_get_match_rows(kt_ctx* ctx, int kind, int64_t k, const int64_t* rows, uint32_t* words /*[k][words_per_row]*/);
/* The same relation from the throttles' side (affectedPods, throttle_controller.go:221-246, clusterthrottle_controller.go:224-270),
 * for k listed throttles, transposed on the device from what the last pass (or kt_admit_queue) left, exactly as
 * kt_get_match_bitmap / kt_get_check would deliver it.  For throttle idx[j], the rows whose bit is set, ascending, are
 * rows[off[j] .. off[j+1]).
 *   RUNNING: the affectedPods relation as kt_get_match_bitmap defines it (finished pods included: the caller splits them by
 *            its flags).
 *   PENDING: the pods the throttle affects; codes[i] = the 2-bit code of (rows[i], idx[j]) that kt_get_check would show.
 * idx entries must lie in [0, M) (KT_ERR_INVALID otherwise); duplicates each get their own segment; k = 0 is valid.  off[0..k]
 * is always written; rows / codes only when off[k] <= cap -- otherwise the caller retries with a larger cap.  codes may be NULL
 * and must be NULL for RUNNING.  Only the words of the listed throttles are read (count, offsets, scan, fill: four launches,
 * one read of off[], one copy of the rows).  Multi-GPU: each rank answers for its own rows. */
int kt_get_match_columns(kt_ctx* ctx, int kind, int64_t k, const int32_t* idx, int64_t* off /*[k+1]*/, int64_t* rows /*[cap]*/,
                         uint8_t* codes /*[cap] or NULL*/, int64_t cap);
/* The scheduling queue summarised per throttle, from what the last pass that ran the check (a kt_evaluate without
 * KT_EVAL_SKIP_CHECK, or kt_admit_queue) wrote for the pending rows [first, first + count), in caller rows: the codes are exactly
 * those kt_get_check delivers for these rows.  row_class[i] (NULL: every row is class 1) applies to row first + i:
 *   0  the row is skipped;
 *   1  the row is counted;
 *   2  the row is counted in status_cnt and held, never in sole_cnt (a pod whose PreFilter fails has no "only blocker").
 * Every output pointer may be NULL.  Sums are exact in int64 under kt_evaluate's value domain; requests may be negative.
 * Only rejected rows (admit byte 0) are read beyond their admit byte.  The call writes nothing another call reads (every getter
 * answers as before it).  count = 0 is valid and yields zeros.  KT_ERR_INVALID for a range outside [0, n_pending) or count < 0;
 * KT_ERR_STATE before a pass has written the pending codes of the current rows and throttle columns, and with a communicator
 * (single GPU only). */
typedef struct kt_check_summary {
  int64_t* status_cnt;    /* [3][m] rows whose code for t is ACTIVE, INSUFFICIENT, POD_REQUESTS_EXCEEDS_THRESHOLD (in that order) */
  int64_t* sole_cnt;      /* [m]    rows of class 1 whose ONLY non-zero code, over all throttles of both kinds, is t's */
  int64_t* held;          /* [R][m] sum of req[r] over the rows with a non-zero code for t */
  uint32_t* held_present; /* [m]    bit r: some such row has resource r present; KT_COUNT_BIT: at least one such row */
} kt_check_summary;
int kt_get_check_summary(kt_ctx* ctx, int64_t first, int64_t count, const uint8_t* row_class /*[count] or NULL*/,
                         const kt_check_summary* out);
/* reconcile(key) for k listed throttles (throttle_controller.go:84-211, clusterthrottle_controller.go:87-214), evaluated at
 * `now` on the running rows as they are now -- uploaded or delta-updated, whether or not a pass has run since.  For entry j:
 *   - out: what a KT_EVAL_FRESH_STATUS pass would report for column idx[j] (used, presence, pod count, throttled with
 *     onEqual = true, CalculateThreshold(now), override_active), shaped [R][k] / [k] as kt_get_reconcile_rows fills them
 *     (any pointer may be NULL);
 *   - rows[off[j] .. off[j+1]): the rows the throttle matches, ascending -- the RUNNING relation of kt_get_match_columns
 *     (counted pods, finished ones included).
 * Arguments as kt_get_match_columns: idx in [0, M) (KT_ERR_INVALID otherwise), duplicates each get their own entry, k = 0 is
 * valid, off[0..k] is always written and rows only when off[k] <= cap.  Only the listed throttles' words are evaluated, and
 * only for the rows whose namespace they can reach; the call writes nothing another call reads (every getter answers as
 * before it).  KT_ERR_STATE before kt_upload_throttles, and with a communicator (single GPU only). */
int kt_reconcile_throttles(kt_ctx* ctx, int64_t now_unix_ns, int64_t k, const int32_t* idx, const kt_reconcile_out* out,
                           int64_t* off /*[k+1]*/, int64_t* rows /*[cap] or NULL*/, int64_t cap);
/* codes: 2 bits per (pending pod, throttle), pod-major, 16 codes per uint32:
 *   code(p,t) = (codes[p*2*words_per_row + (t>>4)] >> (2*(t&15))) & 3
 * admit[p] = 1 iff every affected throttle is KT_CHECK_NOT_THROTTLED (plugin.go:177-180).
 * Either pointer may be NULL. */
int kt_get_check(kt_ctx* ctx, uint32_t* codes /*[p][2*words_per_row]*/, uint8_t* admit /*[p]*/);
/* The same result without the zeros.  A PreFilter caller needs the admit bit of every pod and, for the rejected ones, which
 * throttles said what (plugin.go:182-213): at C2 that is ~10^4 non-zero code words out of 6.4*10^5.
 * kt_set_sparse_check(cap_entries > 0) makes every later pass ALSO append each non-zero code word to a device list of at most
 * cap_entries entries (0 switches it off again; the dense rows are always written).  kt_get_check_sparse copies admit[p]
 * and the entries {pending row, word index j in [0, 2*words_per_row), codes word}: the word is what kt_get_check would have
 * delivered at codes[row*2*words_per_row + j].  Entries are unordered.  *count is the number of non-zero words of the pass;
 * when it exceeds cap (or the device capacity) only the first min(cap, cap_entries) were delivered and the caller should
 * read the dense rows instead. */
int kt_set_sparse_check(kt_ctx* ctx, int64_t cap_entries);
int kt_get_check_sparse(kt_ctx* ctx, uint8_t* admit /*[p]*/, uint32_t* entries /*[cap][3]*/, int64_t cap, int64_t* count);
/* The check result of k listed pending rows only (a PreFilter caller that wants the reasons of ONE rejected pod after a pass
 * over the whole queue): codes[i][2*words_per_row] and admit[i] of rows[i].  Either output may be NULL. */
int kt_get_check_rows(kt_ctx* ctx, int64_t k, const int64_t* rows, uint32_t* codes /*[k][2*words_per_row]*/, uint8_t* admit /*[k]*/);
/* PreFilter for k listed pending rows (plugin.go:148-215), evaluated on the rows, tables, observed status and reservations as
 * they are now -- uploaded or delta-updated, whether or not a pass has run since -- without a pass over the pending table.
 * For entry i the outputs are bit for bit what kt_evaluate(ctx, 0, KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE | flags)
 * followed by kt_get_match_rows(KT_PODS_PENDING) (words) and kt_get_check_rows (codes, admit) would deliver for rows[i].
 * flags is 0 or KT_EVAL_ON_EQUAL (KT_ERR_INVALID otherwise); a given-status check reads no clock.  rows are caller rows in
 * [0, n) (KT_ERR_INVALID otherwise), duplicates are allowed, k = 0 is valid; any output may be NULL.  Only the listed rows are
 * evaluated, each over the words of its own namespace; the call writes nothing another call reads (every getter answers as
 * before it, and one that fails before kt_evaluate still fails).  KT_ERR_STATE before kt_upload_throttles, before
 * kt_upload_status, and with a communicator (single GPU only). */
int kt_check_pending_rows(kt_ctx* ctx, uint32_t flags, int64_t k, const int64_t* rows, uint32_t* words /*[k][words_per_row] or NULL*/,
                          uint32_t* codes /*[k][2*words_per_row] or NULL*/, uint8_t* admit /*[k] or NULL*/);
/* affectedThrottles of k pods that live only in this call (throttle_controller.go:248-269, clusterthrottle_controller.go:272-298):
 * the pod versions an informer event carries, matched against the throttle tables as they are now.  words[i] is bit for bit what
 * kt_get_match_rows(KT_PODS_PENDING) would return for a pending row holding labels[.][i] and ns_id[i] after a
 * KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE pass: responsible && namespace && selector match, a KT_TERM_POD_INVALID term
 * switching the later terms off as in the pass.  Label slots are int64 codes as in kt_upload_pods / kt_update_pod_rows; a
 * namespace id the tables do not cover (negative, or at or above both n_ns and every Throttle's namespace id + 1) gives an
 * all-zero row, as in the pass.  Needs kt_upload_throttles (and the namespaces) only: no pods, status
 * or reservations.  It reads no resident pod row and writes nothing another call reads (every getter answers as before it, and
 * the context's evaluated state is unchanged).  One copy in, one launch, one copy out, one synchronisation.  k = 0 is valid;
 * KT_ERR_INVALID for k < 0 or a null pointer with k > 0; KT_ERR_STATE before kt_upload_throttles and with a communicator
 * (single GPU only). */
int kt_match_pods(kt_ctx* ctx, int64_t k, const int64_t* labels /*[L][k]*/, const int32_t* ns_id /*[k]*/,
                  uint32_t* words /*[k][words_per_row]*/);
/* PreFilter of k pods that live only in this call (plugin.go:148-215): the manifest of a PreFilter, Reserve or Unreserve, checked
 * against the tables, observed status and reservations as they are now, with no pass over the pending table.  Entry i is bit
 * for bit what kt_evaluate(ctx, 0, KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE | flags) followed by
 * kt_get_match_rows(KT_PODS_PENDING) (words) and kt_get_check_rows (codes, admit) would deliver for a pending row holding
 * labels[.][i], req[.][i], present[i] and ns_id[i] -- columns laid out as in kt_upload_pods / kt_update_pod_rows: a
 * KT_TERM_POD_INVALID term switches the later terms off, only the non-zero present requests are compared (Q5), requests may be
 * negative, and a namespace id the tables do not cover gives an all-zero row with admit = 1.  The pass reads no flags of a
 * pending row (they matter to the running rows only), so the call takes none.  flags is 0 or KT_EVAL_ON_EQUAL
 * (KT_ERR_INVALID otherwise); k = 0 is valid; KT_ERR_INVALID for k < 0 or a null input column with k > 0; any output may be NULL.
 * Needs kt_upload_throttles and kt_upload_status (KT_ERR_STATE before either) and no pod rows at all.  It reads no resident pod
 * row and writes nothing another call reads (every getter answers as before it, and one that fails before kt_evaluate still
 * fails).  Value domain: kt_evaluate's.  One staged copy in, two launches (pre-records, check), one copy out, one
 * synchronisation.  KT_ERR_STATE with a communicator (single GPU only). */
int kt_check_pods(kt_ctx* ctx, uint32_t flags, int64_t k, const int64_t* labels /*[L][k]*/, const int64_t* req /*[R][k]*/,
                  const uint32_t* present /*[k]*/, const int32_t* ns_id /*[k]*/, uint32_t* words /*[k][words_per_row] or NULL*/,
                  uint32_t* codes /*[k][2*words_per_row] or NULL*/, uint8_t* admit /*[k] or NULL*/);

/* Device-side status diff (replaces the apiequality.Semantic.DeepEqual(thr.Status, *newStatus) of every reconcile,
 * throttle_controller.go:157 / clusterthrottle_controller.go:160): when an observed status is uploaded (kt_upload_status) every
 * reconciling pass compares what it computed -- used (values and presence), throttled, the calculated threshold (a status whose
 * calculatedAt is unset always differs) -- with it, per responsible throttle, inside the pass.  kt_get_changed delivers how many
 * throttles differ, up to cap of their indices (unordered) and, when flags != NULL, one byte per throttle; kt_get_reconcile_rows
 * the status columns of k listed throttles only, shaped [R][k] / [k] -- so that the download after a reconcile is proportional
 * to what changed, not to M.  Messages and calculatedAt stay on the host (they depend on the spec and the clock alone). */
int kt_get_changed(kt_ctx* ctx, int32_t* idx /*[cap]*/, int64_t cap, int64_t* count, uint8_t* flags /*[m] or NULL*/);
int kt_get_reconcile_rows(kt_ctx* ctx, int64_t k, const int32_t* idx, const kt_reconcile_out* out /* columns shaped for k throttles */);
int kt_get_timing(kt_ctx* ctx, kt_timing* out);

/* ---- host-only introspection (no device needed) -------------------------------- */
/* Compiles a selector table exactly as kt_upload_throttles does and hands the bit-sliced match tables back, so that the
 * table compiler can be checked on a machine without a GPU (tests/test_tables_cpu.py evaluates them with numpy).
 * Every output pointer may be NULL; sizes come back in dims[12] = {M, W, Wp, TPpad, B, rows, NS, n_keydir, n_valrow,
 * n_nsw, max_ns_words, hash_slots}.  First call with NULL arrays to size them.  The tables are never evaluated here. */
int kt_debug_compile_tables(const kt_limits* limits, int32_t m, const kt_throttle_cols* cols, const kt_selector_table* sel,
                            int32_t n_ns, const int64_t* ns_labels, int32_t dims[12], uint32_t* table, uint32_t* need,
                            uint32_t* nsmask, int32_t* nsw_off, int32_t* nsw_idx, uint32_t* keydir, uint32_t* valrow, uint32_t* hash);

/* ---- test seam of the fused pass (diagnostic only, like tracing) ------------------ */
/* At launch the fused pass picks, from the shape, a residency (the build compiled for 512 or for 768 resident threads per SM)
 * and a decide mode (four-lane sub-tiles or lane-per-pod tiles), and sizes its grid to what the device holds.  Most shapes
 * reach only a few of these combinations, so a test forces them here to compare every build and mode with a reference at
 * small sizes.  This is a test seam, not a tuning option: the automatic choices are the product's, and no product path sets
 * a plan.
 *   threads_per_sm  in: 0 automatic, 512 or 768                     out: the build that ran
 *   decide          in: 0 automatic, 1 quad sub-tiles, 2 per-pod    out: the mode that ran
 *   max_ctas        in: 0 what the device holds; else a cap on the grid (clamped to 1..capacity of the chosen build), applied
 *                   before the automatic choices: they see the capped grid.  A grid larger than the device holds is not offered.
 *   grid, capacity  out: CTAs launched; CTAs the chosen build fits on the device at once (occupancy x SMs)
 *   tile, tpc, b, rt  out: the kernel variant of the pass (rt 0: the general family)
 *   n_chk, n_rec, n_fin, n_sub  out: match tiles, reconcile tiles, status tiles, decide pieces
 * kt_debug_set_pass_plan(NULL) or an all-zero plan restores the automatic choices (the default); KT_ERR_INVALID for other
 * values.  While a plan is set, a single-GPU fused pass also checks its in-kernel waits: one that timed out makes kt_sync and
 * the getters return KT_ERR_STATE; and it first fills every output it writes (bitmaps, codes, admit bits, status columns) with
 * a poison pattern, so that work it skipped cannot hide behind the previous pass's results.  kt_debug_get_pass_plan reports what the last fused pass of the context ran
 * (KT_ERR_STATE before the first one). */
typedef struct kt_pass_plan {
  int32_t threads_per_sm;
  int32_t decide;
  uint32_t max_ctas;
  uint32_t grid;
  uint32_t capacity;
  int32_t tile, tpc, b, rt;
  uint32_t n_chk, n_rec, n_fin, n_sub;
} kt_pass_plan;
#define KT_PLAN_DECIDE_QUAD 1
#define KT_PLAN_DECIDE_PER_POD 2
int kt_debug_set_pass_plan(kt_ctx* ctx, const kt_pass_plan* plan);
int kt_debug_get_pass_plan(kt_ctx* ctx, kt_pass_plan* last);
/* The namespace side of the resident tables, as the passes read it (test seam: after kt_update_namespace_rows it must equal what
 * kt_debug_compile_tables gives for the same rows).  dims[5] = {NS, n_nsw, max_ns_words, W, TPpad}; nsmask [NS][W][TPpad], nsw_off [NS+1],
 * nsw_idx [n_nsw] may each be NULL (first call with NULL arrays to size them).  KT_ERR_STATE before kt_upload_throttles. */
int kt_debug_get_ns_tables(kt_ctx* ctx, int32_t dims[5], uint32_t* nsmask, int32_t* nsw_off, int32_t* nsw_idx);

/* ---- row order of the pod tables ------------------------------------------------------ */
/* A pass costs far more when the 32 rows of a warp belong to many namespaces than when they share one.  So the engine may STORE
 * the rows of a kind in another order than the caller uploaded them: sorted by namespace id (stable: rows of one namespace keep
 * the caller's order; rows whose ns lies outside [0, n_ns) form one group at the end).  Every row number that crosses this ABI,
 * in either direction, stays the caller's, and no result changes; only where each row sits in HBM does.
 * The rule, applied on every full upload (kt_upload_pods, _compact, _packed, and so kt_step_submit): the host reads a strided
 * sample of at most 64 groups of 32 consecutive rows from the caller's ns / meta column.  A group is mixed when its rows with
 * flags != 0 hold more than one namespace (empty and deleted rows carry any ns).  When more than one sampled group in four is
 * mixed the rows are laid out by namespace, otherwise as given (rows already sorted by namespace are mixed only at namespace
 * boundaries).  The sample costs no device round trip and no synchronisation.  Row deltas (kt_update_pod_rows) never change
 * the layout: a row that moves to another namespace stays in its slot (correct, only slower) until the next full upload.
 * Test seam, like kt_debug_set_pass_plan: no product path sets a row order.
 *   kt_debug_set_row_order   mode KT_ROW_ORDER_*, applies from the next full upload of the kind (KT_ERR_INVALID for a bad kind
 *                            or mode).
 *   kt_debug_get_row_order   the layout now resident: *clustered = 1 when laid out by namespace; dev_row[i] (NULL or [n]) = the
 *                            device row of caller row i (i itself when as given). */
#define KT_ROW_ORDER_AUTO 0
#define KT_ROW_ORDER_AS_GIVEN 1
#define KT_ROW_ORDER_BY_NAMESPACE 2
int kt_debug_set_row_order(kt_ctx* ctx, int kind, int mode);
int kt_debug_get_row_order(kt_ctx* ctx, int kind, int64_t* dev_row /*[n] or NULL*/, int32_t* clustered);

/* ---- multi-GPU (row-sharded snapshot, one context per GPU) --------------------- */
/* Each context holds a row shard of both pod kinds and a replica of the throttles; the
 * only exchange is one int64 sum all-reduce of the per-throttle partials between the
 * reconcile and finalize kernels.  uid is an ncclUniqueId (128 bytes) created on rank 0. */
/* With a communicator, kt_evaluate is COLLECTIVE: every rank must call it the same number of times.  The exchange happens
 * inside the pass (finalize tiles read the peers' partial sums over NVLink from IPC-mapped windows; one ncclAllReduce between
 * the kernels when the GPUs cannot map each other).  A rank that never arrives does not wedge the others: the in-kernel wait
 * gives up after two seconds and the next kt_get_* / kt_sync returns KT_ERR_STATE. */
int kt_comm_unique_id(uint8_t uid[128]);
int kt_comm_init(kt_ctx* ctx, const uint8_t uid[128], int nranks, int rank);
int kt_comm_destroy(kt_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* KT_B200_H_ */
