// kt_engine.cu -- implementation of the C ABI in include/kt_b200.h: context, HBM-resident snapshot,
// kernel launches, result download, multi-GPU all-reduce.  There is NO CPU evaluation path in this
// library: without a CUDA device every entry point that needs one fails with KT_ERR_CUDA.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <unistd.h>

#include <algorithm>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/kt_b200.h"
#include "kt_kernels.cuh"
#include "kt_admit.cuh"
#include "kt_keyed.cuh"
#include "kt_nsrows.cuh"
#include "kt_order.cuh"
#include "kt_tables.h"

namespace {

using namespace kt;

// ---- grow-only buffers: device memory (DevBuf) and pinned host memory (PinnedBuf) -------------------------
template <cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Free)(void*)>
struct GrowBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) Free(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;  // slack so row appends do not reallocate every time
    cudaError_t e = Alloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() {
    if (p) Free(p);
    p = nullptr;
    cap = 0;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};
using DevBuf = GrowBuf<cudaMalloc, cudaFree>;
using PinnedBuf = GrowBuf<cudaMallocHost, cudaFreeHost>;

struct PodStore {
  int64_t n = 0;
  DevBuf labels, req, present, flags, ns;
  DevBuf roff;              // [Lpad][n] u32: the labels as row offsets into the current selector tables (k_translate_rows)
  DevBuf winfo;             // [n] u32: the words that can apply to the row's namespace (winfo_pack), same life cycle as roff
  bool roff_valid = false;  // false after a full upload or a table compile; row deltas translate their own rows
  DevBuf c_labels, c_req, c_meta;  // staging of the compact transfer format (kt_upload_pods_compact)
  DevBuf c_pairs;                  // label-pair dictionary of the packed transfer format (kt_upload_pods_packed)
  DevBuf c_dict;                   // request-value dictionaries of the same format
  DevBuf t_rows, t_labels, t_req, t_present, t_flags, t_ns;  // grow-only staging of row deltas
  DevBuf t_words;                                            // per-row results gathered into caller order (to_caller_order)
  DevBuf bitmap;  // [n][Wp]
  // The passes MAINTAIN the bitmap (and, for pending rows, the check codes): they store the words of each row's namespace list
  // and nothing else.  Whatever can leave a stale non-zero word outside those lists -- new rows, a row delta, new tables, a
  // buffer that was just allocated -- clears this flag; the next pass zeroes the buffers once before it runs.
  bool bitmap_clean = false;
  // Row order (kt_order.cuh): with `clustered` the columns above hold the caller's rows sorted by namespace, o_caller[device
  // row] = caller row and o_dev[caller row] = device row; without it no map exists and device row == caller row.
  bool clustered = false;
  int order_mode = 0;                        // kt_debug_set_row_order: 0 automatic, 1 as given, 2 by namespace
  DevBuf o_caller, o_dev, o_scratch;         // the maps; sort keys, ping-pong buffers and digit histograms
  DevBuf g_labels, g_req, g_present, g_flags, g_ns;  // the other half of each column: a re-layout gathers into it and swaps
  void release() {
    labels.release(); req.release(); present.release(); flags.release(); ns.release(); bitmap.release(); roff.release(); winfo.release();
    o_caller.release(); o_dev.release(); o_scratch.release();
    g_labels.release(); g_req.release(); g_present.release(); g_flags.release(); g_ns.release();
    roff_valid = false;
    clustered = false;
    c_labels.release(); c_req.release(); c_meta.release(); c_pairs.release(); c_dict.release();
    t_rows.release(); t_labels.release(); t_req.release(); t_present.release(); t_flags.release(); t_ns.release(); t_words.release();
  }
};

// ---- NCCL through dlopen: the library loads without NCCL; only kt_comm_* needs it ------------------
struct Uid128 { char internal[128]; };
struct NcclApi {
  void* handle = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, /*ncclUniqueId by value: 128 bytes*/ Uid128, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
NcclApi g_nccl;
std::mutex g_nccl_mu;
const char* load_nccl() {
  std::lock_guard<std::mutex> lk(g_nccl_mu);
  if (g_nccl.handle) return nullptr;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return "libnccl.so.2 not found";
  g_nccl.GetUniqueId = (int (*)(void*))dlsym(h, "ncclGetUniqueId");
  g_nccl.CommInitRank = (int (*)(void**, int, Uid128, int))dlsym(h, "ncclCommInitRank");
  g_nccl.CommDestroy = (int (*)(void*))dlsym(h, "ncclCommDestroy");
  g_nccl.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(h, "ncclAllReduce");
  g_nccl.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(h, "ncclAllGather");
  g_nccl.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.CommDestroy || !g_nccl.AllReduce) return "NCCL symbols missing";
  g_nccl.handle = h;
  return nullptr;
}
constexpr int kNcclInt64 = 4;  // ncclInt64
constexpr int kNcclSum = 0;    // ncclSum
constexpr int kNcclChar = 0;   // ncclInt8 / ncclChar

// What the ranks tell each other about their exchange window (one ncclAllGather when the window is (re)allocated).
struct PeerInfo {
  cudaIpcMemHandle_t handle;  // 64 bytes
  unsigned long long ptr;     // the raw device pointer: used instead of the handle when the peer lives in this process
  long long pid;
  int device;
  int ok;                     // the rank could allocate / export its window
};

}  // namespace

struct kt_ctx {
  std::mutex mu;
  int device = 0;
  kt_limits lim{};
  std::string err;
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool timing = false;
  kt_timing last{};

  PodStore pods[2];
  // namespaces (host copy: table compilation needs them again when throttles change)
  int32_t n_ns = 0;
  std::vector<int64_t> ns_labels;
  // throttles
  bool have_throttles = false;
  int32_t M = 0;
  int32_t n_ovr = 0;
  SelectorSpec spec;
  HostTables ht;
  DevBuf d_hash, d_keydir, d_valrow, d_table, d_need, d_nsmask, d_nsw_off, d_nsw_idx;
  // After kt_update_namespace_rows the device copies of nsmask / nsw_off / nsw_idx are the current ones (ht keeps the vectors of
  // the last compile, ht.NS and ht.max_ns_words follow the device).  nsw_total: entries of d_nsw_idx in use.
  int32_t nsw_total = 0;
  DevBuf d_nsspec;  // NsSpecView (kt_nsrows.cuh): the namespace side of the selector spec, one block staged by kt_upload_throttles
  size_t nsspec_at[8] = {};
  std::vector<unsigned char> h_nsspec;
  DevBuf d_kind, d_tflags, d_thr, d_thr_present, d_thr_cnt, d_ovr_off, d_ovr_begin, d_ovr_end, d_ovr_flags, d_ovr_thr,
      d_ovr_present, d_ovr_cnt;
  // kt_update_threshold_rows: the resident ovr_off (host copy) and a spare set of override columns that a change of the
  // override counts rebuilds into before the two sets swap
  std::vector<int32_t> h_ovr_off;
  DevBuf s_ovr_off, s_ovr_begin, s_ovr_end, s_ovr_flags, s_ovr_thr, s_ovr_present, s_ovr_cnt;
  bool have_status = false;
  DevBuf d_st_calculated, d_st_calc_thr, d_st_calc_present, d_st_calc_cnt, d_st_used, d_st_used_present, d_st_used_cnt,
      d_st_throttled;
  bool have_reserved = false;
  DevBuf d_reserved, d_reserved_present, d_reserved_cnt;
  // kt_append_throttle_rows: the spare halves the per-throttle arrays are widened into before each pair swaps (append_targets).
  // Kept for the context's life, so that a creation allocates nothing once they are large enough: after the first append the
  // per-throttle columns (thresholds, status, reservations: (3R + 10) x 8 bytes per throttle at most) take twice their size.
  DevBuf w_spare[16];
  // kt_move_throttle_columns: the spare table, need and nsmask the column gather writes into before each pair swaps
  DevBuf g_spare[3];
  // pass state / outputs
  DevBuf d_part;   // 2 x [2R+1][M] u64 by pass parity: a reconciling pass adds into one half and leaves the other zeroed for its successor
  size_t part_stride = 0;  // bytes between the two halves
  unsigned part_parity = 0;  // half that holds the sums of the last reconcile
  DevBuf d_sync;   // 2 x PassSync counters of the fused pass by pass_parity (zero between launches)
  unsigned pass_parity = 0;  // set of counters and half of d_pre the last fused pass used; the next one takes the other
  DevBuf d_trace;  // optional trace rows of the fused pass, one per match / reconcile / status tile
  bool trace = false;
  uint32_t trace_roles[4] = {0, 0, 0, 0};  // match tiles, reconcile tiles, status tiles, CTAs launched
  PassSync* last_sync = nullptr;  // counters of the last fused pass: its error flag is checked when results are fetched
  kt_pass_plan plan{};            // kt_debug_set_pass_plan: forced choices of the fused pass (inputs only; all zero: automatic)
  bool plan_forced = false;
  kt_pass_plan ran{};             // what the last fused pass launched (kt_debug_get_pass_plan)
  bool have_ran = false;
  DevBuf d_changed;  // device-side status diff: {count[2] u32 by pass parity, pad to 16 B, idx[M] i32, flag[M] u8}
  unsigned diff_parity = 0;
  bool have_diff = false;  // the last pass produced a diff (an observed status was uploaded)
  DevBuf d_col_idx, d_col_cnt, d_col_off, d_col_rows;  // per-throttle row lists (kt_admit.cuh ColumnView): kt_admit_queue, kt_get_match_columns
  DevBuf d_adm_state, d_adm_fail, d_adm_counters;      // kt_admit_queue (kt_admit.cuh)
  DevBuf d_key_reach, d_key_scratch, d_key_acc;  // kt_reconcile_throttles (kt_keyed.cuh): device-only scratch of one call
  DevBuf d_chk_pre;                               // kt_check_pending_rows (kt_keyed.cuh): pre-records of one call
  // What one call sends in (listed rows, throttles, pod values) and brings out (a block of results), and the pinned host
  // copy a block lands in when its results are scattered into several caller arrays.  Staging of the call that uses them:
  // no call reads what another left there.
  DevBuf d_call_in, d_call_out;
  PinnedBuf h_call;
  DevBuf d_pre;    // 2 x [M] pre-records by pass_parity, finalize tiles -> decide tiles (kt_kernels.cuh pre_record_bytes)
  size_t pre_stride = 0;  // bytes between the two halves
  DevBuf d_out;    // the reconcile half's per-throttle outputs: ONE status block of M columns (status_layout)
  bool async_uploads = false;  // kt_set_async_uploads
  cudaEvent_t ev_switch = nullptr;  // kt_set_stream: the new stream waits for what was queued on the old one
  // kt_step_submit / kt_step_wait: one pinned result block, one event
  PinnedBuf h_step;
  size_t step_off[3] = {};
  cudaEvent_t ev_step = nullptr;
  int64_t step_first = 0;
  bool step_pending = false;
  DevBuf d_codes, d_admit;
  bool have_codes = false;      // a checking pass wrote d_codes / d_admit for the current pending rows and throttle columns
  DevBuf d_sparse;              // kt_set_sparse_check: {count u32, pad to 16 B, entries [cap][3] u32}
  uint32_t sparse_cap = 0;      // 0: off
  uint32_t sparse_guess = 1024; // entries fetched together with the count (adapts to the last pass)
  uint32_t* h_sparse_count = nullptr;  // pinned
  bool evaluated = false;
  // multi-GPU
  void* comm = nullptr;
  int nranks = 1, rank = 0;
  int sm_count = 0;
  // peer exchange window: [PassSync | this rank's sums, even / odd passes | all ranks' totals, even / odd passes], mapped by
  // every rank.  The fused pass does the all-reduce itself: finalize tiles ADD this rank's sums into every rank's totals
  // over NVLink and raise a per-rank flag (kt_kernels.cuh PartExchange).
  void* win = nullptr;
  size_t win_part_bytes = 0;  // bytes of ONE partial-sum buffer in the current window
  void* peer_win[8] = {};     // peer_win[r] for r != rank (IPC-opened or raw)
  bool peer_ipc[8] = {};
  bool p2p_failed = false;    // no peer access between the GPUs: stay on the NCCL path
  unsigned epoch = 0;         // passes exchanged through the window so far
  bool win_stale = false;     // the throttle set changed: the window's buffers are laid out for another M -> rebuilt (collectively) before the next pass
};

namespace {

int fail(kt_ctx* c, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (c) c->err = buf;
  return code;
}

#define KT_CUDA(c, expr)                                                                                     \
  do {                                                                                                       \
    cudaError_t _e = (expr);                                                                                 \
    if (_e != cudaSuccess) return fail((c), KT_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(_e));    \
  } while (0)

template <class T>
int upload(kt_ctx* c, DevBuf& b, const T* src, size_t count) {
  KT_CUDA(c, b.reserve(count * sizeof(T) + 16));
  if (count) KT_CUDA(c, cudaMemcpyAsync(b.p, src, count * sizeof(T), cudaMemcpyHostToDevice, c->stream));
  return KT_OK;
}
template <class T>
int upload_vec(kt_ctx* c, DevBuf& b, const std::vector<T>& v) { return upload(c, b, v.data(), v.size()); }
template <class T>
const T* staged(const kt_ctx* c, size_t at) {  // piece at `at` of a call's staged copy (stage_pieces), on the device
  return reinterpret_cast<const T*>(c->d_call_in.as<unsigned char>() + at);
}

// The library's last launch on each stream, while that launch is a fused k_pass: evaluate_locked lets the next fused pass start
// its first phase early only behind one (k_pass).  Every other library call that queues work on a stream forgets the stream's
// entry -- set_device at the top of the entry points, launch(), kt_set_stream, kt_destroy -- so the record never names a pass
// that something of the library's was queued behind.
struct LastPass {
  const kt_ctx* ctx = nullptr;  // nullptr: the last launch was not a fused pass
  bool zero_fill = false;       // that pass zero-filled bitmap or code rows
};
std::mutex g_last_pass_mu;
std::map<cudaStream_t, LastPass> g_last_pass;
LastPass last_pass_on(cudaStream_t s) {
  std::lock_guard<std::mutex> lk(g_last_pass_mu);
  auto it = g_last_pass.find(s);
  return it == g_last_pass.end() ? LastPass{} : it->second;
}
void note_pass(cudaStream_t s, const kt_ctx* c, bool zero_fill) {
  std::lock_guard<std::mutex> lk(g_last_pass_mu);
  g_last_pass[s] = LastPass{c, zero_fill};
}
void forget_pass(cudaStream_t s) {
  std::lock_guard<std::mutex> lk(g_last_pass_mu);
  g_last_pass.erase(s);
}

int set_device(kt_ctx* c) {
  forget_pass(c->stream);
  KT_CUDA(c, cudaSetDevice(c->device));
  return KT_OK;
}

int recompile_tables(kt_ctx* c) {
  std::string e = compile_tables(c->lim, c->spec, c->n_ns, c->ns_labels.empty() ? nullptr : c->ns_labels.data(), &c->ht);
  if (!e.empty()) return fail(c, KT_ERR_INVALID, "compile_tables: %s", e.c_str());
  int rc;
  if ((rc = upload_vec(c, c->d_hash, c->ht.hash))) return rc;
  if ((rc = upload_vec(c, c->d_keydir, c->ht.keydir))) return rc;
  if ((rc = upload_vec(c, c->d_valrow, c->ht.valrow))) return rc;
  if ((rc = upload_vec(c, c->d_table, c->ht.table))) return rc;
  if ((rc = upload_vec(c, c->d_need, c->ht.need))) return rc;
  if ((rc = upload_vec(c, c->d_nsmask, c->ht.nsmask))) return rc;
  if ((rc = upload_vec(c, c->d_nsw_off, c->ht.nsw_off))) return rc;
  if ((rc = upload_vec(c, c->d_nsw_idx, c->ht.nsw_idx))) return rc;
  c->nsw_total = (int32_t)c->ht.nsw_idx.size();
  KT_CUDA(c, cudaStreamSynchronize(c->stream));  // host vectors may be rebuilt right after
  for (auto& s : c->pods) s.roff_valid = s.bitmap_clean = false;  // row offsets point into the tables that were just replaced; word lists changed
  return KT_OK;
}

// After a fused pass has completed: did one of its in-kernel waits give up (a peer rank never arrived)?
int check_pass_error(kt_ctx* c) {
  if (!c->last_sync || !c->evaluated) return KT_OK;
  unsigned err = 0;
  KT_CUDA(c, cudaMemcpyAsync(&err, &c->last_sync->error, sizeof err, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  if (!err) return KT_OK;
  KT_CUDA(c, cudaMemsetAsync(c->last_sync, 0, kPassSyncRearm * sizeof(unsigned), c->stream));  // re-arm the counters, keep the ranks' flags
  KT_CUDA(c, cudaMemsetAsync(&c->last_sync->error, 0, sizeof(unsigned), c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  c->evaluated = false;
  return fail(c, KT_ERR_STATE, "the pass timed out waiting for a peer rank (or for its own tiles): results are void");
}
// Before a getter reads what the last pass left: the device, then the pass's own verdict on its waits.
int device_ready(kt_ctx* c) {
  int rc = set_device(c);
  return rc ? rc : check_pass_error(c);
}

// ---- argument checks: one per condition; every entry point calls the ones it needs, in its own order ----------------
int check_kind(kt_ctx* c, const char* call, int kind) {
  if (kind == KT_PODS_RUNNING || kind == KT_PODS_PENDING) return KT_OK;
  return fail(c, KT_ERR_INVALID, "%s: bad pod kind %d", call, kind);
}
// k caller rows in [0, n)
int check_rows(kt_ctx* c, const char* call, int64_t k, const int64_t* rows, int64_t n) {
  for (int64_t i = 0; i < k; ++i)
    if (rows[i] < 0 || rows[i] >= n) return fail(c, KT_ERR_INVALID, "%s: row %lld out of range [0,%lld)", call, (long long)rows[i], (long long)n);
  return KT_OK;
}
// k throttle columns in [0, M)
int check_throttles(kt_ctx* c, const char* call, int64_t k, const int32_t* idx) {
  for (int64_t i = 0; i < k; ++i)
    if (idx[i] < 0 || idx[i] >= c->M) return fail(c, KT_ERR_INVALID, "%s: throttle %d out of range [0,%d)", call, idx[i], c->M);
  return KT_OK;
}
int check_single_gpu(kt_ctx* c, const char* call) {
  if (!c->comm) return KT_OK;
  return fail(c, KT_ERR_STATE, "%s is single-GPU: this context has a communicator", call);
}

TableView table_view(const kt_ctx* c) {
  TableView tb;
  tb.hash = c->d_hash.as<uint4>();
  tb.hash_mask = c->ht.hash_mask;
  tb.keydir = c->d_keydir.as<uint4>();
  tb.valrow = c->d_valrow.as<uint32_t>();
  tb.n_keydir = (uint32_t)c->ht.n_keydir;
  tb.table = c->d_table.as<uint32_t>();
  tb.need = c->d_need.as<uint32_t>();
  tb.nsmask = c->d_nsmask.as<uint32_t>();
  tb.nsw_off = c->d_nsw_off.as<int32_t>();
  tb.nsw_idx = c->d_nsw_idx.as<int32_t>();
  tb.M = c->ht.M; tb.W = c->ht.W; tb.Wp = c->ht.Wp; tb.TPpad = c->ht.TPpad; tb.B = c->ht.B; tb.rows = c->ht.rows; tb.NS = c->ht.NS;
  return tb;
}

ThrottleView throttle_view(const kt_ctx* c) {
  ThrottleView tv{};
  tv.kind = c->d_kind.as<uint8_t>(); tv.flags = c->d_tflags.as<uint8_t>();
  tv.thr = c->d_thr.as<int64_t>(); tv.thr_present = c->d_thr_present.as<uint32_t>(); tv.thr_cnt = c->d_thr_cnt.as<int64_t>();
  tv.ovr_off = c->d_ovr_off.as<int32_t>(); tv.ovr_begin = c->d_ovr_begin.as<int64_t>(); tv.ovr_end = c->d_ovr_end.as<int64_t>();
  tv.ovr_flags = c->d_ovr_flags.as<uint8_t>(); tv.ovr_thr = c->d_ovr_thr.as<int64_t>(); tv.ovr_present = c->d_ovr_present.as<uint32_t>();
  tv.ovr_cnt = c->d_ovr_cnt.as<int64_t>(); tv.n_ovr = c->n_ovr;
  if (c->have_status) {  // GIVEN_STATUS reads it as the check's input; any reconciling pass diffs its outputs against it
    tv.st_calculated = c->d_st_calculated.as<uint8_t>(); tv.st_calc_thr = c->d_st_calc_thr.as<int64_t>();
    tv.st_calc_present = c->d_st_calc_present.as<uint32_t>(); tv.st_calc_cnt = c->d_st_calc_cnt.as<int64_t>();
    tv.st_used = c->d_st_used.as<int64_t>(); tv.st_used_present = c->d_st_used_present.as<uint32_t>();
    tv.st_used_cnt = c->d_st_used_cnt.as<int64_t>(); tv.st_throttled = c->d_st_throttled.as<uint32_t>();
  }
  if (c->have_reserved) {
    tv.reserved = c->d_reserved.as<int64_t>(); tv.reserved_present = c->d_reserved_present.as<uint32_t>();
    tv.reserved_cnt = c->d_reserved_cnt.as<int64_t>();
  }
  return tv;
}

// ---- the status block -----------------------------------------------------------------------------------------------
// The eight kt_reconcile_out columns of m throttles in one block, every column padded to 16 bytes:
//   {used[R][m], used_cnt[m], calc_thr[R][m], calc_cnt[m], used_present[m], throttled[m], calc_present[m], override_active[m]}
// The pass writes its M columns into one (d_out), so that kt_get_reconcile and a step download them in one copy; the keyed
// calls gather or compute their k columns into one of the same shape.
struct StatusLayout {
  size_t used, used_cnt, calc_thr, calc_cnt, used_present, throttled, calc_present, override_active, bytes;
};
StatusLayout status_layout(int R, int64_t m) {
  StatusLayout l;
  size_t at = 0;
  auto col = [&](size_t bytes) {
    const size_t o = at;
    at += (bytes + 15) & ~(size_t)15;
    return o;
  };
  const size_t res = (size_t)R * m * 8;
  l.used = col(res); l.used_cnt = col((size_t)m * 8); l.calc_thr = col(res); l.calc_cnt = col((size_t)m * 8);
  l.used_present = col((size_t)m * 4); l.throttled = col((size_t)m * 4); l.calc_present = col((size_t)m * 4); l.override_active = col((size_t)m);
  l.bytes = at;
  return l;
}
// The columns of the block at `base`: View is ReconcileView over device memory or kt_reconcile_out over a landed host copy.
template <class View>
View status_at(void* base, int R, int64_t m) {
  const StatusLayout l = status_layout(R, m);
  unsigned char* b = static_cast<unsigned char*>(base);
  View v{};
  v.used = reinterpret_cast<int64_t*>(b + l.used); v.used_cnt = reinterpret_cast<int64_t*>(b + l.used_cnt);
  v.calc_thr = reinterpret_cast<int64_t*>(b + l.calc_thr); v.calc_cnt = reinterpret_cast<int64_t*>(b + l.calc_cnt);
  v.used_present = reinterpret_cast<uint32_t*>(b + l.used_present); v.throttled = reinterpret_cast<uint32_t*>(b + l.throttled);
  v.calc_present = reinterpret_cast<uint32_t*>(b + l.calc_present); v.override_active = reinterpret_cast<uint8_t*>(b + l.override_active);
  return v;
}
// A landed block of m columns into the caller's columns, skipping the NULL ones.
void copy_status(const kt_reconcile_out& src, const kt_reconcile_out* dst, int R, int64_t m) {
  auto put = [](void* d, const void* s, size_t bytes) {
    if (d && bytes) std::memcpy(d, s, bytes);
  };
  const size_t res = (size_t)R * m * 8;
  put(dst->used, src.used, res); put(dst->used_cnt, src.used_cnt, (size_t)m * 8);
  put(dst->calc_thr, src.calc_thr, res); put(dst->calc_cnt, src.calc_cnt, (size_t)m * 8);
  put(dst->used_present, src.used_present, (size_t)m * 4); put(dst->throttled, src.throttled, (size_t)m * 4);
  put(dst->calc_present, src.calc_present, (size_t)m * 4); put(dst->override_active, src.override_active, (size_t)m);
}

// The partial-sum buffers of a pass that exchanges nothing with other ranks: a reconciling pass adds into the half of
// part_parity and zeroes the other one for its successor.
PartExchange local_exchange(const kt_ctx* c) {
  PartExchange px{};
  px.mine = px.total = reinterpret_cast<unsigned long long*>(c->d_part.as<unsigned char>() + (size_t)c->part_parity * c->part_stride);
  px.zero_mine = reinterpret_cast<unsigned long long*>(c->d_part.as<unsigned char>() + (size_t)(c->part_parity ^ 1u) * c->part_stride);
  px.sync = c->d_sync.as<PassSync>() + c->pass_parity;
  px.rank = c->rank;
  return px;
}
// The pre-records of the last pass (a fused pass switches halves first: see pass_parity)
unsigned char* pre_records(const kt_ctx* c) { return c->d_pre.as<unsigned char>() + (size_t)c->pass_parity * c->pre_stride; }

PodView pod_view(const PodStore& s) {
  PodView v;
  v.labels = s.labels.as<int64_t>();
  v.roff = s.roff.as<uint32_t>();
  v.winfo = s.winfo.as<uint32_t>();
  v.req = s.req.as<int64_t>();
  v.present = s.present.as<uint32_t>();
  v.flags = s.flags.as<uint32_t>();
  v.ns = s.ns.as<int32_t>();
  v.n = s.n;
  v.zero_fill = s.bitmap_clean ? 0 : 1;
  return v;
}

// Label columns -> row offsets of the current tables, for every row (rows_dev == nullptr) or for k listed rows.
int translate_rows(kt_ctx* c, PodStore& s, int64_t k, const int64_t* rows_dev) {
  const int Lpad = (c->lim.label_slots + 7) & ~7;
  if (k <= 0) return KT_OK;
  k_translate_rows<<<(unsigned)((k + 255) / 256), 256, 0, c->stream>>>(k, rows_dev, table_view(c), Lpad, s.n, s.labels.as<int64_t>(), s.ns.as<int32_t>(),
                                                                          s.roff.as<uint32_t>(), s.winfo.as<uint32_t>());
  KT_CUDA(c, cudaGetLastError());
  return KT_OK;
}
// Before a pass: the store's row offsets must match its labels and the current tables.
int ensure_roff(kt_ctx* c, PodStore& s) {
  if (s.roff_valid || !c->have_throttles) return KT_OK;
  const int Lpad = (c->lim.label_slots + 7) & ~7;
  KT_CUDA(c, s.roff.reserve((size_t)Lpad * s.n * 4 + 16));
  KT_CUDA(c, s.winfo.reserve((size_t)s.n * 4 + 16));
  int rc = translate_rows(c, s, s.n, nullptr);
  if (rc) return rc;
  s.roff_valid = true;
  return KT_OK;
}

// ---- row order (kt_order.cuh) --------------------------------------------------------------------------------------
// The layout of a full upload, chosen on the host from the caller's own arrays, with no device round trip: a strided sample of
// at most kOrderSampleGroups groups of 32 consecutive rows.  A group is mixed when its rows with flags != 0 hold more than one
// namespace (empty and deleted rows carry arbitrary namespaces).  More than one sampled group in kOrderMixedDiv mixed: the rows
// are laid out by namespace; otherwise as given.  Rows sorted by namespace are mixed only where one namespace ends and the
// next begins.
constexpr int64_t kOrderSampleGroups = 64;
constexpr int64_t kOrderMixedDiv = 4;
// row(i, &ns) stores row i's namespace and says whether its flags are non-zero
template <class Row>
bool choose_clustered(const PodStore& s, int64_t n, Row row) {
  if (n <= 0 || s.order_mode == 1) return false;
  if (s.order_mode == 2) return true;
  const int64_t groups = n / 32;
  if (groups == 0) return false;
  const int64_t sample = std::min(groups, kOrderSampleGroups), stride = groups / sample;
  int64_t mixed = 0;
  for (int64_t g = 0; g < sample; ++g) {
    const int64_t r0 = g * stride * 32;
    bool seen = false, mix = false;
    int32_t first = 0;
    for (int j = 0; j < 32 && !mix; ++j) {
      int32_t ns;
      if (!row(r0 + j, &ns)) continue;
      if (!seen) first = ns;
      mix = seen && ns != first;
      seen = true;
    }
    mixed += mix ? 1 : 0;
  }
  return mixed * kOrderMixedDiv > sample;
}

// The n rows just landed in the store's columns (caller order, queued on the stream) -> sorted by namespace: the maps, then
// every row column gathered into its other half.  ns_limit bounds the namespace ids the transfer format can carry, so that
// the radix passes cover only the digits a key can have.
int order_rows(kt_ctx* c, PodStore& s, int64_t n, int64_t ns_limit) {
  if (n > (int64_t)UINT32_MAX) return fail(c, KT_ERR_LIMIT, "%lld rows: a table laid out by namespace holds at most 2^32 - 1", (long long)n);
  const int L = c->lim.label_slots, R = c->lim.n_resources, Lpad = (L + 7) & ~7;
  const int64_t max_key = std::min<int64_t>(c->n_ns, ns_limit - 1);
  int passes = 0;
  while (passes < 4 && (max_key >> (8 * passes)) != 0) ++passes;
  const int nblk = (int)((n + kOrderTile - 1) / kOrderTile);
  const size_t hist_len = (size_t)kOrderDigits * nblk;
  KT_CUDA(c, s.o_caller.reserve((size_t)n * 4 + 16));
  KT_CUDA(c, s.o_dev.reserve((size_t)n * 4 + 16));
  KT_CUDA(c, s.o_scratch.reserve(((size_t)3 * n + hist_len) * 4 + 16));
  uint32_t* sc = s.o_scratch.as<uint32_t>();
  uint32_t* keys[2] = {sc, sc + n};
  uint32_t* vals[2] = {s.o_caller.as<uint32_t>(), sc + 2 * n};
  uint32_t* hist = sc + 3 * n;
  int cur = passes & 1;  // so that the last pass leaves the permutation in o_caller
  const unsigned g = (unsigned)((n + 255) / 256);
  k_order_keys<<<g, 256, 0, c->stream>>>(n, s.ns.as<int32_t>(), (uint32_t)c->n_ns, keys[cur], vals[cur]);
  for (int d = 0; d < passes; ++d, cur ^= 1) {
    k_order_hist<<<nblk, kOrderThreads, 0, c->stream>>>(n, keys[cur], 8 * d, hist, nblk);
    k_order_scan<<<1, 1024, 0, c->stream>>>(hist, (int64_t)hist_len);
    k_order_scatter<<<nblk, kOrderThreads, 0, c->stream>>>(n, keys[cur], vals[cur], 8 * d, hist, nblk, keys[cur ^ 1], vals[cur ^ 1]);
  }
  const uint32_t* caller_of = s.o_caller.as<uint32_t>();
  k_order_invert<<<g, 256, 0, c->stream>>>(n, caller_of, s.o_dev.as<uint32_t>());
  KT_CUDA(c, cudaGetLastError());
  auto gather = [&](DevBuf& col, DevBuf& other, int cols, auto elem) -> int {
    using T = decltype(elem);
    KT_CUDA(c, other.reserve((size_t)cols * n * sizeof(T) + 16));
    const int64_t e = (int64_t)cols * n;
    k_order_gather_cols<T><<<(unsigned)((e + 255) / 256), 256, 0, c->stream>>>(n, cols, caller_of, col.as<T>(), other.as<T>());
    KT_CUDA(c, cudaGetLastError());
    std::swap(col, other);
    return KT_OK;
  };
  int rc;
  if ((rc = gather(s.labels, s.g_labels, Lpad, int64_t{})) || (rc = gather(s.req, s.g_req, R, int64_t{})) ||
      (rc = gather(s.present, s.g_present, 1, uint32_t{})) || (rc = gather(s.flags, s.g_flags, 1, uint32_t{})) || (rc = gather(s.ns, s.g_ns, 1, int32_t{})))
    return rc;
  s.clustered = true;
  return KT_OK;
}
// caller row -> device row, or nullptr when the rows are stored as given
const uint32_t* dev_of(const PodStore& s) { return s.clustered ? s.o_dev.as<uint32_t>() : nullptr; }
// k caller rows -> `buf` on the device, as rows of the store's layout (mapped to device rows when it is laid out by namespace)
int stage_rows(kt_ctx* c, const PodStore& s, DevBuf& buf, int64_t k, const int64_t* rows) {
  int rc = upload(c, buf, rows, (size_t)k);
  if (rc) return rc;
  if (s.clustered) k_order_map_rows<<<(unsigned)((k + 255) / 256), 256, 0, c->stream>>>(k, s.o_dev.as<uint32_t>(), buf.as<int64_t>());
  return KT_OK;
}
// The end of every full upload: the n rows just landed in caller order are laid out by namespace when `cluster`, and
// everything computed from the previous rows is void.
int finish_upload(kt_ctx* c, int kind, int64_t n, bool cluster, int64_t ns_limit, bool roff_valid) {
  PodStore& s = c->pods[kind];
  s.clustered = false;
  if (cluster) {
    int rc = order_rows(c, s, n, ns_limit);
    if (rc) return rc;
  }
  s.n = n;
  s.roff_valid = roff_valid;
  s.bitmap_clean = false;
  c->evaluated = false;
  if (kind == KT_PODS_PENDING) c->have_codes = false;
  if (!c->async_uploads) KT_CUDA(c, cudaStreamSynchronize(c->stream));  // the caller may reuse its buffers as soon as we return
  return KT_OK;
}
// n per-row results of `W` u32 words (bitmap rows, code rows; W = 0: one byte per row) gathered into caller order in the
// store's staging buffer; returns it
template <class T>
const T* to_caller_order(kt_ctx* c, PodStore& s, const T* src, int W, size_t staging_at = 0) {
  const int64_t e = s.n * (W ? W : 1);
  T* dst = reinterpret_cast<T*>(s.t_words.as<unsigned char>() + staging_at);
  if (W) k_order_gather_rows<<<(unsigned)((e + 255) / 256), 256, 0, c->stream>>>(s.n, W, s.o_dev.as<uint32_t>(), (const uint32_t*)src, (uint32_t*)dst);
  else k_order_gather_cols<T><<<(unsigned)((e + 255) / 256), 256, 0, c->stream>>>(s.n, 1, s.o_dev.as<uint32_t>(), src, dst);
  return dst;
}
// The admit bits of the last pass in caller order: d_admit itself, or gathered into the pending store's staging buffer at byte `at`.
int admit_in_caller_order(kt_ctx* c, const unsigned char** out, size_t at = 0) {
  PodStore& pend = c->pods[KT_PODS_PENDING];
  *out = c->d_admit.as<unsigned char>();
  if (!pend.clustered) return KT_OK;
  KT_CUDA(c, pend.t_words.reserve(at + (size_t)pend.n + 16));
  *out = to_caller_order(c, pend, *out, 0, at);
  return KT_OK;
}
// the pass's sparse check entries name device rows: rewritten to caller rows once, on the stream right after the pass
int sparse_to_caller(kt_ctx* c) {
  const PodStore& pend = c->pods[KT_PODS_PENDING];
  if (!c->sparse_cap || !pend.clustered || pend.n == 0) return KT_OK;
  forget_pass(c->stream);
  k_order_sparse_rows<<<(unsigned)c->sm_count * 2, 256, 0, c->stream>>>(c->d_sparse.as<uint32_t>(), c->sparse_cap, c->d_sparse.as<uint32_t>() + 4,
                                                                       pend.o_caller.as<uint32_t>());
  KT_CUDA(c, cudaGetLastError());
  return KT_OK;
}

// ---- peer exchange window ------------------------------------------------------------------------------
constexpr size_t kWinHeader = 256;  // PassSync lives at offset 0, the partial-sum buffers follow
void release_window(kt_ctx* c) {
  for (int r = 0; r < 8; ++r) {
    if (c->peer_win[r] && c->peer_ipc[r]) cudaIpcCloseMemHandle(c->peer_win[r]);
    c->peer_win[r] = nullptr;
    c->peer_ipc[r] = false;
  }
  if (c->win) cudaFree(c->win);
  c->win = nullptr;
  c->win_part_bytes = 0;
}
// Collective over the communicator (every rank reaches it in the same kt_evaluate because M and R are replicated):
// (re)allocate this rank's window, exchange the IPC handles with one ncclAllGather, map the peers' windows.
// Returns KT_OK with c->p2p_failed set when the GPUs cannot reach each other (the caller then uses NCCL).
int ensure_window(kt_ctx* c, size_t part_bytes) {
  if (c->p2p_failed || (c->win && !c->win_stale && c->win_part_bytes >= part_bytes)) return KT_OK;
  c->win_stale = false;
  if (!g_nccl.AllGather || c->nranks > 8) { c->p2p_failed = true; return KT_OK; }
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  release_window(c);
  const size_t want = (part_bytes + part_bytes / 4 + 4096 + 255) & ~(size_t)255;
  PeerInfo mine{};
  mine.pid = (long long)getpid();
  mine.device = c->device;
  void* w = nullptr;
  // [header | this rank's sums x2 parities | all-rank totals x2 | slots x2 parities x nranks: 16 bytes per value (two tagged words)]
  const size_t win_bytes = kWinHeader + 4 * want + 2 * (size_t)c->nranks * 2 * want;
  if (cudaMalloc(&w, win_bytes) == cudaSuccess && cudaMemset(w, 0, win_bytes) == cudaSuccess &&
      cudaIpcGetMemHandle(&mine.handle, w) == cudaSuccess) {
    mine.ok = 1;
    mine.ptr = (unsigned long long)w;
  } else {
    cudaGetLastError();
  }
  DevBuf d_in, d_out;
  KT_CUDA(c, d_in.reserve(sizeof(PeerInfo)));
  KT_CUDA(c, d_out.reserve(sizeof(PeerInfo) * c->nranks));
  KT_CUDA(c, cudaMemcpyAsync(d_in.p, &mine, sizeof mine, cudaMemcpyHostToDevice, c->stream));
  int e = g_nccl.AllGather(d_in.p, d_out.p, sizeof(PeerInfo), kNcclChar, c->comm, c->stream);
  if (e != 0) return fail(c, KT_ERR_NCCL, "ncclAllGather: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(e) : "error");
  std::vector<PeerInfo> all((size_t)c->nranks);
  KT_CUDA(c, cudaMemcpyAsync(all.data(), d_out.p, sizeof(PeerInfo) * c->nranks, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  d_in.release();
  d_out.release();
  bool ok = true;
  for (auto& pi : all) ok = ok && pi.ok;
  for (int r = 0; ok && r < c->nranks; ++r) {
    if (r == c->rank) continue;
    if (all[r].pid == mine.pid) {  // another context of this process (one Go process driving several GPUs)
      int can = 0;
      if (cudaDeviceCanAccessPeer(&can, c->device, all[r].device) != cudaSuccess || !can) { ok = false; break; }
      cudaError_t pe = cudaDeviceEnablePeerAccess(all[r].device, 0);
      if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) { ok = false; break; }
      cudaGetLastError();
      c->peer_win[r] = (void*)all[r].ptr;
    } else {
      void* pw = nullptr;
      if (cudaIpcOpenMemHandle(&pw, all[r].handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = false; break; }
      c->peer_win[r] = pw;
      c->peer_ipc[r] = true;
    }
  }
  // every rank must reach the same verdict: a second tiny all-gather of the local one
  int verdict = ok ? 1 : 0;
  DevBuf d_v, d_vs;
  KT_CUDA(c, d_v.reserve(4));
  KT_CUDA(c, d_vs.reserve(4 * (size_t)c->nranks));
  KT_CUDA(c, cudaMemcpyAsync(d_v.p, &verdict, 4, cudaMemcpyHostToDevice, c->stream));
  e = g_nccl.AllGather(d_v.p, d_vs.p, 4, kNcclChar, c->comm, c->stream);
  if (e != 0) return fail(c, KT_ERR_NCCL, "ncclAllGather: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(e) : "error");
  std::vector<int> verdicts((size_t)c->nranks);
  KT_CUDA(c, cudaMemcpyAsync(verdicts.data(), d_vs.p, 4 * (size_t)c->nranks, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  d_v.release();
  d_vs.release();
  for (int v : verdicts) ok = ok && v;
  c->win = w;
  if (!ok) {
    release_window(c);
    c->p2p_failed = true;
    return KT_OK;
  }
  c->win_part_bytes = want;
  c->epoch = 0;  // fresh windows everywhere: all epochs restart together
  return KT_OK;
}

// ---- launches ------------------------------------------------------------------------------------
// Every kernel goes through cudaLaunchKernelEx so that the dependent ones can carry the programmatic
// stream serialization attribute (PDL): the secondary grid may start while the primary still runs and
// synchronises on it with griddepcontrol.wait where it first needs the primary's results.
// The rule: a kernel launched with PDL either waits at its top (k_pass), or its primary -- the kernel right
// before it in the stream -- was launched by the same call, or it is an early k_pass whose primary is a k_pass
// (evaluate_locked: g_last_pass).  Its primary is otherwise whatever the caller queued last (another pass of this
// context, another context's pass on a shared stream), and the writes it makes before its wait would race with that work.
template <class... KArgs, class... Args>
cudaError_t launch(kt_ctx* c, void (*kern)(KArgs...), unsigned blocks, unsigned threads, size_t smem, bool pdl, Args... args) {
  forget_pass(c->stream);
  cudaError_t e = cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(blocks);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = c->stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

int reconcile_slots(const kt_ctx* c) {
  int s = c->ht.max_ns_words + 2;  // a tile usually spans one or two namespaces
  if (s < 4) s = 4;
  if (s > kMaxSlots) s = kMaxSlots;
  return s;
}
template <int TPC, int B, int RT, bool REG>
cudaError_t launch_reconcile(kt_ctx* c, const PodView& pv, const TableView& tb, unsigned long long* part, unsigned blocks) {
  const int L = c->lim.label_slots, R = c->lim.n_resources, S = reconcile_slots(c);
  return launch(c, k_reconcile<TPC, B, RT, REG>, blocks, kTileReconcile, reconcile_smem_bytes(L, R, S, REG, kTileReconcile), false, pv, tb, L, R, S,
                c->pods[KT_PODS_RUNNING].bitmap.as<uint32_t>(), part);
}
SparseOut sparse_view(const kt_ctx* c) {
  SparseOut sp{nullptr, nullptr, 0};
  if (c->sparse_cap) {
    sp.count = c->d_sparse.as<uint32_t>();
    sp.ent = c->d_sparse.as<uint32_t>() + 4;
    sp.cap = c->sparse_cap;
  }
  return sp;
}
template <int TPC, int B, bool REG>
cudaError_t launch_check(kt_ctx* c, const PodView& pv, const TableView& tb, const PartExchange& px, unsigned blocks, bool pdl) {
  const int L = c->lim.label_slots, R = c->lim.n_resources;
  return launch(c, k_check<TPC, B, REG>, blocks, kTileCheck, check_smem_bytes(L, R, REG, kTileCheck), pdl, pv, tb, L, R,
                (const unsigned char*)pre_records(c), px, c->pods[KT_PODS_PENDING].bitmap.as<uint32_t>(),
                c->d_codes.as<uint32_t>(), c->d_admit.as<unsigned char>(), sparse_view(c));
}
// Occupancy of k_pass compiled for THREADS resident threads per SM: CTAs the device holds at once.
template <int TPC, int B, int RT, bool REG, int TILE, int THREADS>
cudaError_t pass_capacity(kt_ctx* c, size_t smem, unsigned* capacity) {
  int per_sm = 0;
  cudaError_t e = cudaFuncSetAttribute((const void*)k_pass<TPC, B, RT, REG, TILE, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pass<TPC, B, RT, REG, TILE, THREADS>, TILE, smem);
  *capacity = (unsigned)per_sm * (unsigned)c->sm_count;
  return e;
}
// A pass whose first-phase tiles are more than this many rounds of the 512-thread grid runs the 768-thread build.  Measured on
// either side (C4: 3.3 rounds, 46 us both ways; C5 and C2 x 10: 16 rounds, 178 against 167 us); where between 3.3 and 16 the two
// cross has not been measured.
constexpr unsigned kDeepRounds = 8;
template <int TPC, int B, int RT, bool REG, int TILE>
cudaError_t launch_pass(kt_ctx* c, const PassArgs& a0) {
  const int L = c->lim.label_slots, R = c->lim.n_resources;
  size_t smem = reconcile_smem_bytes(L, R, a0.S, REG, TILE);
  const size_t smem_chk = check_smem_bytes(L, R, REG, TILE);
  if (smem_chk > smem) smem = smem_chk;
  PassArgs a = a0;
  a.n_rec = (unsigned)((a.run.n + TILE - 1) / TILE);
  a.n_fin = (unsigned)(((long long)a.tb.M * a.G + TILE - 1) / TILE);
  a.n_chk = (unsigned)((a.pend.n + TILE - 1) / TILE);
  // Persistent grid: as many CTAs as the device holds at once (never more than there are first-phase tiles); each one draws
  // tiles until the ticket counter runs out, so every CTA is placed at the start and the second phase is shared by all of them.
  const unsigned tiles = a.n_chk + a.n_rec;
  // a forced plan (kt_debug_set_pass_plan) caps the grid before both choices below and may override either of them
  const kt_pass_plan& fp = c->plan;
  auto capped = [&](unsigned n) { return fp.max_ctas != 0 && fp.max_ctas < n ? fp.max_ctas : n; };
  unsigned capacity = 0;
  cudaError_t e = pass_capacity<TPC, B, RT, REG, TILE, kPassThreadsShallow>(c, smem, &capacity);
  if (e != cudaSuccess) return e;
  const bool deep = fp.threads_per_sm ? fp.threads_per_sm == kPassThreadsDeep : tiles > kDeepRounds * capped(capacity);
  if (deep && (e = pass_capacity<TPC, B, RT, REG, TILE, kPassThreadsDeep>(c, smem, &capacity)) != cudaSuccess) return e;
  const unsigned avail = capped(capacity);
  const unsigned grid = tiles < avail ? tiles : avail;
  // The decide work: four lanes per pod in sub-tiles of TILE/4 pods spread it over every CTA, but each sub-tile stages its own
  // pre-records and finishes its own constants -- a latency chain of several L2 trips.  That pays while the sub-tiles take at
  // most two rounds of the grid (C4: 625 sub-tiles on 528 CTAs, 46 us against 50 us); beyond that (C5: 3125 sub-tiles on 792 CTAs,
  // 185 us against 167 us) the rounds queue up and lane-per-pod tiles of TILE pods do the same work in a quarter of the pieces.  The
  // factor 2 lies between those two shapes (1.2 and 5.9 rounds); where between them the two cross has not been measured.
  const unsigned n_quad = (unsigned)((a.pend.n + TILE / 4 - 1) / (TILE / 4));
  a.quad = fp.decide ? fp.decide == KT_PLAN_DECIDE_QUAD : n_quad <= 2 * grid;
  a.n_sub = a.quad ? n_quad : a.n_chk;
  if (c->trace) { c->trace_roles[0] = a.n_chk; c->trace_roles[1] = a.n_rec; c->trace_roles[2] = a.n_fin; c->trace_roles[3] = grid; }
  kt_pass_plan& ran = c->ran;
  ran = kt_pass_plan{deep ? kPassThreadsDeep : kPassThreadsShallow, a.quad ? KT_PLAN_DECIDE_QUAD : KT_PLAN_DECIDE_PER_POD, fp.max_ctas, grid, capacity,
                     TILE, TPC, B, RT, a.n_chk, a.n_rec, a.n_fin, a.n_sub};
  return deep ? launch(c, k_pass<TPC, B, RT, REG, TILE, kPassThreadsDeep>, grid, TILE, smem, /*pdl=*/true, a)
              : launch(c, k_pass<TPC, B, RT, REG, TILE, kPassThreadsShallow>, grid, TILE, smem, /*pdl=*/true, a);
}
// The kernel variant, chosen here for every launch: TPC term planes per table entry (1 or 2), B counter bits (2 or 6), RT the
// compile-time bound on R of the register accumulators (0: accumulate in shared memory), REG label rows in registers.  `go`
// is called with one std::integral_constant per template argument.
//   Fast family (REG, RT = 4 for R <= 4, else 8): L <= 8, B = 2 and R <= 8.  General family: any L <= 32, R <= 31, B in {2, 6}.
//   `check`: the check keeps no per-resource registers, so it takes register rows whenever L <= 8 and B = 2, whatever R is --
//   with R > 8 a register-row check runs beside a general reconcile (RT means nothing to it).
template <class Go>
cudaError_t with_variant(const kt_ctx* c, bool check, Go&& go) {
  using B2 = std::integral_constant<int, 2>;
  using B6 = std::integral_constant<int, 6>;
  const bool t1 = c->ht.TPpad == 1, b2 = c->ht.B <= 2;
  const int R = c->lim.n_resources;
  auto by_tpc = [&](auto b, auto rt, auto reg) {
    return t1 ? go(std::integral_constant<int, 1>{}, b, rt, reg) : go(std::integral_constant<int, 2>{}, b, rt, reg);
  };
  if (c->lim.label_slots <= 8 && b2 && (check || R <= 8))
    return R <= 4 ? by_tpc(B2{}, std::integral_constant<int, 4>{}, std::true_type{}) : by_tpc(B2{}, std::integral_constant<int, 8>{}, std::true_type{});
  return b2 ? by_tpc(B2{}, std::integral_constant<int, 0>{}, std::false_type{}) : by_tpc(B6{}, std::integral_constant<int, 0>{}, std::false_type{});
}
cudaError_t dispatch_pass(kt_ctx* c, const PassArgs& a) {
  // ClusterThrottle-heavy tables (a namespace's word list is long): 256 pods share a CTA's accumulator slots
  const bool wide = a.S >= 8;
  return with_variant(c, false, [&](auto tpc, auto b, auto rt, auto reg) {
    if constexpr (reg) {
      if (wide) return launch_pass<tpc, b, rt, reg, 256>(c, a);
    }
    return launch_pass<tpc, b, rt, reg, kTileReconcile>(c, a);
  });
}
cudaError_t dispatch_reconcile(kt_ctx* c, const PodView& pv, const TableView& tb, unsigned long long* part, unsigned blocks) {
  return with_variant(c, false, [&](auto tpc, auto b, auto rt, auto reg) { return launch_reconcile<tpc, b, rt, reg>(c, pv, tb, part, blocks); });
}
cudaError_t dispatch_check(kt_ctx* c, const PodView& pv, const TableView& tb, const PartExchange& px, unsigned blocks, bool pdl) {
  return with_variant(c, true, [&](auto tpc, auto b, auto, auto reg) { return launch_check<tpc, b, reg>(c, pv, tb, px, blocks, pdl); });
}

// The pinned blocks kt_host_alloc / kt_host_alloc_upload handed out (start -> bytes).  Separate allocations may lie side by
// side in the address space, and the runtime refuses a copy that spans two of them: a packed upload sends its columns as one
// transfer only when they lie inside ONE of these blocks.
std::mutex g_host_mu;
std::map<uintptr_t, size_t> g_host_blocks;
void* host_alloc(size_t bytes, unsigned flags) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, flags) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lk(g_host_mu);
  g_host_blocks[(uintptr_t)p] = bytes ? bytes : 1;
  return p;
}
bool in_one_host_block(uintptr_t lo, uintptr_t hi) {
  std::lock_guard<std::mutex> lk(g_host_mu);
  auto it = g_host_blocks.upper_bound(lo);
  if (it == g_host_blocks.begin()) return false;
  --it;
  return hi <= it->first + it->second;
}

}  // namespace

extern "C" {

const char* kt_version(void) { return "kt_b200 0.1 (sm_90a, abi 1)"; }

const char* kt_last_error(const kt_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int kt_create(kt_ctx** out, int device, const kt_limits* lim) {
  if (!out || !lim) return KT_ERR_INVALID;
  *out = nullptr;
  if (lim->abi_version != KT_ABI_VERSION) return KT_ERR_INVALID;
  if (lim->n_resources < 1 || lim->n_resources > KT_MAX_RESOURCES) return KT_ERR_LIMIT;
  if (lim->label_slots < 1 || lim->label_slots > KT_MAX_LABEL_SLOTS) return KT_ERR_LIMIT;
  if (lim->ns_label_slots < 0 || lim->ns_label_slots > KT_MAX_LABEL_SLOTS) return KT_ERR_LIMIT;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return KT_ERR_CUDA;  // no GPU: no fallback, by design
  if (device < 0 || device >= ndev) return KT_ERR_INVALID;
  kt_ctx* c = new kt_ctx();
  c->device = device;
  c->lim = *lim;
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete c;
    return KT_ERR_CUDA;
  }
  c->stream = c->own_stream;
  if (cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || c->sm_count <= 0) { delete c; return KT_ERR_CUDA; }
  for (auto& e : c->ev)
    if (cudaEventCreate(&e) != cudaSuccess) { delete c; return KT_ERR_CUDA; }
  if (cudaEventCreateWithFlags(&c->ev_switch, cudaEventDisableTiming) != cudaSuccess) { kt_destroy(c); return KT_ERR_CUDA; }
  if (c->d_sync.reserve(2 * sizeof(PassSync)) != cudaSuccess || cudaMemset(c->d_sync.p, 0, 2 * sizeof(PassSync)) != cudaSuccess) { kt_destroy(c); return KT_ERR_CUDA; }
  *out = c;
  return KT_OK;
}

void kt_destroy(kt_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  forget_pass(c->stream);
  release_window(c);
  if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
  for (auto& s : c->pods) s.release();
  DevBuf* all[] = {&c->d_hash, &c->d_keydir, &c->d_valrow, &c->d_table, &c->d_need, &c->d_nsmask, &c->d_nsw_off, &c->d_nsw_idx, &c->d_kind, &c->d_tflags, &c->d_thr,
                   &c->d_thr_present, &c->d_thr_cnt, &c->d_ovr_off, &c->d_ovr_begin, &c->d_ovr_end, &c->d_ovr_flags, &c->d_ovr_thr,
                   &c->d_ovr_present, &c->d_ovr_cnt, &c->d_st_calculated, &c->d_st_calc_thr, &c->d_st_calc_present, &c->d_st_calc_cnt,
                   &c->d_st_used, &c->d_st_used_present, &c->d_st_used_cnt, &c->d_st_throttled, &c->d_reserved, &c->d_reserved_present,
                   &c->d_reserved_cnt, &c->d_part, &c->d_sync, &c->d_trace, &c->d_pre, &c->d_changed, &c->d_col_idx, &c->d_col_cnt, &c->d_col_off,
                   &c->d_col_rows, &c->d_adm_state, &c->d_adm_fail, &c->d_adm_counters, &c->d_out, &c->d_codes, &c->d_admit,
                   &c->d_key_reach, &c->d_key_scratch, &c->d_key_acc, &c->d_chk_pre, &c->d_call_in, &c->d_call_out, &c->d_nsspec,
                   &c->s_ovr_off, &c->s_ovr_begin, &c->s_ovr_end, &c->s_ovr_flags, &c->s_ovr_thr, &c->s_ovr_present, &c->s_ovr_cnt};
  c->h_call.release();
  c->h_step.release();
  if (c->ev_step) cudaEventDestroy(c->ev_step);
  if (c->ev_switch) cudaEventDestroy(c->ev_switch);
  if (c->h_sparse_count) cudaFreeHost(c->h_sparse_count);
  c->d_sparse.release();
  for (DevBuf* b : all) b->release();
  for (DevBuf& b : c->w_spare) b.release();
  for (DevBuf& b : c->g_spare) b.release();
  for (auto& e : c->ev)
    if (e) cudaEventDestroy(e);
  if (c->own_stream) cudaStreamDestroy(c->own_stream);
  delete c;
}

int kt_set_stream(kt_ctx* c, void* cuda_stream) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  const cudaStream_t next = cuda_stream ? (cudaStream_t)cuda_stream : c->own_stream;
  if (next == c->stream) return KT_OK;
  int rc = set_device(c);
  if (rc) return rc;
  // work queued on the old stream (async uploads, passes) stays ahead of everything queued on the new one, and a kt_sync on
  // the new stream covers it
  KT_CUDA(c, cudaEventRecord(c->ev_switch, c->stream));
  KT_CUDA(c, cudaStreamWaitEvent(next, c->ev_switch, 0));
  forget_pass(next);
  c->stream = next;
  return KT_OK;
}

int kt_enable_timing(kt_ctx* c, int on) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  c->timing = on != 0;
  return KT_OK;
}

int kt_enable_trace(kt_ctx* c, int on) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  c->trace = on != 0;
  return KT_OK;
}

int64_t kt_get_trace(kt_ctx* c, uint64_t* rows, int64_t cap, uint32_t roles[4]) {
  if (!c || cap < 0 || (cap > 0 && !rows)) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc = set_device(c);
  if (rc) return rc;
  const int64_t total = (int64_t)c->trace_roles[0] + c->trace_roles[1] + c->trace_roles[2];
  if (roles) std::memcpy(roles, c->trace_roles, sizeof c->trace_roles);
  if (!c->trace || !c->d_trace.p || total == 0) return 0;
  const int64_t n = total < cap ? total : cap;
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  if (n > 0) KT_CUDA(c, cudaMemcpy(rows, c->d_trace.p, (size_t)n * kTraceRow * 8, cudaMemcpyDeviceToHost));
  return n;
}

int kt_set_async_uploads(kt_ctx* c, int on) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  c->async_uploads = on != 0;
  return KT_OK;
}

int kt_sync(kt_ctx* c) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc = set_device(c);
  if (rc) return rc;
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  return check_pass_error(c);
}

void* kt_host_alloc(size_t bytes) { return host_alloc(bytes, cudaHostAllocDefault); }
void* kt_host_alloc_upload(size_t bytes) { return host_alloc(bytes, cudaHostAllocWriteCombined); }
void kt_host_free(void* p) {
  if (!p) return;
  {
    std::lock_guard<std::mutex> lk(g_host_mu);
    g_host_blocks.erase((uintptr_t)p);
  }
  cudaFreeHost(p);
}

int kt_upload_pods(kt_ctx* c, int kind, int64_t n, const int64_t* labels, const int64_t* req, const uint32_t* present,
                   const uint32_t* flags, const int32_t* ns_id) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (int rc = check_kind(c, __func__, kind)) return rc;
  if (n < 0 || (n > 0 && (!labels || !req || !present || !flags || !ns_id))) return fail(c, KT_ERR_INVALID, "null pod columns");
  int rc = set_device(c);
  if (rc) return rc;
  PodStore& s = c->pods[kind];
  const int L = c->lim.label_slots, R = c->lim.n_resources;
  // label columns are padded to a multiple of eight slots with KT_LABEL_EMPTY (all bytes 0xFF): the kernels
  // translate labels in unpredicated chunks of eight
  const int Lpad = (L + 7) & ~7;
  KT_CUDA(c, s.labels.reserve((size_t)Lpad * n * 8 + 16));
  if (n) {
    KT_CUDA(c, cudaMemcpyAsync(s.labels.p, labels, (size_t)L * n * 8, cudaMemcpyHostToDevice, c->stream));
    if (Lpad > L) KT_CUDA(c, cudaMemsetAsync(s.labels.as<int64_t>() + (size_t)L * n, 0xFF, (size_t)(Lpad - L) * n * 8, c->stream));
  }
  if ((rc = upload(c, s.req, req, (size_t)R * n))) return rc;
  if ((rc = upload(c, s.present, present, (size_t)n))) return rc;
  if ((rc = upload(c, s.flags, flags, (size_t)n))) return rc;
  if ((rc = upload(c, s.ns, ns_id, (size_t)n))) return rc;
  const bool cluster = choose_clustered(s, n, [&](int64_t i, int32_t* ns) { *ns = ns_id[i]; return flags[i] != 0; });
  return finish_upload(c, kind, n, cluster, (int64_t)1 << 31, false);
}

int kt_upload_pods_compact(kt_ctx* c, int kind, int64_t n, int32_t val_bits, const uint32_t* labels32, const int32_t* req32, const int32_t* req_shift,
                           const uint32_t* present, const uint32_t* meta) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (int rc = check_kind(c, __func__, kind)) return rc;
  if (n < 0 || !req_shift || (n > 0 && (!labels32 || !req32 || !present || !meta))) return fail(c, KT_ERR_INVALID, "null compact pod columns");
  if (val_bits < 1 || val_bits > 31) return fail(c, KT_ERR_INVALID, "val_bits %d outside 1..31", val_bits);
  const int L = c->lim.label_slots, R = c->lim.n_resources, Lpad = (L + 7) & ~7;
  for (int r = 0; r < R; ++r)
    if (req_shift[r] < 0 || req_shift[r] > 32) return fail(c, KT_ERR_INVALID, "req_shift[%d] = %d outside 0..32", r, req_shift[r]);
  int rc = set_device(c);
  if (rc) return rc;
  PodStore& s = c->pods[kind];
  KT_CUDA(c, s.labels.reserve((size_t)Lpad * n * 8 + 16));
  KT_CUDA(c, s.req.reserve((size_t)R * n * 8 + 16));
  KT_CUDA(c, s.flags.reserve((size_t)n * 4 + 16));
  KT_CUDA(c, s.ns.reserve((size_t)n * 4 + 16));
  if ((rc = upload(c, s.c_labels, labels32, (size_t)L * n)) || (rc = upload(c, s.c_req, req32, (size_t)R * n)) ||
      (rc = upload(c, s.c_meta, meta, (size_t)n)) || (rc = upload(c, s.present, present, (size_t)n)))
    return rc;
  if (n > 0) {
    ReqShifts sh{};
    for (int r = 0; r < R; ++r) sh.s[r] = (unsigned char)req_shift[r];
    k_unpack_rows<<<(unsigned)((n + 255) / 256), 256, 0, c->stream>>>(n, L, Lpad, R, val_bits, s.c_labels.as<uint32_t>(), s.c_req.as<int32_t>(), sh,
                                                                      s.c_meta.as<uint32_t>(), s.labels.as<int64_t>(), s.req.as<int64_t>(),
                                                                      s.flags.as<uint32_t>(), s.ns.as<int32_t>());
    KT_CUDA(c, cudaGetLastError());
  }
  const bool cluster = choose_clustered(s, n, [&](int64_t i, int32_t* ns) { *ns = (int32_t)(meta[i] & 0x1fffffffu); return (meta[i] >> 29) != 0; });
  return finish_upload(c, kind, n, cluster, (int64_t)1 << 29, false);
}

static int upload_pods_packed_locked(kt_ctx* c, int kind, int64_t n, const kt_packed_pods* pk);
int kt_upload_pods_packed(kt_ctx* c, int kind, int64_t n, const kt_packed_pods* pk) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  return upload_pods_packed_locked(c, kind, n, pk);
}
static int upload_pods_packed_locked(kt_ctx* c, int kind, int64_t n, const kt_packed_pods* pk) {
  if (int rc = check_kind(c, "kt_upload_pods_packed", kind)) return rc;
  if (n < 0 || !pk || (n > 0 && (!pk->labels16 || !pk->meta))) return fail(c, KT_ERR_INVALID, "null packed pod columns");
  const bool coded = pk->req_codes != nullptr;
  if (coded ? (!pk->req_dict_off || !pk->req_code_bytes) : (!pk->req_shift || (n > 0 && !pk->req32)))
    return fail(c, KT_ERR_INVALID, "packed pod rows need either req32 + req_shift or req_codes + req_dict_off + req_code_bytes");
  const int L = c->lim.label_slots, R = c->lim.n_resources, Lpad = (L + 7) & ~7;
  ReqCodes rc{};
  size_t code_bytes = 0, dict_len = 0;
  if (coded) {
    for (int r = 0; r < R; ++r) {
      const int b = pk->req_code_bytes[r];
      const int64_t d0 = pk->req_dict_off[r], d1 = pk->req_dict_off[r + 1];
      if ((b != 1 && b != 2) || d0 < 0 || d1 < d0 || d1 - d0 > (b == 1 ? 256 : 65536)) return fail(c, KT_ERR_INVALID, "request dictionary of column %d is malformed", r);
      rc.col_off[r] = (uint32_t)code_bytes;
      rc.dict_off[r] = (uint32_t)d0;
      rc.dict_len[r] = (uint32_t)(d1 - d0);
      rc.bytes[r] = (unsigned char)b;
      code_bytes += ((size_t)n * (size_t)b + 3) & ~(size_t)3;
      if (code_bytes >= ((size_t)1 << 32)) return fail(c, KT_ERR_LIMIT, "request code columns exceed 4 GiB");
    }
    dict_len = (size_t)pk->req_dict_off[R];
    if (dict_len > 0 && !pk->req_dict) return fail(c, KT_ERR_INVALID, "null request dictionary");
  }
  if (pk->n_pairs < 0 || pk->n_pairs > 65535 || (pk->n_pairs > 0 && !pk->pairs)) return fail(c, KT_ERR_INVALID, "n_pairs %d outside 0..65535", pk->n_pairs);
  if (pk->ns_bits < 1 || pk->ns_bits + 3 + R > 32) return fail(c, KT_ERR_INVALID, "ns_bits %d: ns_bits + 3 + R must fit 32 bits", pk->ns_bits);
  if (!coded)
    for (int r = 0; r < R; ++r)
      if (pk->req_shift[r] < 0 || pk->req_shift[r] > 32) return fail(c, KT_ERR_INVALID, "req_shift[%d] = %d outside 0..32", r, pk->req_shift[r]);
  int err = set_device(c);
  if (err) return err;
  PodStore& s = c->pods[kind];
  const uint32_t ns_mask = (1u << pk->ns_bits) - 1u;
  const bool cluster = choose_clustered(s, n, [&](int64_t i, int32_t* ns) {
    const uint32_t m = pk->meta[i];
    *ns = (int32_t)(m & ns_mask);
    return ((m >> pk->ns_bits) & 7u) != 0;
  });
  // with tables in place the rows are translated (labels -> table row offsets, namespace -> word info) in the unpacking
  // kernel: one launch and one read of the labels less per upload (rows laid out by namespace are translated after the move)
  const bool fuse = n > 0 && c->have_throttles && !cluster;
  KT_CUDA(c, s.labels.reserve((size_t)Lpad * n * 8 + 16));
  KT_CUDA(c, s.req.reserve((size_t)R * n * 8 + 16));
  KT_CUDA(c, s.present.reserve((size_t)n * 4 + 16));
  KT_CUDA(c, s.flags.reserve((size_t)n * 4 + 16));
  KT_CUDA(c, s.ns.reserve((size_t)n * 4 + 16));
  // The columns a caller carved out of ONE pinned block (bench.py, a Go packer with one arena per snapshot) cross the link as
  // one transfer: five copies of a few hundred KB each cost more in per-copy latency than their bytes.  Detected, not declared:
  // the device-bound arrays span little more than their own size, inside one block from kt_host_alloc / kt_host_alloc_upload
  // (arrays in separate pinned allocations can be neighbours too, and no copy may span two allocations).
  const void* h_ptr[5] = {pk->labels16, pk->pairs, pk->meta, coded ? (const void*)pk->req_codes : (const void*)pk->req32, coded ? (const void*)pk->req_dict : nullptr};
  const size_t h_len[5] = {(size_t)L * n * 2, (size_t)pk->n_pairs * 8, (size_t)n * 4, coded ? code_bytes : (size_t)R * n * 4, coded ? dict_len * 8 : 0};
  uintptr_t lo = UINTPTR_MAX, hi = 0;
  size_t sum = 0;
  for (int i = 0; i < 5; ++i)
    if (h_len[i]) {
      lo = std::min(lo, (uintptr_t)h_ptr[i]);
      hi = std::max(hi, (uintptr_t)h_ptr[i] + h_len[i]);
      sum += h_len[i];
    }
  const bool one_block = n > 0 && sum > 0 && (lo & 15) == 0 && hi - lo <= sum + 2048 && in_one_host_block(lo, hi);
  const uint16_t* d_labels16;
  const int64_t* d_pairs;
  const uint32_t* d_meta;
  const void* d_req;
  if (one_block) {
    KT_CUDA(c, s.c_labels.reserve(hi - lo + 16));
    KT_CUDA(c, cudaMemcpyAsync(s.c_labels.p, (const void*)lo, hi - lo, cudaMemcpyHostToDevice, c->stream));
    const unsigned char* base = s.c_labels.as<unsigned char>();
    auto dev = [&](const void* h) { return h ? (const void*)(base + ((uintptr_t)h - lo)) : nullptr; };
    d_labels16 = (const uint16_t*)dev(pk->labels16);
    d_pairs = (const int64_t*)dev(pk->pairs);
    d_meta = (const uint32_t*)dev(pk->meta);
    d_req = dev(h_ptr[3]);
    if (coded) {
      rc.codes = (const unsigned char*)d_req;
      rc.dict = (const int64_t*)dev(pk->req_dict);
    }
  } else {
    // labels16 travels through the 32-bit staging buffer of the compact format (half of it is used)
    KT_CUDA(c, s.c_labels.reserve((size_t)L * n * 2 + 16));
    if (n > 0) KT_CUDA(c, cudaMemcpyAsync(s.c_labels.p, pk->labels16, (size_t)L * n * 2, cudaMemcpyHostToDevice, c->stream));
    if ((err = upload(c, s.c_pairs, pk->pairs, (size_t)pk->n_pairs)) || (err = upload(c, s.c_meta, pk->meta, (size_t)n))) return err;
    if (coded) {
      if ((err = upload(c, s.c_req, pk->req_codes, code_bytes)) || (err = upload(c, s.c_dict, pk->req_dict, dict_len))) return err;
      rc.codes = s.c_req.as<unsigned char>();
      rc.dict = s.c_dict.as<int64_t>();
    } else if ((err = upload(c, s.c_req, pk->req32, (size_t)R * n))) {
      return err;
    }
    d_labels16 = s.c_labels.as<uint16_t>();
    d_pairs = s.c_pairs.as<int64_t>();
    d_meta = s.c_meta.as<uint32_t>();
    d_req = s.c_req.p;
  }
  if (n > 0) {
    ReqShifts sh{};
    if (!coded)
      for (int r = 0; r < R; ++r) sh.s[r] = (unsigned char)pk->req_shift[r];
    if (fuse) {
      KT_CUDA(c, s.roff.reserve((size_t)Lpad * n * 4 + 16));
      KT_CUDA(c, s.winfo.reserve((size_t)n * 4 + 16));
    }
    k_unpack_packed<<<(unsigned)((n + 255) / 256), 256, 0, c->stream>>>(n, L, Lpad, R, pk->ns_bits, pk->n_pairs, d_pairs, d_labels16,
                                                                        (const int32_t*)d_req, sh, rc, d_meta, s.labels.as<int64_t>(),
                                                                        s.req.as<int64_t>(), s.present.as<uint32_t>(), s.flags.as<uint32_t>(), s.ns.as<int32_t>(),
                                                                        fuse ? 1 : 0, fuse ? table_view(c) : TableView{}, s.roff.as<uint32_t>(), s.winfo.as<uint32_t>());
    KT_CUDA(c, cudaGetLastError());
  }
  return finish_upload(c, kind, n, cluster, (int64_t)1 << pk->ns_bits, fuse);
}

int kt_update_pod_rows(kt_ctx* c, int kind, int64_t k, const int64_t* rows, const int64_t* labels, const int64_t* req,
                       const uint32_t* present, const uint32_t* flags, const int32_t* ns_id) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (int rc = check_kind(c, __func__, kind)) return rc;
  if (k < 0 || (k > 0 && (!rows || !labels || !req || !present || !flags || !ns_id))) return fail(c, KT_ERR_INVALID, "null delta columns");
  if (k == 0) return KT_OK;
  PodStore& s = c->pods[kind];
  if (int rc = check_rows(c, __func__, k, rows, s.n)) return rc;
  int rc = set_device(c);
  if (rc) return rc;
  const int L = c->lim.label_slots, R = c->lim.n_resources;
  // grow-only staging buffers: an informer event must not cost a cudaMalloc/cudaFree pair.  The layout stays: the rows land
  // where the listed caller rows live.
  if ((rc = stage_rows(c, s, s.t_rows, k, rows)) || (rc = upload(c, s.t_labels, labels, (size_t)L * k)) || (rc = upload(c, s.t_req, req, (size_t)R * k)) ||
      (rc = upload(c, s.t_present, present, (size_t)k)) || (rc = upload(c, s.t_flags, flags, (size_t)k)) || (rc = upload(c, s.t_ns, ns_id, (size_t)k)))
    return rc;
  k_scatter_rows<<<(unsigned)((k + 255) / 256), 256, 0, c->stream>>>(k, s.t_rows.as<int64_t>(), L, R, s.n, s.t_labels.as<int64_t>(), s.t_req.as<int64_t>(),
                                                                     s.t_present.as<uint32_t>(), s.t_flags.as<uint32_t>(), s.t_ns.as<int32_t>(),
                                                                     s.labels.as<int64_t>(), s.req.as<int64_t>(), s.present.as<uint32_t>(),
                                                                     s.flags.as<uint32_t>(), s.ns.as<int32_t>());
  KT_CUDA(c, cudaGetLastError());
  // the delta keeps the store's row offsets current: only the scattered rows are translated again (same stream, after the scatter)
  if (s.roff_valid && (rc = translate_rows(c, s, k, s.t_rows.as<int64_t>()))) return rc;
  s.bitmap_clean = false;  // a row that changed namespace (or stopped being counted) leaves words behind: the next pass zero-fills
  KT_CUDA(c, cudaStreamSynchronize(c->stream));  // the caller may reuse its buffers as soon as we return
  c->evaluated = false;
  return KT_OK;
}

namespace {
// The namespace side of the selector spec (NsSpecView, kt_nsrows.cuh) in one device block, after the tables of a throttle upload
// were compiled (term_unsat comes from there).  Read by kt_update_namespace_rows only.
int stage_ns_spec(kt_ctx* c) {
  const SelectorSpec& s = c->spec;
  const size_t M = (size_t)s.m, nt = s.term_flags.size(), nq = s.req_key.size(), nv = s.req_vals.size();
  std::vector<uint8_t> tf(nt);
  for (size_t i = 0; i < nt; ++i)
    tf[i] = (uint8_t)((s.term_flags[i] & (KT_TERM_NS_INVALID | KT_TERM_POD_INVALID)) | (c->ht.term_unsat[i] ? kTermUnsat : 0));
  const struct {
    const void* p;
    size_t bytes;
  } part[8] = {{s.term_off.data(), (M + 1) * 4}, {s.ns_req_off.data(), s.ns_req_off.size() * 4}, {tf.data(), nt}, {s.req_key.data(), nq * 4},
               {s.req_op.data(), nq}, {s.req_val_off.data(), s.req_val_off.size() * 4}, {s.req_vals.data(), nv * 4}, {s.ns_id.data(), M * 4}};
  size_t total = 0;
  for (int i = 0; i < 8; ++i) {
    c->nsspec_at[i] = total;
    total += (part[i].bytes + 15) & ~(size_t)15;
  }
  c->h_nsspec.assign(total, 0);
  for (int i = 0; i < 8; ++i)
    if (part[i].bytes) std::memcpy(c->h_nsspec.data() + c->nsspec_at[i], part[i].p, part[i].bytes);
  return upload_vec(c, c->d_nsspec, c->h_nsspec);
}
NsSpecView ns_spec_view(const kt_ctx* c) {
  const unsigned char* b = c->d_nsspec.as<unsigned char>();
  NsSpecView v;
  v.term_off = reinterpret_cast<const int32_t*>(b + c->nsspec_at[0]); v.ns_req_off = reinterpret_cast<const int32_t*>(b + c->nsspec_at[1]);
  v.term_flags = b + c->nsspec_at[2]; v.req_key = reinterpret_cast<const uint32_t*>(b + c->nsspec_at[3]); v.req_op = b + c->nsspec_at[4];
  v.req_val_off = reinterpret_cast<const int32_t*>(b + c->nsspec_at[5]); v.req_vals = reinterpret_cast<const uint32_t*>(b + c->nsspec_at[6]);
  v.ns_id = reinterpret_cast<const int32_t*>(b + c->nsspec_at[7]);
  v.kind = c->d_kind.as<uint8_t>(); v.flags = c->d_tflags.as<uint8_t>();
  v.M = c->ht.M; v.W = c->ht.W; v.TPpad = c->ht.TPpad;
  return v;
}
}  // namespace

int kt_upload_namespaces(kt_ctx* c, int32_t n_ns, const int64_t* labels) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (n_ns < 0 || (n_ns > 0 && c->lim.ns_label_slots > 0 && !labels)) return fail(c, KT_ERR_INVALID, "null namespace labels");
  int rc = set_device(c);
  if (rc) return rc;
  c->n_ns = n_ns;
  c->ns_labels.assign(labels, labels + (size_t)c->lim.ns_label_slots * n_ns);
  c->evaluated = false;
  if (c->have_throttles) return recompile_tables(c);
  return KT_OK;
}

int kt_upload_throttles(kt_ctx* c, int32_t m, const kt_throttle_cols* cols, const kt_selector_table* sel) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  std::string e = copy_selector_spec(m, cols, sel, &c->spec);
  if (!e.empty()) return fail(c, KT_ERR_INVALID, "selector table: %s", e.c_str());
  if (m > 0 && (!cols->thr || !cols->thr_present || !cols->thr_cnt || !cols->ovr_off)) return fail(c, KT_ERR_INVALID, "null threshold columns");
  const int32_t n_ovr = m > 0 ? cols->ovr_off[m] : 0;
  if (m > 0 && (cols->ovr_off[0] != 0 || n_ovr != cols->n_ovr)) return fail(c, KT_ERR_INVALID, "ovr_off must span [0, n_ovr]");
  for (int32_t t = 0; t < m; ++t)
    if (cols->ovr_off[t] > cols->ovr_off[t + 1]) return fail(c, KT_ERR_INVALID, "ovr_off not monotone");
  if (n_ovr > 0 && (!cols->ovr_begin || !cols->ovr_end || !cols->ovr_flags || !cols->ovr_thr || !cols->ovr_present || !cols->ovr_cnt))
    return fail(c, KT_ERR_INVALID, "null override columns");
  int rc = set_device(c);
  if (rc) return rc;
  const int R = c->lim.n_resources;
  c->M = m;
  c->n_ovr = n_ovr;
  if (m > 0) c->h_ovr_off.assign(cols->ovr_off, cols->ovr_off + m + 1);
  else c->h_ovr_off.assign(1, 0);
  if ((rc = upload(c, c->d_kind, cols->kind, (size_t)m)) || (rc = upload(c, c->d_tflags, cols->flags, (size_t)m)) ||
      (rc = upload(c, c->d_thr, cols->thr, (size_t)R * m)) || (rc = upload(c, c->d_thr_present, cols->thr_present, (size_t)m)) ||
      (rc = upload(c, c->d_thr_cnt, cols->thr_cnt, (size_t)m)) || (rc = upload(c, c->d_ovr_off, cols->ovr_off, (size_t)m + 1)) ||
      (rc = upload(c, c->d_ovr_begin, cols->ovr_begin, (size_t)n_ovr)) || (rc = upload(c, c->d_ovr_end, cols->ovr_end, (size_t)n_ovr)) ||
      (rc = upload(c, c->d_ovr_flags, cols->ovr_flags, (size_t)n_ovr)) || (rc = upload(c, c->d_ovr_thr, cols->ovr_thr, (size_t)R * n_ovr)) ||
      (rc = upload(c, c->d_ovr_present, cols->ovr_present, (size_t)n_ovr)) || (rc = upload(c, c->d_ovr_cnt, cols->ovr_cnt, (size_t)n_ovr)))
    return rc;
  // per-throttle pass state
  const size_t part_bytes = (size_t)(2 * R + 1) * m * sizeof(unsigned long long);
  c->part_stride = (part_bytes + 255) & ~(size_t)255;
  KT_CUDA(c, c->d_part.reserve(2 * c->part_stride + 16));
  KT_CUDA(c, cudaMemsetAsync(c->d_part.p, 0, c->d_part.cap, c->stream));
  c->part_parity = 0;
  c->win_stale = c->win != nullptr;  // laid out for the previous M
  c->pre_stride = (size_t)((m + 31) & ~31) * pre_record_bytes(R);  // whole 32-throttle words: a decide slot is staged as one block
  KT_CUDA(c, c->d_pre.reserve(2 * c->pre_stride + 16));
  KT_CUDA(c, c->d_changed.reserve(16 + (size_t)m * 5 + 16));
  KT_CUDA(c, cudaMemsetAsync(c->d_changed.p, 0, 16, c->stream));
  c->have_diff = false;
  const size_t out_bytes = status_layout(R, m).bytes;
  KT_CUDA(c, c->d_out.reserve(out_bytes + 16));
  KT_CUDA(c, c->h_call.reserve(out_bytes));  // kt_get_reconcile lands the block there
  c->have_throttles = true;
  c->have_status = false;
  c->have_reserved = false;
  c->evaluated = false;
  c->have_codes = false;
  if ((rc = recompile_tables(c))) return rc;
  return stage_ns_spec(c);
}

int kt_upload_status(kt_ctx* c, const kt_status_cols* st) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_upload_status before kt_upload_throttles");
  if (!st || !st->calculated || !st->calc_thr || !st->calc_present || !st->calc_cnt || !st->used || !st->used_present || !st->used_cnt ||
      !st->throttled)
    return fail(c, KT_ERR_INVALID, "null status columns");
  int rc = set_device(c);
  if (rc) return rc;
  const size_t m = (size_t)c->M, R = (size_t)c->lim.n_resources;
  if ((rc = upload(c, c->d_st_calculated, st->calculated, m)) || (rc = upload(c, c->d_st_calc_thr, st->calc_thr, R * m)) ||
      (rc = upload(c, c->d_st_calc_present, st->calc_present, m)) || (rc = upload(c, c->d_st_calc_cnt, st->calc_cnt, m)) ||
      (rc = upload(c, c->d_st_used, st->used, R * m)) || (rc = upload(c, c->d_st_used_present, st->used_present, m)) ||
      (rc = upload(c, c->d_st_used_cnt, st->used_cnt, m)) || (rc = upload(c, c->d_st_throttled, st->throttled, m)))
    return rc;
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  c->have_status = true;
  c->evaluated = false;
  return KT_OK;
}

int kt_set_reserved(kt_ctx* c, const int64_t* reserved, const uint32_t* present, const int64_t* cnt) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_set_reserved before kt_upload_throttles");
  if (!reserved && !present && !cnt) { c->have_reserved = false; c->evaluated = false; return KT_OK; }
  if (!reserved || !present || !cnt) return fail(c, KT_ERR_INVALID, "reserved columns must be all set or all null");
  int rc = set_device(c);
  if (rc) return rc;
  const size_t m = (size_t)c->M, R = (size_t)c->lim.n_resources;
  if ((rc = upload(c, c->d_reserved, reserved, R * m)) || (rc = upload(c, c->d_reserved_present, present, m)) ||
      (rc = upload(c, c->d_reserved_cnt, cnt, m)))
    return rc;
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  c->have_reserved = true;
  c->evaluated = false;
  return KT_OK;
}

// ---- throttle-side column deltas ------------------------------------------------------------------------------------
namespace {
// k listed throttle columns: in [0, M) and distinct (a scatter of two values into one column has no defined winner)
int check_distinct_throttles(kt_ctx* c, const char* call, int64_t k, const int32_t* idx) {
  if (int rc = check_throttles(c, call, k, idx)) return rc;
  std::vector<int32_t> s(idx, idx + k);
  std::sort(s.begin(), s.end());
  auto d = std::adjacent_find(s.begin(), s.end());
  if (d != s.end()) return fail(c, KT_ERR_INVALID, "%s: throttle %d listed twice", call, *d);
  return KT_OK;
}
// The listed columns in ONE host-to-device copy: the pieces packed back to back into the pinned call block (each padded to 16
// bytes), copied into d_call_in.  at[i] is piece i's offset there.
struct Piece {
  const void* src;
  size_t bytes;
};
int stage_pieces(kt_ctx* c, std::initializer_list<Piece> pieces, size_t* at) {
  size_t total = 0, i = 0;
  for (const Piece& p : pieces) {
    at[i++] = total;
    total += (p.bytes + 15) & ~(size_t)15;
  }
  KT_CUDA(c, c->h_call.reserve(total));
  KT_CUDA(c, c->d_call_in.reserve(total + 16));
  i = 0;
  for (const Piece& p : pieces) {
    if (p.bytes) std::memcpy(c->h_call.as<unsigned char>() + at[i], p.src, p.bytes);
    ++i;
  }
  KT_CUDA(c, cudaMemcpyAsync(c->d_call_in.p, c->h_call.p, total, cudaMemcpyHostToDevice, c->stream));
  return KT_OK;
}
}  // namespace

int kt_update_status_rows(kt_ctx* c, int64_t k, const int32_t* idx, const kt_status_cols* st) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (k < 0) return fail(c, KT_ERR_INVALID, "kt_update_status_rows: k = %lld", (long long)k);
  if (k > 0 && (!idx || !st || !st->calculated || !st->calc_thr || !st->calc_present || !st->calc_cnt || !st->used || !st->used_present ||
                !st->used_cnt || !st->throttled))
    return fail(c, KT_ERR_INVALID, "kt_update_status_rows: null column with k = %lld", (long long)k);
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_update_status_rows before kt_upload_throttles");
  if (!c->have_status) return fail(c, KT_ERR_STATE, "kt_update_status_rows replaces columns of an uploaded status: kt_upload_status first");
  if (k == 0) return KT_OK;
  if (int rc = check_distinct_throttles(c, __func__, k, idx)) return rc;
  int rc = set_device(c);
  if (rc) return rc;
  const int R = c->lim.n_resources, M = c->M;
  const size_t K = (size_t)k, res = (size_t)R * K * 8;
  size_t at[9];
  if ((rc = stage_pieces(c, {{idx, K * 4}, {st->calculated, K}, {st->calc_thr, res}, {st->calc_present, K * 4}, {st->calc_cnt, K * 8},
                             {st->used, res}, {st->used_present, K * 4}, {st->used_cnt, K * 8}, {st->throttled, K * 4}}, at)))
    return rc;
  const unsigned char* in = c->d_call_in.as<unsigned char>();
  StatusScatter src;
  src.calculated = in + at[1]; src.calc_thr = reinterpret_cast<const int64_t*>(in + at[2]);
  src.calc_present = reinterpret_cast<const uint32_t*>(in + at[3]); src.calc_cnt = reinterpret_cast<const int64_t*>(in + at[4]);
  src.used = reinterpret_cast<const int64_t*>(in + at[5]); src.used_present = reinterpret_cast<const uint32_t*>(in + at[6]);
  src.used_cnt = reinterpret_cast<const int64_t*>(in + at[7]); src.throttled = reinterpret_cast<const uint32_t*>(in + at[8]);
  k_scatter_status<<<(unsigned)((k + 127) / 128), 128, 0, c->stream>>>(
      k, reinterpret_cast<const int32_t*>(in + at[0]), R, M, src, c->d_st_calculated.as<uint8_t>(), c->d_st_calc_thr.as<int64_t>(),
      c->d_st_calc_present.as<uint32_t>(), c->d_st_calc_cnt.as<int64_t>(), c->d_st_used.as<int64_t>(), c->d_st_used_present.as<uint32_t>(),
      c->d_st_used_cnt.as<int64_t>(), c->d_st_throttled.as<uint32_t>());
  KT_CUDA(c, cudaGetLastError());
  KT_CUDA(c, cudaStreamSynchronize(c->stream));  // the caller may reuse its buffers as soon as we return
  c->evaluated = false;
  return KT_OK;
}

int kt_update_reserved_rows(kt_ctx* c, int64_t k, const int32_t* idx, const int64_t* reserved, const uint32_t* present, const int64_t* cnt) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (k < 0) return fail(c, KT_ERR_INVALID, "kt_update_reserved_rows: k = %lld", (long long)k);
  if (k > 0 && (!idx || !reserved || !present || !cnt)) return fail(c, KT_ERR_INVALID, "kt_update_reserved_rows: null column with k = %lld", (long long)k);
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_update_reserved_rows before kt_upload_throttles");
  if (k == 0) return KT_OK;
  if (int rc = check_distinct_throttles(c, __func__, k, idx)) return rc;
  int rc = set_device(c);
  if (rc) return rc;
  const int R = c->lim.n_resources, M = c->M;
  const size_t K = (size_t)k;
  if (!c->have_reserved) {  // nothing reserved so far (or the columns belong to an earlier throttle set): every other column is zero
    const size_t m = (size_t)M;
    KT_CUDA(c, c->d_reserved.reserve((size_t)R * m * 8 + 16));
    KT_CUDA(c, c->d_reserved_present.reserve(m * 4 + 16));
    KT_CUDA(c, c->d_reserved_cnt.reserve(m * 8 + 16));
    KT_CUDA(c, cudaMemsetAsync(c->d_reserved.p, 0, (size_t)R * m * 8, c->stream));
    KT_CUDA(c, cudaMemsetAsync(c->d_reserved_present.p, 0, m * 4, c->stream));
    KT_CUDA(c, cudaMemsetAsync(c->d_reserved_cnt.p, 0, m * 8, c->stream));
  }
  size_t at[4];
  if ((rc = stage_pieces(c, {{idx, K * 4}, {reserved, (size_t)R * K * 8}, {present, K * 4}, {cnt, K * 8}}, at))) return rc;
  const unsigned char* in = c->d_call_in.as<unsigned char>();
  k_scatter_reserved<<<(unsigned)((k + 127) / 128), 128, 0, c->stream>>>(
      k, reinterpret_cast<const int32_t*>(in + at[0]), R, M, reinterpret_cast<const int64_t*>(in + at[1]), reinterpret_cast<const uint32_t*>(in + at[2]),
      reinterpret_cast<const int64_t*>(in + at[3]), c->d_reserved.as<int64_t>(), c->d_reserved_present.as<uint32_t>(), c->d_reserved_cnt.as<int64_t>());
  KT_CUDA(c, cudaGetLastError());
  KT_CUDA(c, cudaStreamSynchronize(c->stream));  // the caller may reuse its buffers as soon as we return
  c->have_reserved = true;
  c->evaluated = false;
  return KT_OK;
}

int kt_update_threshold_rows(kt_ctx* c, int64_t k, const int32_t* idx, const kt_throttle_cols* cols) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (k < 0) return fail(c, KT_ERR_INVALID, "kt_update_threshold_rows: k = %lld", (long long)k);
  if (k > 0 && (!idx || !cols || !cols->thr || !cols->thr_present || !cols->thr_cnt || !cols->ovr_off))
    return fail(c, KT_ERR_INVALID, "kt_update_threshold_rows: null column with k = %lld", (long long)k);
  if (cols && (cols->kind || cols->ns_id || cols->flags))
    return fail(c, KT_ERR_INVALID, "kt_update_threshold_rows: kind, ns_id and flags feed the tables (kt_upload_throttles) and must be NULL");
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_update_threshold_rows before kt_upload_throttles");
  if (k == 0) return KT_OK;
  if (int rc = check_distinct_throttles(c, __func__, k, idx)) return rc;
  const int32_t* in_off = cols->ovr_off;
  const int32_t n_in = in_off[k];
  if (in_off[0] != 0 || n_in != cols->n_ovr) return fail(c, KT_ERR_INVALID, "kt_update_threshold_rows: ovr_off must span [0, n_ovr]");
  for (int64_t i = 0; i < k; ++i)
    if (in_off[i] > in_off[i + 1]) return fail(c, KT_ERR_INVALID, "kt_update_threshold_rows: ovr_off not monotone");
  if (n_in > 0 && (!cols->ovr_begin || !cols->ovr_end || !cols->ovr_flags || !cols->ovr_thr || !cols->ovr_present || !cols->ovr_cnt))
    return fail(c, KT_ERR_INVALID, "kt_update_threshold_rows: null override columns");
  const int R = c->lim.n_resources, M = c->M;
  const std::vector<int32_t>& old_off = c->h_ovr_off;
  bool same_counts = true;
  for (int64_t i = 0; i < k && same_counts; ++i) same_counts = in_off[i + 1] - in_off[i] == old_off[(size_t)idx[i] + 1] - old_off[(size_t)idx[i]];
  // the new layout when some count changes: every column keeps its count but the listed ones
  std::vector<int32_t> new_off, sorted, pos;
  if (!same_counts) {
    std::vector<int64_t> cnt((size_t)M);
    for (int t = 0; t < M; ++t) cnt[(size_t)t] = old_off[(size_t)t + 1] - old_off[(size_t)t];
    for (int64_t i = 0; i < k; ++i) cnt[(size_t)idx[i]] = in_off[i + 1] - in_off[i];
    new_off.assign((size_t)M + 1, 0);
    int64_t run = 0;
    for (int t = 0; t < M; ++t) {
      run += cnt[(size_t)t];
      if (run > INT32_MAX) return fail(c, KT_ERR_INVALID, "kt_update_threshold_rows: more than 2^31-1 overrides");
      new_off[(size_t)t + 1] = (int32_t)run;
    }
    std::vector<std::pair<int32_t, int32_t>> by_col((size_t)k);
    for (int64_t i = 0; i < k; ++i) by_col[(size_t)i] = {idx[i], (int32_t)i};
    std::sort(by_col.begin(), by_col.end());
    for (auto& p : by_col) { sorted.push_back(p.first); pos.push_back(p.second); }
  }
  int rc = set_device(c);
  if (rc) return rc;
  const size_t K = (size_t)k, N = (size_t)n_in;
  size_t at[14];
  if ((rc = stage_pieces(c, {{idx, K * 4}, {cols->thr, (size_t)R * K * 8}, {cols->thr_present, K * 4}, {cols->thr_cnt, K * 8}, {in_off, (K + 1) * 4},
                             {cols->ovr_begin, N * 8}, {cols->ovr_end, N * 8}, {cols->ovr_flags, N}, {cols->ovr_thr, (size_t)R * N * 8},
                             {cols->ovr_present, N * 4}, {cols->ovr_cnt, N * 8}, {new_off.data(), new_off.size() * 4}, {sorted.data(), sorted.size() * 4},
                             {pos.data(), pos.size() * 4}}, at)))
    return rc;
  OverrideCols src{staged<int64_t>(c, at[5]), staged<int64_t>(c, at[6]), staged<uint8_t>(c, at[7]), staged<int64_t>(c, at[8]),
                   staged<uint32_t>(c, at[9]), staged<int64_t>(c, at[10]), n_in};
  OverrideOut resident{c->d_ovr_begin.as<int64_t>(), c->d_ovr_end.as<int64_t>(), c->d_ovr_flags.as<uint8_t>(), c->d_ovr_thr.as<int64_t>(),
                       c->d_ovr_present.as<uint32_t>(), c->d_ovr_cnt.as<int64_t>(), c->n_ovr};
  k_scatter_thresholds<<<(unsigned)((k + 127) / 128), 128, 0, c->stream>>>(
      k, staged<int32_t>(c, at[0]), R, M, staged<int64_t>(c, at[1]), staged<uint32_t>(c, at[2]), staged<int64_t>(c, at[3]),
      staged<int32_t>(c, at[4]), src, c->d_ovr_off.as<int32_t>(), same_counts, c->d_thr.as<int64_t>(), c->d_thr_present.as<uint32_t>(),
      c->d_thr_cnt.as<int64_t>(), resident);
  KT_CUDA(c, cudaGetLastError());
  if (!same_counts) {
    const int32_t n_new = new_off[(size_t)M];
    const size_t n = (size_t)n_new;
    KT_CUDA(c, c->s_ovr_off.reserve(((size_t)M + 1) * 4 + 16));
    KT_CUDA(c, c->s_ovr_begin.reserve(n * 8 + 16));
    KT_CUDA(c, c->s_ovr_end.reserve(n * 8 + 16));
    KT_CUDA(c, c->s_ovr_flags.reserve(n + 16));
    KT_CUDA(c, c->s_ovr_thr.reserve((size_t)R * n * 8 + 16));
    KT_CUDA(c, c->s_ovr_present.reserve(n * 4 + 16));
    KT_CUDA(c, c->s_ovr_cnt.reserve(n * 8 + 16));
    const OverrideCols old{resident.begin, resident.end, resident.flags, resident.thr, resident.present, resident.cnt, resident.n};
    const OverrideOut out{c->s_ovr_begin.as<int64_t>(), c->s_ovr_end.as<int64_t>(), c->s_ovr_flags.as<uint8_t>(), c->s_ovr_thr.as<int64_t>(),
                          c->s_ovr_present.as<uint32_t>(), c->s_ovr_cnt.as<int64_t>(), n_new};
    k_rebuild_overrides<<<(unsigned)((M + 1 + 127) / 128), 128, 0, c->stream>>>(
        M, R, k, staged<int32_t>(c, at[12]), staged<int32_t>(c, at[13]), staged<int32_t>(c, at[11]), c->d_ovr_off.as<int32_t>(), old,
        staged<int32_t>(c, at[4]), src, c->s_ovr_off.as<int32_t>(), out, nullptr);
    KT_CUDA(c, cudaGetLastError());
    std::swap(c->d_ovr_off, c->s_ovr_off); std::swap(c->d_ovr_begin, c->s_ovr_begin); std::swap(c->d_ovr_end, c->s_ovr_end);
    std::swap(c->d_ovr_flags, c->s_ovr_flags); std::swap(c->d_ovr_thr, c->s_ovr_thr); std::swap(c->d_ovr_present, c->s_ovr_present);
    std::swap(c->d_ovr_cnt, c->s_ovr_cnt);
    c->n_ovr = n_new;
    c->h_ovr_off.swap(new_off);
  }
  KT_CUDA(c, cudaStreamSynchronize(c->stream));  // the caller may reuse its buffers as soon as we return
  // as after kt_upload_throttles: a pass is needed again before the getters that read one (status and reservations are kept)
  c->evaluated = false;
  c->have_codes = false;
  c->have_diff = false;
  return KT_OK;
}

// ---- namespace row deltas (kt_nsrows.cuh) ---------------------------------------------------------------------------
namespace {
// After some nsmask entries changed on the device: the word lists of all NS namespaces rebuilt from nsmask (the caller reserved
// d_nsw_off, d_nsw_idx and d_call_out for NS), the words inlined with the resident pod rows refreshed, and the total and the
// longest list brought back through the call block at res_at with the call's one synchronisation.
int rebuild_ns_words(kt_ctx* c, int32_t NS, size_t res_at) {
  const int32_t W = c->ht.W, TPpad = c->ht.TPpad;
  int32_t* out = c->d_call_out.as<int32_t>();  // {total, longest list, -, -}, then cnt[NS]
  const unsigned ns_blocks = (unsigned)((NS + 7) / 8);
  if (NS > 0) {
    k_ns_count<<<ns_blocks, 256, 0, c->stream>>>(NS, W, TPpad, c->d_nsmask.as<uint32_t>(), out + 4);
    KT_CUDA(c, cudaGetLastError());
  }
  k_ns_scan<<<1, kNsScanThreads, 0, c->stream>>>(NS, out + 4, c->d_nsw_off.as<int32_t>(), out);
  KT_CUDA(c, cudaGetLastError());
  if (NS > 0) {
    k_ns_fill<<<ns_blocks, 256, 0, c->stream>>>(NS, W, TPpad, c->d_nsmask.as<uint32_t>(), c->d_nsw_off.as<int32_t>(), c->d_nsw_idx.as<int32_t>());
    KT_CUDA(c, cudaGetLastError());
  }
  c->ht.NS = NS;
  for (auto& s : c->pods) {  // the row offsets stay valid (the pod-label tables keep their rows); the inlined words may not
    if (s.roff_valid && s.n > 0) {
      k_ns_winfo<<<(unsigned)((s.n + 255) / 256), 256, 0, c->stream>>>(s.n, table_view(c), s.ns.as<int32_t>(), s.winfo.as<uint32_t>());
      KT_CUDA(c, cudaGetLastError());
    }
    s.bitmap_clean = false;  // the word lists changed
  }
  int32_t* res = reinterpret_cast<int32_t*>(c->h_call.as<unsigned char>() + res_at);
  KT_CUDA(c, cudaMemcpyAsync(res, out, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));  // the caller may reuse its buffers; the pass plan needs the longest list
  c->nsw_total = res[0];
  c->ht.max_ns_words = res[1];
  return KT_OK;
}
}  // namespace

int kt_update_namespace_rows(kt_ctx* c, int32_t n_ns, int64_t k, const int32_t* idx, const int64_t* labels) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  const int LN = c->lim.ns_label_slots;
  if (k < 0) return fail(c, KT_ERR_INVALID, "kt_update_namespace_rows: k = %lld", (long long)k);
  if (k > 0 && (!idx || (LN > 0 && !labels))) return fail(c, KT_ERR_INVALID, "kt_update_namespace_rows: null column with k = %lld", (long long)k);
  if (n_ns < c->n_ns) return fail(c, KT_ERR_INVALID, "kt_update_namespace_rows: n_ns %d < %d (namespace rows are never removed)", n_ns, c->n_ns);
  for (int64_t i = 0; i < k; ++i)
    if (idx[i] < 0 || idx[i] >= n_ns) return fail(c, KT_ERR_INVALID, "kt_update_namespace_rows: namespace %d out of range [0,%d)", idx[i], n_ns);
  {
    std::vector<int32_t> s(idx, idx + k);
    std::sort(s.begin(), s.end());
    auto d = std::adjacent_find(s.begin(), s.end());
    if (d != s.end()) return fail(c, KT_ERR_INVALID, "kt_update_namespace_rows: namespace %d listed twice", *d);
  }
  const int32_t old_n = c->n_ns;
  if (k == 0 && n_ns == old_n) return KT_OK;
  // the stored rows, as kt_upload_namespaces would hold them: [LN][n_ns], rows the count grew by label-less
  if (n_ns != old_n) {
    std::vector<int64_t> grown((size_t)LN * n_ns, KT_LABEL_EMPTY);
    for (int s = 0; s < LN; ++s)
      std::copy(c->ns_labels.begin() + (size_t)s * old_n, c->ns_labels.begin() + (size_t)(s + 1) * old_n, grown.begin() + (size_t)s * n_ns);
    c->ns_labels.swap(grown);
  }
  for (int64_t i = 0; i < k; ++i)
    for (int s = 0; s < LN; ++s) c->ns_labels[(size_t)s * n_ns + idx[i]] = labels[(size_t)s * k + i];
  c->n_ns = n_ns;
  c->evaluated = false;
  if (!c->have_throttles) return KT_OK;  // the next kt_upload_throttles compiles these rows
  int rc = set_device(c);
  if (rc) return rc;
  // the rows to evaluate: the listed ones and the unlisted ones the count grew by
  std::vector<int32_t> rows(idx, idx + k);
  {
    std::vector<char> listed((size_t)(n_ns - old_n), 0);
    for (int64_t i = 0; i < k; ++i)
      if (idx[i] >= old_n) listed[(size_t)(idx[i] - old_n)] = 1;
    for (int32_t ns = old_n; ns < n_ns; ++ns)
      if (!listed[(size_t)(ns - old_n)]) rows.push_back(ns);
  }
  const int32_t kd = (int32_t)rows.size();
  std::vector<int64_t> lab((size_t)LN * kd);
  for (int s = 0; s < LN; ++s)
    for (int32_t i = 0; i < kd; ++i) lab[(size_t)s * kd + i] = c->ns_labels[(size_t)s * n_ns + rows[(size_t)i]];
  const int32_t W = c->ht.W, TPpad = c->ht.TPpad, old_NS = c->ht.NS, NS = std::max(n_ns, old_NS);
  const size_t row_bytes = (size_t)W * TPpad * 4;
  const size_t cap_rows = c->d_nsmask.cap > 16 ? (c->d_nsmask.cap - 16) / row_bytes : 0;
  if ((size_t)NS > cap_rows) {  // grow by doubling; the rows above old_NS are all evaluated below
    DevBuf grown;
    KT_CUDA(c, grown.reserve(std::max<size_t>((size_t)NS, 2 * (size_t)old_NS) * row_bytes + 16));
    if (old_NS > 0) KT_CUDA(c, cudaMemcpyAsync(grown.p, c->d_nsmask.p, (size_t)old_NS * row_bytes, cudaMemcpyDeviceToDevice, c->stream));
    std::swap(c->d_nsmask, grown);
    grown.release();
  }
  KT_CUDA(c, c->d_nsw_off.reserve(((size_t)NS + 1) * 4 + 16));
  // unchanged rows keep their counts, an evaluated row has at most W words
  KT_CUDA(c, c->d_nsw_idx.reserve(std::min((size_t)NS * W, (size_t)c->nsw_total + (size_t)kd * W) * 4 + 16));
  KT_CUDA(c, c->d_call_out.reserve(((size_t)NS + 4) * 4 + 16));
  static const int32_t result_slot[4] = {};
  size_t at[3];
  if ((rc = stage_pieces(c, {{rows.data(), (size_t)kd * 4}, {lab.data(), lab.size() * 8}, {result_slot, sizeof result_slot}}, at))) return rc;
  const unsigned char* in = c->d_call_in.as<unsigned char>();
  const NsSpecView sp = ns_spec_view(c);
  for (int32_t y0 = 0; y0 < kd; y0 += 65535) {
    const dim3 grid((unsigned)((W + 7) / 8), (unsigned)std::min(kd - y0, 65535));
    k_ns_rows<<<grid, 256, 0, c->stream>>>(sp, y0, kd, reinterpret_cast<const int32_t*>(in + at[0]), reinterpret_cast<const int64_t*>(in + at[1]), LN,
                                           n_ns, c->d_nsmask.as<uint32_t>());
    KT_CUDA(c, cudaGetLastError());
  }
  return rebuild_ns_words(c, NS, at[2]);
}

// ---- selector column deltas (kt_tables.cc patch_columns, kt_nsrows.cuh k_ns_cols) --------------------------------------
namespace {
// The spec of m columns with column idx[i] taking column i of d (kind, ns_id, flags and terms), the others old column base[t]
// -- or, without base, old column t: every column at or above old.m is then listed.  base[t] == -1 makes an empty column
// (ClusterThrottle, ns_id -1, flags 0, no terms).  The CSR is laid out again column by column: every term's podSelector
// requirements first, then every term's namespaceSelector ones.
SelectorSpec splice_spec(const SelectorSpec& old, int64_t k, const int32_t* idx, const SelectorSpec& d, int32_t m, const int32_t* base = nullptr) {
  const int32_t M = m;
  std::vector<int32_t> from((size_t)M, -1);
  for (int64_t i = 0; i < k; ++i) from[(size_t)idx[i]] = (int32_t)i;
  SelectorSpec s;
  s.m = M;
  s.kind.assign((size_t)M, KT_KIND_CLUSTERTHROTTLE); s.flags.assign((size_t)M, 0); s.ns_id.assign((size_t)M, -1);
  s.term_off.assign(1, 0);
  std::vector<std::pair<const SelectorSpec*, int32_t>> terms;  // (source, term) in the new order
  for (int32_t t = 0; t < M; ++t) {
    const int32_t i = from[(size_t)t];
    const SelectorSpec& src = i >= 0 ? d : old;
    const int32_t col = i >= 0 ? i : base ? base[t] : t;
    if (col < 0 || col >= src.m) {
      s.term_off.push_back((int32_t)terms.size());
      continue;
    }
    s.kind[(size_t)t] = src.kind[(size_t)col]; s.flags[(size_t)t] = src.flags[(size_t)col]; s.ns_id[(size_t)t] = src.ns_id[(size_t)col];
    for (int32_t term = src.term_off[(size_t)col]; term < src.term_off[(size_t)col + 1]; ++term) {
      terms.emplace_back(&src, term);
      s.term_flags.push_back(src.term_flags[(size_t)term]);
    }
    s.term_off.push_back((int32_t)terms.size());
  }
  s.req_val_off.assign(1, 0);
  auto push_reqs = [&](const SelectorSpec& src, int32_t q0, int32_t q1) {
    for (int32_t q = q0; q < q1; ++q) {
      s.req_key.push_back(src.req_key[(size_t)q]);
      s.req_op.push_back(src.req_op[(size_t)q]);
      s.req_vals.insert(s.req_vals.end(), src.req_vals.begin() + src.req_val_off[(size_t)q], src.req_vals.begin() + src.req_val_off[(size_t)q + 1]);
      s.req_val_off.push_back((int32_t)s.req_vals.size());
    }
  };
  s.pod_req_off.assign(1, 0);
  for (auto& st : terms) {
    push_reqs(*st.first, st.first->pod_req_off[(size_t)st.second], st.first->pod_req_off[(size_t)st.second + 1]);
    s.pod_req_off.push_back((int32_t)s.req_key.size());
  }
  s.ns_req_off.assign(1, (int32_t)s.req_key.size());
  for (auto& st : terms) {
    push_reqs(*st.first, st.first->ns_req_off[(size_t)st.second], st.first->ns_req_off[(size_t)st.second + 1]);
    s.ns_req_off.push_back((int32_t)s.req_key.size());
  }
  return s;
}
}  // namespace

int kt_update_selector_rows(kt_ctx* c, int64_t k, const int32_t* idx, const kt_throttle_cols* cols, const kt_selector_table* sel,
                            int32_t* recompiled) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (recompiled) *recompiled = 0;
  if (k < 0) return fail(c, KT_ERR_INVALID, "kt_update_selector_rows: k = %lld", (long long)k);
  if (k > 0 && (!idx || !cols || !cols->kind || !cols->ns_id || !cols->flags || !sel || !sel->term_off))
    return fail(c, KT_ERR_INVALID, "kt_update_selector_rows: null column with k = %lld", (long long)k);
  if (cols && (cols->thr || cols->thr_present || cols->thr_cnt || cols->ovr_off || cols->ovr_begin || cols->ovr_end || cols->ovr_flags ||
               cols->ovr_thr || cols->ovr_present || cols->ovr_cnt))
    return fail(c, KT_ERR_INVALID, "kt_update_selector_rows: threshold and override columns (kt_update_threshold_rows) must be NULL");
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_update_selector_rows before kt_upload_throttles");
  if (k == 0) return KT_OK;
  if (int rc = check_distinct_throttles(c, __func__, k, idx)) return rc;
  SelectorSpec d;
  const std::string e = copy_selector_spec((int32_t)k, cols, sel, &d);
  if (!e.empty()) return fail(c, KT_ERR_INVALID, "kt_update_selector_rows: selector table: %s", e.c_str());
  SelectorSpec spec = splice_spec(c->spec, k, idx, d, c->spec.m);
  int rc = set_device(c);
  if (rc) return rc;
  const bool fits = patch_columns(c->lim, c->spec, spec, std::vector<int32_t>(idx, idx + k), &c->ht);
  c->spec = std::move(spec);
  // as after kt_upload_throttles: a pass is needed again before the getters that read one (status and reservations are kept)
  c->evaluated = false;
  c->have_codes = false;
  c->have_diff = false;
  const size_t K = (size_t)k;
  if (!fits) {  // the listed columns' kind and flags, then the tables compiled again from the patched spec (kt_upload_namespaces)
    size_t at[3];
    if ((rc = stage_pieces(c, {{idx, K * 4}, {cols->kind, K}, {cols->flags, K}}, at))) return rc;
    k_scatter_kind_flags<<<(unsigned)((k + 127) / 128), 128, 0, c->stream>>>(k, staged<int32_t>(c, at[0]), staged<uint8_t>(c, at[1]), staged<uint8_t>(c, at[2]),
                                                                           c->d_kind.as<uint8_t>(), c->d_tflags.as<uint8_t>());
    KT_CUDA(c, cudaGetLastError());
    if ((rc = recompile_tables(c)) || (rc = stage_ns_spec(c))) return rc;
    KT_CUDA(c, cudaStreamSynchronize(c->stream));
    if (recompiled) *recompiled = 1;
    return KT_OK;
  }
  // the 32-throttle words the listed columns live in, ascending, and their recompiled table and need slices
  std::vector<int32_t> words(idx, idx + k);
  for (int32_t& w : words) w >>= 5;
  std::sort(words.begin(), words.end());
  words.erase(std::unique(words.begin(), words.end()), words.end());
  const HostTables& h = c->ht;
  const size_t nw = words.size(), tlen = (size_t)h.rows * h.TPpad * 2, nlen = (size_t)h.TPpad * h.B;
  std::vector<uint32_t> tab(nw * tlen), nd(nw * nlen);
  for (size_t j = 0; j < nw; ++j) {
    std::copy(h.table.begin() + (size_t)words[j] * tlen, h.table.begin() + (size_t)(words[j] + 1) * tlen, tab.begin() + j * tlen);
    std::copy(h.need.begin() + (size_t)words[j] * nlen, h.need.begin() + (size_t)(words[j] + 1) * nlen, nd.begin() + j * nlen);
  }
  const int32_t NS = h.NS, W = h.W, LN = c->lim.ns_label_slots;
  KT_CUDA(c, c->d_nsw_off.reserve(((size_t)NS + 1) * 4 + 16));
  // the unlisted words keep their entries, a listed word is in at most every list
  KT_CUDA(c, c->d_nsw_idx.reserve(std::min((size_t)NS * W, (size_t)c->nsw_total + (size_t)NS * nw) * 4 + 16));
  KT_CUDA(c, c->d_call_out.reserve(((size_t)NS + 4) * 4 + 16));
  static const int32_t result_slot[4] = {};
  size_t at[8];
  if ((rc = stage_pieces(c, {{idx, K * 4}, {cols->kind, K}, {cols->flags, K}, {words.data(), nw * 4}, {tab.data(), tab.size() * 4},
                             {nd.data(), nd.size() * 4}, {c->ns_labels.data(), c->ns_labels.size() * 8}, {result_slot, sizeof result_slot}}, at)))
    return rc;
  k_scatter_kind_flags<<<(unsigned)((k + 127) / 128), 128, 0, c->stream>>>(k, staged<int32_t>(c, at[0]), staged<uint8_t>(c, at[1]), staged<uint8_t>(c, at[2]),
                                                                         c->d_kind.as<uint8_t>(), c->d_tflags.as<uint8_t>());
  KT_CUDA(c, cudaGetLastError());
  const unsigned tblocks = (unsigned)std::min<size_t>((nw * tlen + 255) / 256, 4096), nblocks = (unsigned)std::min<size_t>((nw * nlen + 255) / 256, 4096);
  k_scatter_words<<<tblocks, 256, 0, c->stream>>>((int64_t)nw, staged<int32_t>(c, at[3]), (int64_t)tlen, staged<uint32_t>(c, at[4]), c->d_table.as<uint32_t>());
  KT_CUDA(c, cudaGetLastError());
  k_scatter_words<<<nblocks, 256, 0, c->stream>>>((int64_t)nw, staged<int32_t>(c, at[3]), (int64_t)nlen, staged<uint32_t>(c, at[5]), c->d_need.as<uint32_t>());
  KT_CUDA(c, cudaGetLastError());
  if ((rc = stage_ns_spec(c))) return rc;  // term ranges, requirements and ns_id of the patched spec
  if (NS > 0) {
    k_ns_cols<<<(unsigned)(((int64_t)NS * (int64_t)nw + 7) / 8), 256, 0, c->stream>>>(ns_spec_view(c), NS, (int32_t)nw, staged<int32_t>(c, at[3]),
                                                                                       staged<int64_t>(c, at[6]), LN, c->n_ns, c->d_nsmask.as<uint32_t>());
    KT_CUDA(c, cudaGetLastError());
  }
  return rebuild_ns_words(c, NS, at[7]);
}

// ---- column appends (kt_tables.cc patch_columns, kt_nsrows.cuh k_widen_cols) ------------------------------------------
namespace {
// A resident per-throttle array an append widens: [rows][M] elements of esize bytes, swapped with its spare once widened.
struct AppendTarget {
  DevBuf* buf;
  int64_t rows;
  int32_t esize;
  int add;  // index of the staged piece holding its new columns [rows][k], or -1: the new columns are zero
};
// The spec's kind and flags and the threshold columns (new columns staged at pieces 0-4), then the status and the reservations
// when they are held (new columns zero: no calculatedAt, nothing used, nothing reserved).
std::vector<AppendTarget> append_targets(kt_ctx* c) {
  const int64_t R = c->lim.n_resources;
  std::vector<AppendTarget> v = {{&c->d_kind, 1, 1, 0}, {&c->d_tflags, 1, 1, 1}, {&c->d_thr, R, 8, 2}, {&c->d_thr_present, 1, 4, 3},
                                 {&c->d_thr_cnt, 1, 8, 4}};
  if (c->have_status)
    v.insert(v.end(), {{&c->d_st_calculated, 1, 1, -1}, {&c->d_st_calc_thr, R, 8, -1}, {&c->d_st_calc_present, 1, 4, -1},
                       {&c->d_st_calc_cnt, 1, 8, -1}, {&c->d_st_used, R, 8, -1}, {&c->d_st_used_present, 1, 4, -1},
                       {&c->d_st_used_cnt, 1, 8, -1}, {&c->d_st_throttled, 1, 4, -1}});
  if (c->have_reserved)
    v.insert(v.end(), {{&c->d_reserved, R, 8, -1}, {&c->d_reserved_present, 1, 4, -1}, {&c->d_reserved_cnt, 1, 8, -1}});
  return v;
}
// Reserve b for `bytes`, keeping its first `keep` bytes: a grown buffer replaces b and the old one goes to `old`, to be released
// once the stream has passed the copy.
int reserve_keep(kt_ctx* c, DevBuf& b, size_t bytes, size_t keep, DevBuf& old) {
  if (bytes <= b.cap) return KT_OK;
  DevBuf grown;
  KT_CUDA(c, grown.reserve(bytes));
  if (keep) KT_CUDA(c, cudaMemcpyAsync(grown.p, b.p, keep, cudaMemcpyDeviceToDevice, c->stream));
  std::swap(b, grown);
  std::swap(old, grown);
  return KT_OK;
}
}  // namespace

int kt_append_throttle_rows(kt_ctx* c, int64_t k, const kt_throttle_cols* cols, const kt_selector_table* sel, int32_t* recompiled) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (recompiled) *recompiled = 0;
  if (k < 0) return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: k = %lld", (long long)k);
  if (k > 0 && (!cols || !cols->kind || !cols->ns_id || !cols->flags || !cols->thr || !cols->thr_present || !cols->thr_cnt || !cols->ovr_off ||
                !sel || !sel->term_off))
    return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: null column with k = %lld", (long long)k);
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_append_throttle_rows before kt_upload_throttles");
  if (k == 0) return KT_OK;
  const int32_t M0 = c->M;
  if (k > (int64_t)INT32_MAX - M0) return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: more than 2^31-1 throttles");
  const int32_t* in_off = cols->ovr_off;
  const int32_t n_in = in_off[k];
  if (in_off[0] != 0 || n_in != cols->n_ovr) return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: ovr_off must span [0, n_ovr]");
  for (int64_t i = 0; i < k; ++i)
    if (in_off[i] > in_off[i + 1]) return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: ovr_off not monotone");
  if (n_in > 0 && (!cols->ovr_begin || !cols->ovr_end || !cols->ovr_flags || !cols->ovr_thr || !cols->ovr_present || !cols->ovr_cnt))
    return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: null override columns");
  if ((int64_t)c->n_ovr + n_in > INT32_MAX) return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: more than 2^31-1 overrides");
  SelectorSpec d;
  const std::string e = copy_selector_spec((int32_t)k, cols, sel, &d);
  if (!e.empty()) return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: selector table: %s", e.c_str());
  const int32_t M1 = M0 + (int32_t)k;
  std::vector<int32_t> idx((size_t)k), pos((size_t)k);
  for (int32_t i = 0; i < (int32_t)k; ++i) { idx[(size_t)i] = M0 + i; pos[(size_t)i] = i; }
  int rc = set_device(c);
  if (rc) return rc;
  const int32_t W0 = c->ht.W;
  SelectorSpec spec = splice_spec(c->spec, k, idx.data(), d, M1);
  const bool fits = patch_columns(c->lim, c->spec, spec, idx, &c->ht);
  c->spec = std::move(spec);
  // as after kt_upload_throttles: a pass is needed again before the getters that read one (status and reservations are kept)
  c->evaluated = false;
  c->have_codes = false;
  c->have_diff = false;
  const int R = c->lim.n_resources;
  const size_t K = (size_t)k, N = (size_t)n_in;
  // the override layout: the resident entries keep their offsets, the new columns' follow them
  std::vector<int32_t> new_off(c->h_ovr_off);
  new_off.resize((size_t)M1 + 1);
  for (int64_t i = 0; i < k; ++i) new_off[(size_t)M0 + 1 + i] = c->n_ovr + in_off[i + 1];
  const int32_t n_new = new_off[(size_t)M1];
  // pass state sized by M, as kt_upload_throttles reserves it
  const size_t part_bytes = (size_t)(2 * R + 1) * M1 * sizeof(unsigned long long);
  c->part_stride = (part_bytes + 255) & ~(size_t)255;
  KT_CUDA(c, c->d_part.reserve(2 * c->part_stride + 16));
  KT_CUDA(c, cudaMemsetAsync(c->d_part.p, 0, c->d_part.cap, c->stream));
  c->part_parity = 0;
  c->win_stale = c->win != nullptr;  // laid out for the previous M
  c->pre_stride = (size_t)((M1 + 31) & ~31) * pre_record_bytes(R);
  KT_CUDA(c, c->d_pre.reserve(2 * c->pre_stride + 16));
  KT_CUDA(c, c->d_changed.reserve(16 + (size_t)M1 * 5 + 16));
  KT_CUDA(c, cudaMemsetAsync(c->d_changed.p, 0, 16, c->stream));
  const size_t out_bytes = status_layout(R, M1).bytes;
  KT_CUDA(c, c->d_out.reserve(out_bytes + 16));
  KT_CUDA(c, c->h_call.reserve(out_bytes));  // (before the staged copy: a grown block would drop it)
  // the widened arrays' spare halves and the spare override set
  const std::vector<AppendTarget> tg = append_targets(c);
  for (size_t j = 0; j < tg.size(); ++j) KT_CUDA(c, c->w_spare[j].reserve((size_t)tg[j].rows * M1 * tg[j].esize + 16));
  KT_CUDA(c, c->s_ovr_off.reserve(((size_t)M1 + 1) * 4 + 16));
  KT_CUDA(c, c->s_ovr_begin.reserve((size_t)n_new * 8 + 16));
  KT_CUDA(c, c->s_ovr_end.reserve((size_t)n_new * 8 + 16));
  KT_CUDA(c, c->s_ovr_flags.reserve((size_t)n_new + 16));
  KT_CUDA(c, c->s_ovr_thr.reserve((size_t)R * n_new * 8 + 16));
  KT_CUDA(c, c->s_ovr_present.reserve((size_t)n_new * 4 + 16));
  KT_CUDA(c, c->s_ovr_cnt.reserve((size_t)n_new * 8 + 16));
  // In place: the words from the one the first new column lands in up to the new W are recompiled on the host and cross as
  // slices; when W grows, table and need grow (the existing words keep their place) and nsmask is restrided on the device.
  const HostTables& h = c->ht;
  const int32_t w0 = M0 >> 5, W1 = h.W, NS = h.NS, LN = c->lim.ns_label_slots;
  const size_t tlen = (size_t)h.rows * h.TPpad * 2, nlen = (size_t)h.TPpad * h.B, ns_row0 = (size_t)W0 * h.TPpad, ns_row1 = (size_t)W1 * h.TPpad;
  std::vector<int32_t> words;
  DevBuf old_table, old_need, old_nsmask;
  bool nsmask_widen = false;
  if (fits) {
    for (int32_t w = w0; w < W1; ++w) words.push_back(w);
    if ((rc = reserve_keep(c, c->d_table, (size_t)W1 * tlen * 4 + 16, (size_t)w0 * tlen * 4, old_table)) ||
        (rc = reserve_keep(c, c->d_need, (size_t)W1 * nlen * 4 + 16, (size_t)w0 * nlen * 4, old_need)))
      return rc;
    if (W1 > W0 && NS > 0) {
      nsmask_widen = true;
      std::swap(old_nsmask, c->d_nsmask);
      KT_CUDA(c, c->d_nsmask.reserve((size_t)NS * ns_row1 * 4 + 16));
    }
    KT_CUDA(c, c->d_nsw_off.reserve(((size_t)NS + 1) * 4 + 16));
    // the untouched words keep their entries, a touched word is in at most every list
    KT_CUDA(c, c->d_nsw_idx.reserve(std::min((size_t)NS * W1, (size_t)c->nsw_total + (size_t)NS * words.size()) * 4 + 16));
    KT_CUDA(c, c->d_call_out.reserve(((size_t)NS + 4) * 4 + 16));
  }
  const size_t nw = words.size();
  static const int32_t result_slot[4] = {};
  size_t at[20];
  if ((rc = stage_pieces(c, {{cols->kind, K}, {cols->flags, K}, {cols->thr, (size_t)R * K * 8}, {cols->thr_present, K * 4}, {cols->thr_cnt, K * 8},
                             {in_off, (K + 1) * 4}, {cols->ovr_begin, N * 8}, {cols->ovr_end, N * 8}, {cols->ovr_flags, N},
                             {cols->ovr_thr, (size_t)R * N * 8}, {cols->ovr_present, N * 4}, {cols->ovr_cnt, N * 8}, {new_off.data(), new_off.size() * 4},
                             {idx.data(), K * 4}, {pos.data(), K * 4}, {fits ? &h.table[(size_t)w0 * tlen] : nullptr, nw * tlen * 4},
                             {fits ? &h.need[(size_t)w0 * nlen] : nullptr, nw * nlen * 4}, {words.data(), nw * 4},
                             {c->ns_labels.data(), fits ? c->ns_labels.size() * 8 : 0}, {result_slot, sizeof result_slot}},
                            at)))
    return rc;
  // one launch restrides every widened array (and lands the table and need slices, and restrides nsmask, in place)
  WidenBatch wb{};
  int64_t widest = 0;
  auto add_array = [&](const void* src, const void* add, void* dst, int64_t rows, int64_t m_old, int64_t m_new, int32_t esize) {
    wb.a[wb.n++] = WidenArray{static_cast<const unsigned char*>(src), static_cast<const unsigned char*>(add), static_cast<unsigned char*>(dst),
                              rows, m_old, m_new, esize};
    widest = std::max(widest, rows * m_new);
  };
  for (size_t j = 0; j < tg.size(); ++j)
    add_array(tg[j].buf->p, tg[j].add >= 0 ? staged<unsigned char>(c, at[tg[j].add]) : nullptr, c->w_spare[j].p, tg[j].rows, M0, M1, tg[j].esize);
  if (fits) {  // the slices of words [w0, W1) over the table and need (reserve_keep kept the words below w0)
    add_array(nullptr, staged<unsigned char>(c, at[15]), c->d_table.as<uint32_t>() + (size_t)w0 * tlen, 1, 0, (int64_t)(nw * tlen), 4);
    add_array(nullptr, staged<unsigned char>(c, at[16]), c->d_need.as<uint32_t>() + (size_t)w0 * nlen, 1, 0, (int64_t)(nw * nlen), 4);
    if (nsmask_widen) add_array(old_nsmask.p, nullptr, c->d_nsmask.p, NS, (int64_t)ns_row0, (int64_t)ns_row1, 4);
  }
  const unsigned wblocks = (unsigned)std::min<int64_t>((widest + 255) / 256, 2048);
  k_widen_cols<<<dim3(std::max(wblocks, 1u), (unsigned)wb.n), 256, 0, c->stream>>>(wb);
  KT_CUDA(c, cudaGetLastError());
  for (size_t j = 0; j < tg.size(); ++j) std::swap(*tg[j].buf, c->w_spare[j]);
  // the override columns rebuilt into the spare set, the new columns' entries appended
  const OverrideCols src{staged<int64_t>(c, at[6]), staged<int64_t>(c, at[7]), staged<uint8_t>(c, at[8]), staged<int64_t>(c, at[9]),
                         staged<uint32_t>(c, at[10]), staged<int64_t>(c, at[11]), n_in};
  const OverrideCols old{c->d_ovr_begin.as<int64_t>(), c->d_ovr_end.as<int64_t>(), c->d_ovr_flags.as<uint8_t>(), c->d_ovr_thr.as<int64_t>(),
                         c->d_ovr_present.as<uint32_t>(), c->d_ovr_cnt.as<int64_t>(), c->n_ovr};
  const OverrideOut out{c->s_ovr_begin.as<int64_t>(), c->s_ovr_end.as<int64_t>(), c->s_ovr_flags.as<uint8_t>(), c->s_ovr_thr.as<int64_t>(),
                        c->s_ovr_present.as<uint32_t>(), c->s_ovr_cnt.as<int64_t>(), n_new};
  k_rebuild_overrides<<<(unsigned)((M1 + 1 + 127) / 128), 128, 0, c->stream>>>(M1, R, k, staged<int32_t>(c, at[13]), staged<int32_t>(c, at[14]),
                                                                             staged<int32_t>(c, at[12]), c->d_ovr_off.as<int32_t>(), old,
                                                                             staged<int32_t>(c, at[5]), src, c->s_ovr_off.as<int32_t>(), out, nullptr);
  KT_CUDA(c, cudaGetLastError());
  std::swap(c->d_ovr_off, c->s_ovr_off); std::swap(c->d_ovr_begin, c->s_ovr_begin); std::swap(c->d_ovr_end, c->s_ovr_end);
  std::swap(c->d_ovr_flags, c->s_ovr_flags); std::swap(c->d_ovr_thr, c->s_ovr_thr); std::swap(c->d_ovr_present, c->s_ovr_present);
  std::swap(c->d_ovr_cnt, c->s_ovr_cnt);
  c->M = M1;
  c->n_ovr = n_new;
  c->h_ovr_off.swap(new_off);
  if (!fits) {  // the tables compiled again from the grown spec (kt_upload_namespaces)
    if ((rc = recompile_tables(c)) || (rc = stage_ns_spec(c))) return rc;
    KT_CUDA(c, cudaStreamSynchronize(c->stream));
    if (recompiled) *recompiled = 1;
    return KT_OK;
  }
  if ((rc = stage_ns_spec(c))) return rc;  // term ranges, requirements and ns_id of the grown spec
  if (NS > 0) {
    k_ns_cols<<<(unsigned)(((int64_t)NS * (int64_t)nw + 7) / 8), 256, 0, c->stream>>>(ns_spec_view(c), NS, (int32_t)nw, staged<int32_t>(c, at[17]),
                                                                                       staged<int64_t>(c, at[18]), LN, c->n_ns, c->d_nsmask.as<uint32_t>());
    KT_CUDA(c, cudaGetLastError());
  }
  if ((rc = rebuild_ns_words(c, NS, at[19]))) return rc;
  old_table.release();  // the stream has passed every read of the old buffers (rebuild_ns_words synchronised)
  old_need.release();
  old_nsmask.release();
  return KT_OK;
}

// ---- column moves (kt_nsrows.cuh k_gather_bits; k_widen_cols and k_rebuild_overrides through a column map) --------------
int kt_move_throttle_columns(kt_ctx* c, int32_t m, const int32_t* src) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (m < 0) return fail(c, KT_ERR_INVALID, "kt_move_throttle_columns: m = %d", m);
  if (m > 0 && !src) return fail(c, KT_ERR_INVALID, "kt_move_throttle_columns: null src with m = %d", m);
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_move_throttle_columns before kt_upload_throttles");
  const int32_t M0 = c->M;
  std::vector<char> named((size_t)M0, 0);
  for (int32_t j = 0; j < m; ++j) {
    if (src[j] < -1 || src[j] >= M0)
      return fail(c, KT_ERR_INVALID, "kt_move_throttle_columns: column %d from %d, out of range [-1,%d)", j, src[j], M0);
    if (src[j] >= 0 && named[(size_t)src[j]]++) return fail(c, KT_ERR_INVALID, "kt_move_throttle_columns: column %d listed twice", src[j]);
  }
  int rc = set_device(c);
  if (rc) return rc;
  const int R = c->lim.n_resources;
  HostTables& h = c->ht;
  // The gathered spec, its term_unsat entries and override offsets.  The row dictionary, TPpad, B and NS are kept: no column is
  // compiled, so the table and need bits are gathered on the device and brought back for the host mirror (patch_columns reads
  // it), which costs one copy of the two arrays instead of a bit-by-bit permutation of them on the host.
  SelectorSpec spec = splice_spec(c->spec, 0, nullptr, SelectorSpec{}, m, src);
  std::vector<uint8_t> unsat;
  unsat.reserve(spec.term_flags.size());
  std::vector<int32_t> new_off((size_t)m + 1, 0);
  for (int32_t j = 0; j < m; ++j) {
    const int32_t t = src[j];
    int32_t n = 0;
    if (t >= 0) {
      unsat.insert(unsat.end(), h.term_unsat.begin() + c->spec.term_off[(size_t)t], h.term_unsat.begin() + c->spec.term_off[(size_t)t + 1]);
      n = c->h_ovr_off[(size_t)t + 1] - c->h_ovr_off[(size_t)t];
    }
    new_off[(size_t)j + 1] = new_off[(size_t)j] + n;  // at most n_ovr: every previous column is named once at most
  }
  const int32_t n_new = new_off[(size_t)m];
  const int32_t W0 = h.W, W1 = std::max(1, (m + 31) / 32), NS = h.NS, TPpad = h.TPpad;
  const size_t tlen = (size_t)h.rows * TPpad * 2, nlen = (size_t)TPpad * h.B;
  // pass state sized by M, as kt_upload_throttles reserves it
  const size_t part_bytes = (size_t)(2 * R + 1) * m * sizeof(unsigned long long);
  c->part_stride = (part_bytes + 255) & ~(size_t)255;
  KT_CUDA(c, c->d_part.reserve(2 * c->part_stride + 16));
  KT_CUDA(c, cudaMemsetAsync(c->d_part.p, 0, c->d_part.cap, c->stream));
  c->part_parity = 0;
  c->win_stale = c->win != nullptr;  // laid out for the previous M
  c->pre_stride = (size_t)((m + 31) & ~31) * pre_record_bytes(R);
  KT_CUDA(c, c->d_pre.reserve(2 * c->pre_stride + 16));
  KT_CUDA(c, c->d_changed.reserve(16 + (size_t)m * 5 + 16));
  KT_CUDA(c, cudaMemsetAsync(c->d_changed.p, 0, 16, c->stream));
  const size_t out_bytes = status_layout(R, m).bytes;
  KT_CUDA(c, c->d_out.reserve(out_bytes + 16));
  // the restrided arrays' spare halves, the spare override set, the gathered bit arrays and the word lists
  const std::vector<AppendTarget> tg = append_targets(c);
  for (size_t j = 0; j < tg.size(); ++j) KT_CUDA(c, c->w_spare[j].reserve((size_t)tg[j].rows * m * tg[j].esize + 16));
  KT_CUDA(c, c->s_ovr_off.reserve(((size_t)m + 1) * 4 + 16));
  KT_CUDA(c, c->s_ovr_begin.reserve((size_t)n_new * 8 + 16));
  KT_CUDA(c, c->s_ovr_end.reserve((size_t)n_new * 8 + 16));
  KT_CUDA(c, c->s_ovr_flags.reserve((size_t)n_new + 16));
  KT_CUDA(c, c->s_ovr_thr.reserve((size_t)R * n_new * 8 + 16));
  KT_CUDA(c, c->s_ovr_present.reserve((size_t)n_new * 4 + 16));
  KT_CUDA(c, c->s_ovr_cnt.reserve((size_t)n_new * 8 + 16));
  KT_CUDA(c, c->g_spare[0].reserve((size_t)W1 * tlen * 4 + 16));
  KT_CUDA(c, c->g_spare[1].reserve((size_t)W1 * nlen * 4 + 16));
  KT_CUDA(c, c->g_spare[2].reserve((size_t)NS * W1 * TPpad * 4 + 16));
  KT_CUDA(c, c->d_nsw_off.reserve(((size_t)NS + 1) * 4 + 16));
  KT_CUDA(c, c->d_nsw_idx.reserve((size_t)NS * W1 * 4 + 16));
  KT_CUDA(c, c->d_call_out.reserve(((size_t)NS + 4) * 4 + 16));
  // the pinned call block: the staged pieces, then where the gathered table and need land (reserved first: a grown block would
  // drop the staged pieces)
  auto pad = [](size_t b) { return (b + 15) & ~(size_t)15; };
  const size_t land = pad((size_t)m * 4) + pad(((size_t)m + 1) * 4) + 16, tbytes = (size_t)W1 * tlen * 4, nbytes = (size_t)W1 * nlen * 4;
  KT_CUDA(c, c->h_call.reserve(std::max(out_bytes, land + tbytes + nbytes)));
  static const int32_t result_slot[4] = {};
  size_t at[3];
  if ((rc = stage_pieces(c, {{src, (size_t)m * 4}, {new_off.data(), new_off.size() * 4}, {result_slot, sizeof result_slot}}, at))) return rc;
  const int32_t* map = staged<int32_t>(c, at[0]);
  // one launch restrides every per-throttle array through the map
  WidenBatch wb{};
  int64_t widest = 0;
  for (size_t j = 0; j < tg.size(); ++j) {
    wb.a[wb.n++] = WidenArray{static_cast<const unsigned char*>(tg[j].buf->p), nullptr, static_cast<unsigned char*>(c->w_spare[j].p), tg[j].rows,
                              M0, m, tg[j].esize, map};
    widest = std::max(widest, tg[j].rows * m);
  }
  const unsigned wblocks = (unsigned)std::min<int64_t>((widest + 255) / 256, 2048);
  k_widen_cols<<<dim3(std::max(wblocks, 1u), (unsigned)wb.n), 256, 0, c->stream>>>(wb);
  KT_CUDA(c, cudaGetLastError());
  for (size_t j = 0; j < tg.size(); ++j) std::swap(*tg[j].buf, c->w_spare[j]);
  // the override columns rebuilt into the spare set through the map
  const OverrideCols old{c->d_ovr_begin.as<int64_t>(), c->d_ovr_end.as<int64_t>(), c->d_ovr_flags.as<uint8_t>(), c->d_ovr_thr.as<int64_t>(),
                         c->d_ovr_present.as<uint32_t>(), c->d_ovr_cnt.as<int64_t>(), c->n_ovr};
  const OverrideOut out{c->s_ovr_begin.as<int64_t>(), c->s_ovr_end.as<int64_t>(), c->s_ovr_flags.as<uint8_t>(), c->s_ovr_thr.as<int64_t>(),
                        c->s_ovr_present.as<uint32_t>(), c->s_ovr_cnt.as<int64_t>(), n_new};
  k_rebuild_overrides<<<(unsigned)((m + 1 + 127) / 128), 128, 0, c->stream>>>(m, R, 0, nullptr, nullptr, staged<int32_t>(c, at[1]),
                                                                            c->d_ovr_off.as<int32_t>(), old, nullptr, OverrideCols{},
                                                                            c->s_ovr_off.as<int32_t>(), out, map);
  KT_CUDA(c, cudaGetLastError());
  std::swap(c->d_ovr_off, c->s_ovr_off); std::swap(c->d_ovr_begin, c->s_ovr_begin); std::swap(c->d_ovr_end, c->s_ovr_end);
  std::swap(c->d_ovr_flags, c->s_ovr_flags); std::swap(c->d_ovr_thr, c->s_ovr_thr); std::swap(c->d_ovr_present, c->s_ovr_present);
  std::swap(c->d_ovr_cnt, c->s_ovr_cnt);
  // table, need and nsmask gathered by column in one launch
  GatherBitsBatch gb{};
  gb.a[0] = GatherBitsArray{c->d_table.as<uint32_t>(), c->g_spare[0].as<uint32_t>(), 1, (int64_t)tlen, W0, W1, true};
  gb.a[1] = GatherBitsArray{c->d_need.as<uint32_t>(), c->g_spare[1].as<uint32_t>(), 1, (int64_t)nlen, W0, W1, false};
  gb.a[2] = GatherBitsArray{c->d_nsmask.as<uint32_t>(), c->g_spare[2].as<uint32_t>(), NS, TPpad, W0, W1, false};
  gb.map = map;
  gb.m = m;
  int64_t items = 0;
  for (const GatherBitsArray& a : gb.a) items = std::max(items, a.outer * a.w_new * ((a.len + 31) / 32));
  const unsigned gblocks = (unsigned)std::min<int64_t>((items + 7) / 8, 4096);
  k_gather_bits<<<dim3(std::max(gblocks, 1u), 3), 256, 0, c->stream>>>(gb);
  KT_CUDA(c, cudaGetLastError());
  std::swap(c->d_table, c->g_spare[0]);
  std::swap(c->d_need, c->g_spare[1]);
  std::swap(c->d_nsmask, c->g_spare[2]);
  unsigned char* landed = c->h_call.as<unsigned char>() + land;
  if (tbytes) KT_CUDA(c, cudaMemcpyAsync(landed, c->d_table.p, tbytes, cudaMemcpyDeviceToHost, c->stream));
  if (nbytes) KT_CUDA(c, cudaMemcpyAsync(landed + tbytes, c->d_need.p, nbytes, cudaMemcpyDeviceToHost, c->stream));
  // the host side of the new layout
  c->spec = std::move(spec);
  h.term_unsat.swap(unsat);
  h.M = m;
  h.W = W1;
  h.Wp = words_per_row(m);
  h.TP = 1;
  for (int32_t t = 0; t < m; ++t) h.TP = std::max(h.TP, c->spec.term_off[(size_t)t + 1] - c->spec.term_off[(size_t)t]);
  c->M = m;
  c->n_ovr = n_new;
  c->h_ovr_off.swap(new_off);
  // as after kt_upload_throttles: a pass is needed again before the getters that read one (status and reservations are kept)
  c->evaluated = false;
  c->have_codes = false;
  c->have_diff = false;
  if ((rc = stage_ns_spec(c)) || (rc = rebuild_ns_words(c, NS, at[2]))) return rc;  // rebuild_ns_words synchronises
  const uint32_t* lt = reinterpret_cast<const uint32_t*>(landed);
  h.table.assign(lt, lt + (size_t)W1 * tlen);
  h.need.assign(lt + (size_t)W1 * tlen, lt + (size_t)W1 * (tlen + nlen));
  return KT_OK;
}

int32_t kt_match_words(const kt_ctx* c) { return c && c->have_throttles ? c->ht.Wp : 0; }

static int evaluate_locked(kt_ctx* c, int64_t now, uint32_t flags);
int kt_evaluate(kt_ctx* c, int64_t now, uint32_t flags) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  return evaluate_locked(c, now, flags);
}
static int evaluate_locked(kt_ctx* c, int64_t now, uint32_t flags) {
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_evaluate before kt_upload_throttles");
  const bool given = flags & KT_EVAL_GIVEN_STATUS;
  const bool do_rec = !(flags & KT_EVAL_SKIP_RECONCILE), do_chk = !(flags & KT_EVAL_SKIP_CHECK);
  if (given && !c->have_status) return fail(c, KT_ERR_STATE, "KT_EVAL_GIVEN_STATUS without kt_upload_status");
  if (!do_rec && !given && do_chk) return fail(c, KT_ERR_INVALID, "KT_EVAL_SKIP_RECONCILE needs KT_EVAL_GIVEN_STATUS");
  const LastPass prev = last_pass_on(c->stream);  // (set_device forgets it)
  int rc = set_device(c);
  if (rc) return rc;
  const int R = c->lim.n_resources, M = c->M, Wp = c->ht.Wp;
  PodStore& run = c->pods[KT_PODS_RUNNING];
  PodStore& pend = c->pods[KT_PODS_PENDING];
  {
    // A buffer allocated here holds whatever the allocator hands back; a pass that does not write it (a check-only pass leaves
    // the running bitmap alone, a reconcile-only pass the codes) must not let the getters deliver that: zeroed once on allocation.
    const void* b0 = run.bitmap.p; const void* b1 = pend.bitmap.p; const void* b2 = c->d_codes.p; const void* b3 = c->d_admit.p;
    KT_CUDA(c, run.bitmap.reserve((size_t)run.n * Wp * 4 + 16));
    KT_CUDA(c, pend.bitmap.reserve((size_t)pend.n * Wp * 4 + 16));
    KT_CUDA(c, c->d_codes.reserve((size_t)pend.n * 2 * Wp * 4 + 16));
    KT_CUDA(c, c->d_admit.reserve((size_t)pend.n + 16));
    if (run.bitmap.p != b0) run.bitmap_clean = false;
    if (pend.bitmap.p != b1 || c->d_codes.p != b2) pend.bitmap_clean = false;
    const std::pair<DevBuf*, const void*> grown[] = {{&run.bitmap, b0}, {&pend.bitmap, b1}, {&c->d_codes, b2}, {&c->d_admit, b3}};
    for (const auto& g : grown)
      if (g.first->p != g.second) KT_CUDA(c, cudaMemsetAsync(g.first->p, 0, g.first->cap, c->stream));
  }
  if (do_rec && (rc = ensure_roff(c, run))) return rc;   // no-ops unless rows or tables changed since the last pass
  if (do_chk && (rc = ensure_roff(c, pend))) return rc;
  const TableView tb = table_view(c);
  int launches = 0;
  const bool tm = c->timing;

  const ThrottleView tv = throttle_view(c);
  ReconcileView ov = status_at<ReconcileView>(c->d_out.p, R, M);
  c->have_diff = c->have_status && do_rec && M > 0;
  if (c->have_diff) {
    c->diff_parity ^= 1u;
    uint32_t* cnt = c->d_changed.as<uint32_t>();
    ov.changed_count = cnt + c->diff_parity;
    ov.changed_count_next = cnt + (c->diff_parity ^ 1u);
    ov.changed_idx = reinterpret_cast<int32_t*>(c->d_changed.as<unsigned char>() + 16);
    ov.changed_flag = c->d_changed.as<unsigned char>() + 16 + (size_t)M * 4;
  }
  int G = 1;
  while (G < R + 1) G <<= 1;  // finalize lanes per throttle: resources + the pod count, padded to a power of two
  // partial sums: a reconciling pass takes the half its predecessor left zeroed and zeroes the other one for its successor
  if (do_rec) c->part_parity ^= 1u;
  PartExchange px = local_exchange(c);

  // ---- the whole pass in one launch (k_pass), both halves asked for.  With several ranks the all-reduce happens
  // inside it: finalize tiles add this rank's partial sums into every rank's totals over NVLink (exchange windows). ----
  const bool multi = c->comm && c->nranks > 1;
  const bool whole = !tm && do_rec && do_chk && M > 0 && run.n > 0 && pend.n > 0;
  if (whole && multi) {
    if ((rc = ensure_window(c, (size_t)(2 * R + 1) * M * 8))) return rc;
    if (!c->p2p_failed) {
      unsigned epoch = ++c->epoch;
      if (epoch == 0) epoch = c->epoch = 1;  // 0 is what an untouched slot carries
      const size_t mine_off = kWinHeader + (size_t)(epoch & 1) * c->win_part_bytes, zmine_off = kWinHeader + (size_t)((epoch + 1) & 1) * c->win_part_bytes;
      const size_t total_off = mine_off + 2 * c->win_part_bytes;
      const size_t slots_off = kWinHeader + 4 * c->win_part_bytes + (size_t)(epoch & 1) * c->nranks * 2 * c->win_part_bytes;
      unsigned char* base = reinterpret_cast<unsigned char*>(c->win);
      px.sync = reinterpret_cast<PassSync*>(base);
      px.mine = reinterpret_cast<unsigned long long*>(base + mine_off);
      px.total = reinterpret_cast<unsigned long long*>(base + total_off);
      px.zero_mine = reinterpret_cast<unsigned long long*>(base + zmine_off);
      px.slots = reinterpret_cast<unsigned long long*>(base + slots_off);
      px.len = (unsigned)((2 * R + 1) * M);
      px.epoch = epoch;
      px.npeers = 0;
      for (int r = 0; r < c->nranks; ++r) {
        if (r == c->rank) continue;
        unsigned char* pb = reinterpret_cast<unsigned char*>(c->peer_win[r]);
        px.peer_slots[px.npeers] = reinterpret_cast<unsigned long long*>(pb + slots_off);
        px.peer_rank[px.npeers] = r;
        ++px.npeers;
      }
    }
  }
  if (whole && (!multi || !c->p2p_failed)) {
    if (c->plan_forced) {
      // Test seam: every output and pre-record of the pass is poisoned first (the bitmaps and code rows are zero-filled again by
      // the pass, as after new rows), so that a piece of work a forced plan never ran cannot hide behind the last pass's results.
      for (DevBuf* b : {&run.bitmap, &pend.bitmap, &c->d_codes, &c->d_admit, &c->d_pre, &c->d_out})
        if (b->p) KT_CUDA(c, cudaMemsetAsync(b->p, 0xA5, b->cap, c->stream));
      run.bitmap_clean = pend.bitmap_clean = false;
    }
    // counters and pre-records of the other parity: an early successor uses them while this pass may still read its own
    c->pass_parity ^= 1u;
    if (px.npeers == 0) px.sync = c->d_sync.as<PassSync>() + c->pass_parity;
    PassArgs a{};
    a.run = pod_view(run); a.pend = pod_view(pend); a.tb = tb; a.tv = tv; a.out = ov; a.px = px;
    a.run_bitmap = run.bitmap.as<uint32_t>(); a.pend_bitmap = pend.bitmap.as<uint32_t>(); a.codes = c->d_codes.as<uint32_t>();
    a.admit = c->d_admit.as<unsigned char>(); a.pre = pre_records(c); a.sync = px.sync;
    // Early: the first phase runs before the wait for the previous grid (k_pass has the argument).  Only behind a fused pass of
    // this library -- of another context, or of this one when neither pass zero-fills (a zero-fill clears words the other pass
    // writes or reads) -- and not across GPUs.  Anything queued between the two (copies, plain kernels, a stream switch) is
    // waited for in full before this pass starts, whatever the flag says.
    const bool zero_fill = a.run.zero_fill || a.pend.zero_fill;
    a.early = px.npeers == 0 && prev.ctx && (prev.ctx != c || (!prev.zero_fill && !zero_fill));
    a.sparse = sparse_view(c);
    a.now = (long long)now; a.eval_flags = flags; a.L = c->lim.label_slots; a.R = R; a.S = reconcile_slots(c); a.G = G;
    a.n_rec = (unsigned)((run.n + kTileReconcile - 1) / kTileReconcile);
    a.n_fin = (unsigned)(((long long)M * G + kTileReconcile - 1) / kTileReconcile);
    a.n_chk = (unsigned)((pend.n + kTileReconcile - 1) / kTileReconcile);
    if (c->trace) {
      const size_t rows = (size_t)a.n_chk + a.n_rec + a.n_fin;  // one per match, reconcile and status tile (at 128-row tiles: an upper bound for 256-row ones)
      KT_CUDA(c, c->d_trace.reserve(rows * kTraceRow * 8));  // (k_pass clears each row it writes: no memset between queued passes)
      a.trace = c->d_trace.as<unsigned long long>();
    }
    KT_CUDA(c, dispatch_pass(c, a));
    note_pass(c->stream, c, zero_fill);
    if ((rc = sparse_to_caller(c))) return rc;
    c->have_ran = true;
    run.bitmap_clean = pend.bitmap_clean = true;  // zero-filled (if need be) and written by this pass: maintained from here on
    // only a pass that waits for OTHER ranks can time out; under a forced plan the waits on its own tiles are checked as well
    // (a wait on a larger ticket would stall there, on a grid of a few CTAs, and must not pass as void results)
    c->last_sync = (multi && !c->p2p_failed) || c->plan_forced ? a.sync : nullptr;
    c->last = kt_timing{};
    c->last.launches = 1;
    c->evaluated = true;
    c->have_codes = true;
    return KT_OK;
  }

  // ---- separate kernels, PDL-chained: partial passes (SKIP_*), per-kernel timing, NCCL all-reduce in between ----
  if (px.npeers > 0) px = local_exchange(c);  // the window was set up but the one-launch pass is not taken after all: this rank's own buffers
  if (tm) KT_CUDA(c, cudaEventRecord(c->ev[0], c->stream));
  bool own_primary = false;  // the kernel right before k_finalize in the stream is this call's
  if (do_rec && run.n > 0 && M > 0) {
    const PodView pv = pod_view(run);
    const unsigned blocks = (unsigned)((run.n + kTileReconcile - 1) / kTileReconcile);
    KT_CUDA(c, dispatch_reconcile(c, pv, tb, px.mine, blocks));
    run.bitmap_clean = true;
    own_primary = true;
    ++launches;
  }
  if (tm) KT_CUDA(c, cudaEventRecord(c->ev[1], c->stream));
  if (do_rec && multi && M > 0) {
    // the single exchange of the pass: int64 sum of the per-throttle partials over NVLink
    int e = g_nccl.AllReduce(px.mine, px.mine, (size_t)(2 * R + 1) * M, kNcclInt64, kNcclSum, c->comm, c->stream);
    if (e != 0) return fail(c, KT_ERR_NCCL, "ncclAllReduce: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(e) : "error");
    own_primary = true;
  }
  if (tm) KT_CUDA(c, cudaEventRecord(c->ev[2], c->stream));
  if (M > 0) {
    // PDL: overlaps its launch + override merge with the tail of k_reconcile (or of the all-reduce kernel).  k_finalize writes
    // pre-records and zeroes the other partial-sum half BEFORE its wait, so without a primary of this call (a check-only pass:
    // the kernel ahead is the caller's previous launch, maybe a k_pass still reading pre-records) it is a plain launch.
    const long long lanes = (long long)M * G;
    KT_CUDA(c, launch(c, k_finalize, (unsigned)((lanes + 127) / 128), 128, 0, /*pdl=*/!tm && own_primary, tv, M, R, G, (long long)now, flags, px, ov,
                      pre_records(c)));
    ++launches;
  }
  if (tm) KT_CUDA(c, cudaEventRecord(c->ev[3], c->stream));
  if (do_chk && pend.n > 0) {
    const PodView pv = pod_view(pend);
    const unsigned blocks = (unsigned)((pend.n + kTileCheck - 1) / kTileCheck);
    if (c->sparse_cap) KT_CUDA(c, cudaMemsetAsync(c->d_sparse.p, 0, 4, c->stream));  // k_check appends; nobody in it can clear first
    KT_CUDA(c, dispatch_check(c, pv, tb, px, blocks, /*pdl=*/!tm && M > 0));  // its primary: this call's k_finalize
    pend.bitmap_clean = true;
    ++launches;
  }
  if (tm) KT_CUDA(c, cudaEventRecord(c->ev[4], c->stream));
  if (do_chk && (rc = sparse_to_caller(c))) return rc;  // after the timed kernels: delivering results is not the pass
  c->last = kt_timing{};
  c->last.launches = launches;
  c->evaluated = true;
  if (do_chk) c->have_codes = true;
  return KT_OK;
}

// ---- per-throttle row lists (kt_admit.cuh ColumnView) ---------------------------------------------------------------
// Counts, offsets and the scan on the stream, then one read of the total (also the whole off[] when off_host is given); the
// fill is queued only when `fill_cap` admits the total (a negative fill_cap: always).  v.bitmap, Wp, first, count, idx, k and
// codes are the caller's; the scratch buffers are the context's grow-only d_col_*, the codes beside the rows.
static int build_columns(kt_ctx* c, ColumnView& v, int64_t* total, int64_t* off_host, int64_t fill_cap = -1) {
  v.nblk = (int)((v.count + kColBlock - 1) / kColBlock);
  KT_CUDA(c, c->d_col_cnt.reserve((size_t)v.nblk * (size_t)v.k * 4 + 16));
  KT_CUDA(c, c->d_col_off.reserve((size_t)(v.k + 1) * 8 + 16));
  v.cnt = c->d_col_cnt.as<int32_t>();
  v.off = c->d_col_off.as<int64_t>();
  const int64_t warps = (int64_t)v.nblk * ((v.k + 31) / 32);
  if (warps > 0) k_col_count<<<(unsigned)((warps + 3) / 4), 128, 0, c->stream>>>(v);
  k_col_lengths<<<(unsigned)((v.k + 255) / 256), 256, 0, c->stream>>>(v);
  k_col_starts<<<1, 1024, 0, c->stream>>>(v);
  KT_CUDA(c, cudaGetLastError());
  if (off_host) KT_CUDA(c, cudaMemcpyAsync(off_host, v.off, (size_t)(v.k + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
  else KT_CUDA(c, cudaMemcpyAsync(total, v.off + v.k, 8, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  if (off_host) *total = off_host[v.k];
  if (fill_cap >= 0 && *total > fill_cap) return KT_OK;
  KT_CUDA(c, c->d_col_rows.reserve((size_t)*total * (v.codes ? 9 : 8) + 16));
  v.rows = c->d_col_rows.as<int64_t>();
  v.codes_out = c->d_col_rows.as<uint8_t>() + (size_t)*total * 8;
  if (warps > 0 && *total > 0) k_col_fill<<<(unsigned)((warps + 3) / 4), 128, 0, c->stream>>>(v);
  KT_CUDA(c, cudaGetLastError());
  return KT_OK;
}

// ---- queue-ordered greedy admission on the device (kt_admit.cuh) ----------------------------------------------------
int kt_admit_queue(kt_ctx* c, int64_t first, int64_t count, uint32_t flags, int32_t* rounds_out, int64_t* admitted_out) {
  if (!c || first < 0 || count < 0) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_admit_queue before kt_upload_throttles");
  if (!c->have_status) return fail(c, KT_ERR_STATE, "kt_admit_queue checks against the observed status: kt_upload_status first");
  PodStore& pend = c->pods[KT_PODS_PENDING];
  if (first + count > pend.n) return fail(c, KT_ERR_INVALID, "queue rows [%lld, %lld) outside the pending table (%lld rows)", (long long)first, (long long)(first + count), (long long)pend.n);
  // 1. one pending-only pass: affectedThrottles rows, pre-records (PreFilter's view: observed status + reservations); its
  // order-free codes are overwritten below for the queue rows
  int rc = evaluate_locked(c, 0, KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE | (flags & KT_EVAL_ON_EQUAL));
  if (rc) return rc;
  if (rounds_out) *rounds_out = 0;
  if (admitted_out) *admitted_out = 0;
  if (count == 0 || c->M == 0) return KT_OK;
  const int R = c->lim.n_resources, M = c->M;
  AdmitView a{};
  a.first = first; a.count = count; a.req = pend.req.as<int64_t>(); a.present = pend.present.as<uint32_t>(); a.bitmap = pend.bitmap.as<uint32_t>();
  a.n = pend.n; a.Wp = c->ht.Wp; a.W = c->ht.W; a.M = M; a.R = R; a.pre = pre_records(c);
  KT_CUDA(c, c->d_adm_state.reserve((size_t)count + 16));
  KT_CUDA(c, c->d_adm_fail.reserve((size_t)count * 4 + 16));
  KT_CUDA(c, c->d_adm_counters.reserve(16));
  a.state = c->d_adm_state.as<uint8_t>();
  a.fail = c->d_adm_fail.as<uint32_t>(); a.counters = c->d_adm_counters.as<uint32_t>();
  a.codes = c->d_codes.as<uint32_t>(); a.admit = c->d_admit.as<unsigned char>(); a.rowmap = dev_of(pend);
  // 2. every throttle's toucher list (CSR over the queue, built once)
  ColumnView v{};
  v.bitmap = a.bitmap; v.Wp = a.Wp; v.first = first; v.count = count; v.k = M; v.rowmap = a.rowmap;
  int64_t nnz = 0;
  if ((rc = build_columns(c, v, &nnz, nullptr))) return rc;
  a.tl_off = v.off; a.tl_pod = v.rows;
  KT_CUDA(c, cudaMemsetAsync(a.state, 0, (size_t)count, c->stream));
  // 3. rounds: until a round STARTED with nobody undecided (its loads were exact, and so are the codes it wrote)
  uint32_t counters[2] = {(uint32_t)count, 0};
  int rounds = 0;
  while (true) {
    const uint32_t undecided_before = counters[0];
    k_admit_begin<<<(unsigned)((count + 255) / 256), 256, 0, c->stream>>>(a);
    const unsigned blocks = (unsigned)((M + 3) / 4);
    if (R <= 4) k_admit_round<4><<<blocks, 128, 0, c->stream>>>(a);
    else if (R <= 8) k_admit_round<8><<<blocks, 128, 0, c->stream>>>(a);
    else k_admit_round<32><<<blocks, 128, 0, c->stream>>>(a);
    k_admit_update<<<(unsigned)((count + 255) / 256), 256, 0, c->stream>>>(a);
    KT_CUDA(c, cudaGetLastError());
    KT_CUDA(c, cudaMemcpyAsync(counters, a.counters, 8, cudaMemcpyDeviceToHost, c->stream));
    KT_CUDA(c, cudaStreamSynchronize(c->stream));
    ++rounds;
    if (undecided_before == 0) break;
    if (rounds > count + 2) return fail(c, KT_ERR_STATE, "kt_admit_queue did not converge");
  }
  if (rounds_out) *rounds_out = rounds;
  if (admitted_out) *admitted_out = counters[1];
  return KT_OK;
}

// ---- one end-to-end step in one call ------------------------------------------------------------------------------------
int kt_step_submit(kt_ctx* c, int64_t n_running, const kt_packed_pods* running, int64_t n_pending, const kt_packed_pods* pending, int64_t now, uint32_t flags) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->sparse_cap) return fail(c, KT_ERR_STATE, "kt_step_submit needs kt_set_sparse_check (the check result travels as admit bits + non-zero code words)");
  const bool saved = c->async_uploads;
  c->async_uploads = true;  // nothing in a step waits for the host before kt_step_wait
  int rc = KT_OK;
  if (running) rc = upload_pods_packed_locked(c, KT_PODS_RUNNING, n_running, running);
  if (!rc && pending) rc = upload_pods_packed_locked(c, KT_PODS_PENDING, n_pending, pending);
  if (!rc) rc = evaluate_locked(c, now, flags);
  c->async_uploads = saved;
  if (rc) return rc;
  forget_pass(c->stream);  // the result copies follow the pass
  // results -> ONE pinned block: [status block | admit | sparse count | first entries]
  const int64_t P = c->pods[KT_PODS_PENDING].n;
  const size_t out_bytes = status_layout(c->lim.n_resources, c->M).bytes;
  const size_t off_admit = (out_bytes + 63) & ~(size_t)63, off_cnt = (off_admit + (size_t)P + 63) & ~(size_t)63, off_ent = off_cnt + 16;
  KT_CUDA(c, c->h_step.reserve(off_ent + (size_t)c->sparse_cap * 12 + 64));
  if (!c->ev_step) KT_CUDA(c, cudaEventCreateWithFlags(&c->ev_step, cudaEventDisableTiming));
  unsigned char* hb = c->h_step.as<unsigned char>();
  if (out_bytes) KT_CUDA(c, cudaMemcpyAsync(hb, c->d_out.p, out_bytes, cudaMemcpyDeviceToHost, c->stream));
  if (P > 0) {
    const unsigned char* src;
    if ((rc = admit_in_caller_order(c, &src))) return rc;
    KT_CUDA(c, cudaMemcpyAsync(hb + off_admit, src, (size_t)P, cudaMemcpyDeviceToHost, c->stream));
  }
  int64_t first = c->sparse_guess < c->sparse_cap ? c->sparse_guess : c->sparse_cap;
  if (P == 0) first = 0;
  // the count and the entries sit next to each other on the device ({count, pad to 16 B, entries}): one copy
  KT_CUDA(c, cudaMemcpyAsync(hb + off_cnt, c->d_sparse.p, 16 + (size_t)first * 12, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaEventRecord(c->ev_step, c->stream));
  c->step_first = first;
  c->step_off[0] = off_admit; c->step_off[1] = off_cnt; c->step_off[2] = off_ent;
  c->step_pending = true;
  return KT_OK;
}

int kt_step_wait(kt_ctx* c, kt_step_result* out) {
  if (!c || !out) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->step_pending) return fail(c, KT_ERR_STATE, "kt_step_wait without kt_step_submit");
  int rc = set_device(c);
  if (rc) return rc;
  KT_CUDA(c, cudaEventSynchronize(c->ev_step));
  c->step_pending = false;
  if ((rc = check_pass_error(c))) return rc;
  unsigned char* hb = c->h_step.as<unsigned char>();
  const int64_t P = c->pods[KT_PODS_PENDING].n;
  const int64_t total = P > 0 ? (int64_t)*reinterpret_cast<uint32_t*>(hb + c->step_off[1]) : 0;
  const int64_t have = total < (int64_t)c->sparse_cap ? total : (int64_t)c->sparse_cap;
  if (have > c->step_first) {  // more rejected pairs than the last pass had: fetch the rest
    KT_CUDA(c, cudaMemcpyAsync(hb + c->step_off[2] + (size_t)c->step_first * 12, c->d_sparse.as<unsigned char>() + 16 + (size_t)c->step_first * 12,
                               (size_t)(have - c->step_first) * 12, cudaMemcpyDeviceToHost, c->stream));
    KT_CUDA(c, cudaStreamSynchronize(c->stream));
  }
  int64_t g = total + total / 4 + 256;
  if (g > (int64_t)c->sparse_cap) g = c->sparse_cap;
  c->sparse_guess = (uint32_t)g;
  out->n_pending = P;
  out->n_sparse = total;
  out->admit = hb + c->step_off[0];
  out->entries = reinterpret_cast<const uint32_t*>(hb + c->step_off[2]);
  out->status = status_at<kt_reconcile_out>(hb, c->lim.n_resources, c->M);
  return KT_OK;
}

int kt_get_timing(kt_ctx* c, kt_timing* out) {
  if (!c || !out) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc = set_device(c);
  if (rc) return rc;
  if (c->timing && c->evaluated) {
    KT_CUDA(c, cudaEventSynchronize(c->ev[4]));
    cudaEventElapsedTime(&c->last.reconcile_ms, c->ev[0], c->ev[1]);
    cudaEventElapsedTime(&c->last.allreduce_ms, c->ev[1], c->ev[2]);
    cudaEventElapsedTime(&c->last.finalize_ms, c->ev[2], c->ev[3]);
    cudaEventElapsedTime(&c->last.check_ms, c->ev[3], c->ev[4]);
    cudaEventElapsedTime(&c->last.total_ms, c->ev[0], c->ev[4]);
  }
  *out = c->last;
  return KT_OK;
}

int kt_get_reconcile(kt_ctx* c, const kt_reconcile_out* o) {
  if (!c || !o) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_reconcile before kt_evaluate");
  if (int rc = device_ready(c)) return rc;
  const int R = c->lim.n_resources, M = c->M;
  // one copy of the whole block into the pinned mirror, then plain host copies into the caller's columns
  const size_t bytes = status_layout(R, M).bytes;
  KT_CUDA(c, c->h_call.reserve(bytes));
  if (bytes) KT_CUDA(c, cudaMemcpyAsync(c->h_call.p, c->d_out.p, bytes, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  copy_status(status_at<kt_reconcile_out>(c->h_call.p, R, M), o, R, M);
  return KT_OK;
}

int kt_get_changed(kt_ctx* c, int32_t* idx, int64_t cap, int64_t* count, uint8_t* flags) {
  if (!c || !count || cap < 0 || (cap > 0 && !idx)) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_changed before kt_evaluate");
  if (!c->have_diff) return fail(c, KT_ERR_STATE, "kt_get_changed: the last pass had no observed status to diff against (kt_upload_status) or did not reconcile");
  if (int rc = device_ready(c)) return rc;
  uint32_t n = 0;
  KT_CUDA(c, cudaMemcpyAsync(&n, c->d_changed.as<uint32_t>() + c->diff_parity, 4, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  *count = n;
  const int64_t have = (int64_t)n < cap ? (int64_t)n : cap;
  if (have > 0) KT_CUDA(c, cudaMemcpyAsync(idx, c->d_changed.as<unsigned char>() + 16, (size_t)have * 4, cudaMemcpyDeviceToHost, c->stream));
  if (flags && c->M > 0) KT_CUDA(c, cudaMemcpyAsync(flags, c->d_changed.as<unsigned char>() + 16 + (size_t)c->M * 4, (size_t)c->M, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  return KT_OK;
}

int kt_get_reconcile_rows(kt_ctx* c, int64_t k, const int32_t* idx, const kt_reconcile_out* o) {
  if (!c || !o || k < 0 || (k > 0 && !idx)) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_reconcile_rows before kt_evaluate");
  if (k == 0) return KT_OK;
  if (int rc = check_throttles(c, __func__, k, idx)) return rc;
  if (int rc = device_ready(c)) return rc;
  const int R = c->lim.n_resources, M = c->M;
  // the listed columns gathered into a status block of k columns: the download is proportional to what changed, not to M
  const size_t bytes = status_layout(R, k).bytes;
  if (int rc = upload(c, c->d_call_in, idx, (size_t)k)) return rc;
  KT_CUDA(c, c->d_call_out.reserve(bytes));
  KT_CUDA(c, c->h_call.reserve(bytes));
  k_gather_status<<<(unsigned)((k + 127) / 128), 128, 0, c->stream>>>(k, c->d_call_in.as<int32_t>(), R, M, status_at<ReconcileView>(c->d_out.p, R, M),
                                                                      status_at<ReconcileView>(c->d_call_out.p, R, k));
  KT_CUDA(c, cudaGetLastError());
  KT_CUDA(c, cudaMemcpyAsync(c->h_call.p, c->d_call_out.p, bytes, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  copy_status(status_at<kt_reconcile_out>(c->h_call.p, R, k), o, R, k);
  return KT_OK;
}

// ---- PreFilter for k listed pending rows (kt_keyed.cuh) -------------------------------------------------------------
// The pre-records of every throttle into d_chk_pre: the pass's prep half, GIVEN_STATUS (no clock is read).
int rows_prep(kt_ctx* c, uint32_t eval_flags) {
  const int M = c->M, R = c->lim.n_resources;
  if (M == 0) return KT_OK;
  KT_CUDA(c, c->d_chk_pre.reserve((size_t)M * pre_record_bytes(R) + 16));
  int G = 1;
  while (G < R + 1) G <<= 1;
  const long long lanes = (long long)M * G;
  k_rows_prep<<<(unsigned)((lanes + 127) / 128), 128, 0, c->stream>>>(throttle_view(c), M, R, G, eval_flags, c->d_chk_pre.as<unsigned char>());
  KT_CUDA(c, cudaGetLastError());
  return KT_OK;
}
// The block the keyed checks fetch from: admit[k] (padded to 16 B) | codes[k][2 Wp] | words[k][Wp], zeroed on the device so that
// every word outside a pod's namespace list reads 0; `fetch` is the prefix that holds the outputs the caller asked for.
struct CheckBlock {
  size_t adm_bytes, code_bytes, word_bytes, fetch;
  CheckBlock(int64_t k, int Wp, bool words, bool codes)
      : adm_bytes(((size_t)k + 15) & ~(size_t)15), code_bytes((size_t)k * 2 * Wp * 4), word_bytes((size_t)k * Wp * 4),
        fetch(words ? adm_bytes + code_bytes + word_bytes : codes ? adm_bytes + code_bytes : adm_bytes) {}
  size_t bytes() const { return adm_bytes + code_bytes + word_bytes; }
};
int kt_check_pending_rows(kt_ctx* c, uint32_t flags, int64_t k, const int64_t* rows, uint32_t* words, uint32_t* codes, uint8_t* admit) {
  if (!c || k < 0 || (k > 0 && !rows)) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (flags & ~KT_EVAL_ON_EQUAL) return fail(c, KT_ERR_INVALID, "kt_check_pending_rows: flags must be 0 or KT_EVAL_ON_EQUAL, not %u", flags);
  if (int rc = check_single_gpu(c, __func__)) return rc;
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_check_pending_rows before kt_upload_throttles");
  if (!c->have_status) return fail(c, KT_ERR_STATE, "kt_check_pending_rows checks against the observed status: kt_upload_status first");
  PodStore& pend = c->pods[KT_PODS_PENDING];
  if (int rc = check_rows(c, __func__, k, rows, pend.n)) return rc;
  if (k == 0) return KT_OK;
  int rc = set_device(c);
  if (rc) return rc;
  if ((rc = ensure_roff(c, pend))) return rc;  // rows or tables changed since the offsets were translated (what the next pass does first)
  const int R = c->lim.n_resources, Wp = c->ht.Wp;
  const uint32_t eval_flags = KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE | flags;
  const CheckBlock blk(k, Wp, words, codes);
  const size_t adm_bytes = blk.adm_bytes, code_bytes = blk.code_bytes, word_bytes = blk.word_bytes;
  if ((rc = upload(c, c->d_call_in, rows, (size_t)k))) return rc;
  KT_CUDA(c, c->d_call_out.reserve(blk.bytes() + 16));
  KT_CUDA(c, c->h_call.reserve(blk.fetch));
  KT_CUDA(c, cudaMemsetAsync(c->d_call_out.p, 0, blk.bytes(), c->stream));
  if ((rc = rows_prep(c, eval_flags))) return rc;
  unsigned char* ob = c->d_call_out.as<unsigned char>();
  RowsArgs a{};
  a.pods = pod_view(pend);
  a.tb = table_view(c);
  a.L = c->lim.label_slots; a.R = R; a.k = k;
  a.rows = c->d_call_in.as<int64_t>();
  a.dev_of = dev_of(pend);
  a.pre = c->d_chk_pre.as<unsigned char>();
  a.admit = ob;
  a.codes = reinterpret_cast<uint32_t*>(ob + adm_bytes);
  a.words = reinterpret_cast<uint32_t*>(ob + adm_bytes + code_bytes);
  KT_CUDA(c, with_variant(c, true, [&](auto tpc, auto b, auto, auto reg) {
    return launch(c, k_check_rows<tpc, b, reg>, (unsigned)((k + kRowsTile - 1) / kRowsTile), kRowsTile, rows_smem_bytes(a.L, R, reg), false, a);
  }));
  KT_CUDA(c, cudaMemcpyAsync(c->h_call.p, ob, blk.fetch, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  const unsigned char* hb = c->h_call.as<unsigned char>();
  if (admit) std::memcpy(admit, hb, (size_t)k);
  if (codes) std::memcpy(codes, hb + adm_bytes, code_bytes);
  if (words) std::memcpy(words, hb + adm_bytes + code_bytes, word_bytes);
  return KT_OK;
}

// ---- PreFilter of k pods given by value (kt_keyed.cuh) ----------------------------------------------------------------
int kt_check_pods(kt_ctx* c, uint32_t flags, int64_t k, const int64_t* labels, const int64_t* req, const uint32_t* present, const int32_t* ns_id,
                  uint32_t* words, uint32_t* codes, uint8_t* admit) {
  if (!c || k < 0) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  const int L = c->lim.label_slots, R = c->lim.n_resources;
  if (k > 0 && (!labels || !req || !present || !ns_id)) return fail(c, KT_ERR_INVALID, "kt_check_pods: null input column with k = %lld", (long long)k);
  if (flags & ~KT_EVAL_ON_EQUAL) return fail(c, KT_ERR_INVALID, "kt_check_pods: flags must be 0 or KT_EVAL_ON_EQUAL, not %u", flags);
  if (int rc = check_single_gpu(c, __func__)) return rc;
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_check_pods before kt_upload_throttles");
  if (!c->have_status) return fail(c, KT_ERR_STATE, "kt_check_pods checks against the observed status: kt_upload_status first");
  if (k == 0) return KT_OK;
  int rc = set_device(c);
  if (rc) return rc;
  const int Wp = c->ht.Wp;
  // the inputs in one copy: labels [L][k] | req [R][k] | present [k] | ns [k]
  const size_t lab_bytes = (size_t)L * k * 8, req_bytes = (size_t)R * k * 8;
  std::vector<unsigned char> hin(lab_bytes + req_bytes + (size_t)k * 8);
  std::memcpy(hin.data(), labels, lab_bytes);
  std::memcpy(hin.data() + lab_bytes, req, req_bytes);
  std::memcpy(hin.data() + lab_bytes + req_bytes, present, (size_t)k * 4);
  std::memcpy(hin.data() + lab_bytes + req_bytes + (size_t)k * 4, ns_id, (size_t)k * 4);
  if ((rc = upload_vec(c, c->d_call_in, hin))) return rc;
  const CheckBlock blk(k, Wp, words, codes);
  KT_CUDA(c, c->d_call_out.reserve(blk.bytes() + 16));
  KT_CUDA(c, c->h_call.reserve(blk.fetch));
  KT_CUDA(c, cudaMemsetAsync(c->d_call_out.p, 0, blk.bytes(), c->stream));
  if ((rc = rows_prep(c, KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE | flags))) return rc;
  const unsigned char* ib = c->d_call_in.as<unsigned char>();
  unsigned char* ob = c->d_call_out.as<unsigned char>();
  PodsArgs a{};
  a.tb = table_view(c);
  a.L = L; a.R = R; a.k = k;
  a.labels = reinterpret_cast<const int64_t*>(ib);
  a.req = reinterpret_cast<const int64_t*>(ib + lab_bytes);
  a.present = reinterpret_cast<const uint32_t*>(ib + lab_bytes + req_bytes);
  a.ns = reinterpret_cast<const int32_t*>(ib + lab_bytes + req_bytes + (size_t)k * 4);
  a.pre = c->d_chk_pre.as<unsigned char>();
  a.admit = ob;
  a.codes = reinterpret_cast<uint32_t*>(ob + blk.adm_bytes);
  a.words = reinterpret_cast<uint32_t*>(ob + blk.adm_bytes + blk.code_bytes);
  KT_CUDA(c, with_variant(c, true, [&](auto tpc, auto b, auto, auto reg) {
    return launch(c, k_check_pods<tpc, b, reg>, (unsigned)((k + kRowsTile - 1) / kRowsTile), kRowsTile, rows_smem_bytes(L, R, reg), false, a);
  }));
  KT_CUDA(c, cudaMemcpyAsync(c->h_call.p, ob, blk.fetch, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  const unsigned char* hb = c->h_call.as<unsigned char>();
  if (admit) std::memcpy(admit, hb, (size_t)k);
  if (codes) std::memcpy(codes, hb + blk.adm_bytes, blk.code_bytes);
  if (words) std::memcpy(words, hb + blk.adm_bytes + blk.code_bytes, blk.word_bytes);
  return KT_OK;
}

// ---- affectedThrottles of k pods given by value (kt_keyed.cuh) ------------------------------------------------------
int kt_match_pods(kt_ctx* c, int64_t k, const int64_t* labels, const int32_t* ns_id, uint32_t* words) {
  if (!c || k < 0) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  const int L = c->lim.label_slots;
  if (k > 0 && ((L > 0 && !labels) || !ns_id || !words)) return fail(c, KT_ERR_INVALID, "kt_match_pods: null pointer with k = %lld", (long long)k);
  if (int rc = check_single_gpu(c, __func__)) return rc;
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_match_pods before kt_upload_throttles");
  if (k == 0) return KT_OK;
  int rc = set_device(c);
  if (rc) return rc;
  const int Wp = c->ht.Wp;
  // the inputs in one copy: labels [L][k] | ns [k]
  const size_t lab_bytes = (size_t)L * k * 8;
  std::vector<unsigned char> hin(lab_bytes + (size_t)k * 4);
  if (lab_bytes) std::memcpy(hin.data(), labels, lab_bytes);
  std::memcpy(hin.data() + lab_bytes, ns_id, (size_t)k * 4);
  if ((rc = upload_vec(c, c->d_call_in, hin))) return rc;
  KT_CUDA(c, c->d_call_out.reserve((size_t)k * Wp * 4 + 16));
  MatchArgs a{};
  a.tb = table_view(c);
  a.L = L; a.k = k;
  a.labels = c->d_call_in.as<int64_t>();
  a.ns = reinterpret_cast<const int32_t*>(c->d_call_in.as<unsigned char>() + lab_bytes);
  a.words = c->d_call_out.as<uint32_t>();
  KT_CUDA(c, with_variant(c, true, [&](auto tpc, auto b, auto, auto reg) {
    return launch(c, k_match_pods<tpc, b, reg>, (unsigned)((k + kRowsTile - 1) / kRowsTile), kRowsTile, match_smem_bytes(L, reg), false, a);
  }));
  KT_CUDA(c, cudaMemcpyAsync(words, a.words, (size_t)k * Wp * 4, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  return KT_OK;
}

int kt_get_check_rows(kt_ctx* c, int64_t k, const int64_t* rows, uint32_t* codes, uint8_t* admit) {
  if (!c || k < 0 || (k > 0 && !rows)) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_check_rows before kt_evaluate");
  if (k == 0) return KT_OK;
  PodStore& s = c->pods[KT_PODS_PENDING];
  if (int rc = check_rows(c, __func__, k, rows, s.n)) return rc;
  if (int rc = device_ready(c)) return rc;
  const int Wc = 2 * c->ht.Wp;
  // the output block: admit[k] (padded to 16 B) | codes[k][Wc] -- one copy fetches the prefix the caller asked for
  const size_t adm_bytes = ((size_t)k + 15) & ~(size_t)15, code_bytes = (size_t)k * Wc * 4;
  const size_t fetch = codes ? adm_bytes + code_bytes : adm_bytes;
  if (int rc = stage_rows(c, s, c->d_call_in, k, rows)) return rc;
  KT_CUDA(c, c->d_call_out.reserve(adm_bytes + code_bytes + 16));
  KT_CUDA(c, c->h_call.reserve(fetch));
  const int64_t* d_rows = c->d_call_in.as<int64_t>();
  unsigned char* ob = c->d_call_out.as<unsigned char>();
  k_gather_bytes<<<(unsigned)((k + 255) / 256), 256, 0, c->stream>>>(k, d_rows, c->d_admit.as<unsigned char>(), ob);
  k_gather_rows<<<(unsigned)((k + 7) / 8), 256, 0, c->stream>>>(k, d_rows, Wc, c->d_codes.as<uint32_t>(), reinterpret_cast<uint32_t*>(ob + adm_bytes));
  KT_CUDA(c, cudaGetLastError());
  KT_CUDA(c, cudaMemcpyAsync(c->h_call.p, ob, fetch, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  const unsigned char* hb = c->h_call.as<unsigned char>();
  if (admit) std::memcpy(admit, hb, (size_t)k);
  if (codes) std::memcpy(codes, hb + adm_bytes, code_bytes);
  return KT_OK;
}

int kt_get_match_bitmap(kt_ctx* c, int kind, uint32_t* words) {
  if (!c || !words) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (int rc = check_kind(c, __func__, kind)) return rc;
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_match_bitmap before kt_evaluate");
  int rc = set_device(c);
  if (rc) return rc;
  PodStore& s = c->pods[kind];
  const uint32_t* src = s.bitmap.as<uint32_t>();
  if (s.clustered && s.n > 0) {
    KT_CUDA(c, s.t_words.reserve((size_t)s.n * c->ht.Wp * 4 + 16));
    src = to_caller_order(c, s, src, c->ht.Wp);
  }
  if (s.n > 0) KT_CUDA(c, cudaMemcpyAsync(words, src, (size_t)s.n * c->ht.Wp * 4, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  return KT_OK;
}

int kt_get_match_rows(kt_ctx* c, int kind, int64_t k, const int64_t* rows, uint32_t* words) {
  if (!c || k < 0 || (k > 0 && (!rows || !words))) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (int rc = check_kind(c, __func__, kind)) return rc;
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_match_rows before kt_evaluate");
  if (k == 0) return KT_OK;
  PodStore& s = c->pods[kind];
  if (int rc = check_rows(c, __func__, k, rows, s.n)) return rc;
  int rc = set_device(c);
  if (rc) return rc;
  const int Wp = c->ht.Wp;
  if ((rc = stage_rows(c, s, c->d_call_in, k, rows))) return rc;
  KT_CUDA(c, c->d_call_out.reserve((size_t)k * Wp * 4 + 16));
  k_gather_rows<<<(unsigned)((k + 7) / 8), 256, 0, c->stream>>>(k, c->d_call_in.as<int64_t>(), Wp, s.bitmap.as<uint32_t>(), c->d_call_out.as<uint32_t>());
  KT_CUDA(c, cudaGetLastError());
  KT_CUDA(c, cudaMemcpyAsync(words, c->d_call_out.p, (size_t)k * Wp * 4, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  return KT_OK;
}

int kt_get_match_columns(kt_ctx* c, int kind, int64_t k, const int32_t* idx, int64_t* off, int64_t* rows, uint8_t* codes, int64_t cap) {
  if (!c || k < 0 || cap < 0 || !off || (k > 0 && !idx) || (cap > 0 && !rows)) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (int rc = check_kind(c, __func__, kind)) return rc;
  if (kind == KT_PODS_RUNNING && codes) return fail(c, KT_ERR_INVALID, "kt_get_match_columns: codes belong to the pending rows");
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_match_columns before kt_evaluate");
  if (int rc = check_throttles(c, __func__, k, idx)) return rc;
  int rc = device_ready(c);
  if (rc) return rc;
  off[0] = 0;
  if (k == 0) return KT_OK;
  PodStore& s = c->pods[kind];
  KT_CUDA(c, c->d_col_idx.reserve((size_t)k * 4 + 16));
  KT_CUDA(c, cudaMemcpyAsync(c->d_col_idx.p, idx, (size_t)k * 4, cudaMemcpyHostToDevice, c->stream));
  ColumnView v{};
  v.bitmap = s.bitmap.as<uint32_t>(); v.Wp = c->ht.Wp; v.first = 0; v.count = s.n; v.idx = c->d_col_idx.as<int32_t>(); v.k = k;
  v.codes = codes ? c->d_codes.as<uint32_t>() : nullptr;
  v.rowmap = dev_of(s);
  int64_t total = 0;
  if ((rc = build_columns(c, v, &total, off, cap))) return rc;
  if (total > cap || total == 0) return KT_OK;  // off[] says how much room the rows need
  KT_CUDA(c, cudaMemcpyAsync(rows, v.rows, (size_t)total * 8, cudaMemcpyDeviceToHost, c->stream));
  if (codes) KT_CUDA(c, cudaMemcpyAsync(codes, v.codes_out, (size_t)total, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  return KT_OK;
}

// ---- reconcile(key) for k listed throttles (kt_keyed.cuh) ---------------------------------------------------------------
int kt_reconcile_throttles(kt_ctx* c, int64_t now, int64_t k, const int32_t* idx, const kt_reconcile_out* o, int64_t* off, int64_t* rows, int64_t cap) {
  if (!c || !o || !off || k < 0 || cap < 0 || (k > 0 && !idx) || (cap > 0 && !rows)) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (int rc = check_single_gpu(c, __func__)) return rc;
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_reconcile_throttles before kt_upload_throttles");
  if (int rc = check_throttles(c, __func__, k, idx)) return rc;
  const int M = c->M, R = c->lim.n_resources;
  off[0] = 0;
  if (k == 0) return KT_OK;
  int rc = set_device(c);
  if (rc) return rc;
  PodStore& run = c->pods[KT_PODS_RUNNING];
  if ((rc = ensure_roff(c, run))) return rc;  // rows or tables changed since the offsets were translated (a pure function of both)
  // the listed words and their listed bits; entry e sums into compact throttle cidx[e] = j * 32 + bit
  std::vector<int32_t> words;
  std::vector<uint32_t> masks;
  std::vector<int32_t> slot((size_t)c->ht.W, -1), cidx((size_t)k);
  for (int64_t e = 0; e < k; ++e) {
    const int w = idx[e] >> 5;
    if (slot[(size_t)w] < 0) { slot[(size_t)w] = (int32_t)words.size(); words.push_back(w); masks.push_back(0u); }
    masks[(size_t)slot[(size_t)w]] |= 1u << (idx[e] & 31);
    cidx[(size_t)e] = slot[(size_t)w] * 32 + (idx[e] & 31);
  }
  const int nw = (int)words.size(), NC = (nw + 31) / 32, NJ = nw * 32, NS = c->ht.NS;
  const size_t n = (size_t)run.n;
  // one upload: words[nw] | masks[nw] | idx[k] | cidx[k]
  std::vector<int32_t> list;
  list.reserve((size_t)2 * nw + 2 * (size_t)k);
  list.insert(list.end(), words.begin(), words.end());
  for (uint32_t m : masks) list.push_back((int32_t)m);
  list.insert(list.end(), idx, idx + k);
  list.insert(list.end(), cidx.begin(), cidx.end());
  if ((rc = upload_vec(c, c->d_call_in, list))) return rc;
  const int32_t* d_words = c->d_call_in.as<int32_t>();
  const uint32_t* d_masks = c->d_call_in.as<uint32_t>() + nw;
  const int32_t* d_idx = d_words + 2 * nw;
  const int32_t* d_cidx = d_idx + k;
  KT_CUDA(c, c->d_key_reach.reserve((size_t)NS * NC * 4 + 16));
  KT_CUDA(c, c->d_key_scratch.reserve(n * nw * 4 + 16));
  const size_t acc_bytes = (size_t)NJ * ((size_t)R * 8 + 8 + 4);
  KT_CUDA(c, c->d_key_acc.reserve(acc_bytes + 16));
  if (n) KT_CUDA(c, cudaMemsetAsync(c->d_key_scratch.p, 0, n * nw * 4, c->stream));
  KT_CUDA(c, cudaMemsetAsync(c->d_key_acc.p, 0, acc_bytes, c->stream));
  const TableView tb = table_view(c);
  if (NS > 0) k_keyed_reach<<<(unsigned)(((int64_t)NS * NC + 255) / 256), 256, 0, c->stream>>>(tb, nw, d_words, d_masks, NC, c->d_key_reach.as<uint32_t>());
  KT_CUDA(c, cudaGetLastError());
  KeyedArgs a{};
  a.pods = pod_view(run);
  a.tb = tb;
  a.L = c->lim.label_slots; a.R = R; a.nw = nw; a.words = d_words; a.masks = d_masks; a.reach = c->d_key_reach.as<uint32_t>(); a.NC = NC;
  a.scratch = c->d_key_scratch.as<uint32_t>();
  a.used = c->d_key_acc.as<unsigned long long>();
  a.cnt = a.used + (size_t)R * NJ;
  a.pres = reinterpret_cast<uint32_t*>(a.cnt + NJ);
  a.smem_acc = keyed_smem_acc_bytes(nw, R) <= kKeyedSmemAcc ? 1 : 0;
  if (n && NS > 0) {
    const int64_t tiles = (int64_t)((n + kKeyedTile - 1) / kKeyedTile);
    const unsigned grid = (unsigned)std::min<int64_t>(tiles, (int64_t)c->sm_count * 8);
    KT_CUDA(c, with_variant(c, false, [&](auto tpc, auto b, auto rt, auto reg) {
      const size_t smem = keyed_smem_bytes(nw, R, a.L, reg, a.smem_acc);
      return launch(c, k_keyed_rows<tpc, b, rt, reg>, grid, kKeyedTile, smem, false, a);
    }));
  }
  // the status of the k columns: a status block of k columns, as kt_get_reconcile_rows gathers it
  const size_t bytes = status_layout(R, k).bytes;
  KT_CUDA(c, c->d_call_out.reserve(bytes));
  KT_CUDA(c, c->h_call.reserve(bytes));
  k_keyed_status<<<(unsigned)((k + 127) / 128), 128, 0, c->stream>>>(k, d_idx, d_cidx, R, M, NJ, throttle_view(c), (long long)now, a.used, a.cnt, a.pres,
                                                                   status_at<ReconcileView>(c->d_call_out.p, R, k));
  KT_CUDA(c, cudaGetLastError());
  KT_CUDA(c, cudaMemcpyAsync(c->h_call.p, c->d_call_out.p, bytes, cudaMemcpyDeviceToHost, c->stream));
  // the matched rows: the scratch transposed (ColumnView over the compact words)
  ColumnView v{};
  v.bitmap = a.scratch; v.Wp = nw; v.first = 0; v.count = (int64_t)n; v.idx = d_cidx; v.k = k;
  v.rowmap = dev_of(run);  // the scratch is indexed by device row; the lists come out in caller rows
  int64_t total = 0;
  if ((rc = build_columns(c, v, &total, off, cap))) return rc;  // (synchronises the stream: the status block has landed)
  copy_status(status_at<kt_reconcile_out>(c->h_call.p, R, k), o, R, k);
  if (total > cap || total == 0) return KT_OK;  // off[] says how much room the rows need
  KT_CUDA(c, cudaMemcpyAsync(rows, v.rows, (size_t)total * 8, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  return KT_OK;
}

int kt_get_check(kt_ctx* c, uint32_t* codes, uint8_t* admit) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_check before kt_evaluate");
  int rc = device_ready(c);
  if (rc) return rc;
  PodStore& pend = c->pods[KT_PODS_PENDING];
  const int64_t P = pend.n;
  const size_t code_bytes = (size_t)P * 2 * c->ht.Wp * 4;
  const uint32_t* src_codes = c->d_codes.as<uint32_t>();
  if (codes && P > 0 && pend.clustered) {  // caller order through the staging buffer: codes, then admit behind them
    KT_CUDA(c, pend.t_words.reserve(code_bytes + (size_t)P + 16));
    src_codes = to_caller_order(c, pend, src_codes, 2 * c->ht.Wp);
  }
  if (codes && P > 0) KT_CUDA(c, cudaMemcpyAsync(codes, src_codes, code_bytes, cudaMemcpyDeviceToHost, c->stream));
  if (admit && P > 0) {
    const unsigned char* src;
    if ((rc = admit_in_caller_order(c, &src, codes ? code_bytes : 0))) return rc;
    KT_CUDA(c, cudaMemcpyAsync(admit, src, (size_t)P, cudaMemcpyDeviceToHost, c->stream));
  }
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  return KT_OK;
}

// ---- the scheduling queue summarised per throttle (kt_keyed.cuh) ------------------------------------------------------
int kt_get_check_summary(kt_ctx* c, int64_t first, int64_t count, const uint8_t* row_class, const kt_check_summary* o) {
  if (!c || !o) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  PodStore& pend = c->pods[KT_PODS_PENDING];
  if (first < 0 || count < 0 || first > pend.n - count)
    return fail(c, KT_ERR_INVALID, "rows [%lld, %lld + %lld) outside the pending table (%lld rows)", (long long)first, (long long)first, (long long)count, (long long)pend.n);
  if (int rc = check_single_gpu(c, __func__)) return rc;
  if (!c->evaluated || !c->have_codes) return fail(c, KT_ERR_STATE, "kt_get_check_summary before a pass wrote the pending codes");
  int rc = device_ready(c);
  if (rc) return rc;
  const int M = c->M, R = c->lim.n_resources;
  // one output block: status_cnt [3][M] | sole_cnt [M] | held [R][M] | held_present [M]; all zero when there is nothing to summarise
  const size_t u64s = (size_t)(4 + R) * M, out_bytes = u64s * 8 + (size_t)M * 4;
  KT_CUDA(c, c->h_call.reserve(out_bytes + 16));
  unsigned char* h = c->h_call.as<unsigned char>();
  if (count > 0 && M > 0) {
    if (row_class && (rc = upload(c, c->d_call_in, row_class, (size_t)count))) return rc;
    KT_CUDA(c, c->d_call_out.reserve(out_bytes + 16));
    unsigned char* ob = c->d_call_out.as<unsigned char>();
    KT_CUDA(c, cudaMemsetAsync(ob, 0, out_bytes, c->stream));
    SummaryArgs a{};
    a.first = first; a.count = count; a.n = pend.n; a.Wc = 2 * c->ht.Wp; a.R = R; a.M = M;
    a.codes = c->d_codes.as<uint32_t>(); a.admit = c->d_admit.as<unsigned char>();
    a.req = pend.req.as<int64_t>(); a.present = pend.present.as<uint32_t>();
    a.caller_of = pend.clustered ? pend.o_caller.as<uint32_t>() : nullptr;
    a.row_class = row_class ? c->d_call_in.as<unsigned char>() : nullptr;
    unsigned long long* u = reinterpret_cast<unsigned long long*>(ob);
    a.status_cnt = o->status_cnt ? u : nullptr;
    a.sole_cnt = o->sole_cnt ? u + (size_t)3 * M : nullptr;
    a.held = o->held ? u + (size_t)4 * M : nullptr;
    a.held_present = o->held_present ? reinterpret_cast<uint32_t*>(u + u64s) : nullptr;
    const int64_t rows = pend.clustered ? pend.n : count;
    const int64_t blocks = std::min<int64_t>((rows + kSummaryThreads - 1) / kSummaryThreads, (int64_t)c->sm_count * 8);
    k_check_summary<<<(unsigned)std::max<int64_t>(blocks, 1), kSummaryThreads, 0, c->stream>>>(a);
    KT_CUDA(c, cudaGetLastError());
    KT_CUDA(c, cudaMemcpyAsync(h, ob, out_bytes, cudaMemcpyDeviceToHost, c->stream));
    KT_CUDA(c, cudaStreamSynchronize(c->stream));
  } else {
    std::memset(h, 0, out_bytes);
  }
  if (o->status_cnt) std::memcpy(o->status_cnt, h, (size_t)3 * M * 8);
  if (o->sole_cnt) std::memcpy(o->sole_cnt, h + (size_t)3 * M * 8, (size_t)M * 8);
  if (o->held) std::memcpy(o->held, h + (size_t)4 * M * 8, (size_t)R * M * 8);
  if (o->held_present) std::memcpy(o->held_present, h + u64s * 8, (size_t)M * 4);
  return KT_OK;
}

int kt_set_sparse_check(kt_ctx* c, int64_t cap_entries) {
  if (!c || cap_entries < 0 || cap_entries > (int64_t)1 << 28) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc = set_device(c);
  if (rc) return rc;
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  c->sparse_cap = 0;
  if (cap_entries == 0) return KT_OK;
  KT_CUDA(c, c->d_sparse.reserve(16 + (size_t)cap_entries * 12));
  KT_CUDA(c, cudaMemsetAsync(c->d_sparse.p, 0, 16, c->stream));
  if (!c->h_sparse_count) KT_CUDA(c, cudaHostAlloc((void**)&c->h_sparse_count, 16, cudaHostAllocDefault));
  c->sparse_cap = (uint32_t)cap_entries;
  c->evaluated = false;  // the list belongs to a pass that ran with it switched on
  return KT_OK;
}

int kt_get_check_sparse(kt_ctx* c, uint8_t* admit, uint32_t* entries, int64_t cap, int64_t* count) {
  if (!c || !count || cap < 0 || (cap > 0 && !entries)) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_check_sparse before kt_evaluate");
  if (!c->sparse_cap) return fail(c, KT_ERR_STATE, "kt_get_check_sparse without kt_set_sparse_check");
  int rc = device_ready(c);
  if (rc) return rc;
  const int64_t P = c->pods[KT_PODS_PENDING].n;
  const int64_t room = cap < (int64_t)c->sparse_cap ? cap : (int64_t)c->sparse_cap;
  // one round trip in the common case: the count and as many entries as the last pass produced (plus slack) together
  int64_t first = c->sparse_guess < room ? c->sparse_guess : room;
  if (P == 0) first = 0;
  if (admit && P > 0) {
    const unsigned char* src;
    if ((rc = admit_in_caller_order(c, &src))) return rc;
    KT_CUDA(c, cudaMemcpyAsync(admit, src, (size_t)P, cudaMemcpyDeviceToHost, c->stream));
  }
  KT_CUDA(c, cudaMemcpyAsync(c->h_sparse_count, c->d_sparse.p, 4, cudaMemcpyDeviceToHost, c->stream));
  if (first > 0) KT_CUDA(c, cudaMemcpyAsync(entries, c->d_sparse.as<uint32_t>() + 4, (size_t)first * 12, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  const int64_t total = P > 0 ? (int64_t)*c->h_sparse_count : 0;
  *count = total;  // may exceed cap / the device capacity: the caller then reads the dense rows (kt_get_check)
  const int64_t have = total < room ? total : room;
  if (have > first) {
    KT_CUDA(c, cudaMemcpyAsync(entries + 3 * first, c->d_sparse.as<uint32_t>() + 4 + 3 * first, (size_t)(have - first) * 12, cudaMemcpyDeviceToHost, c->stream));
    KT_CUDA(c, cudaStreamSynchronize(c->stream));
  }
  int64_t g = total + total / 4 + 256;
  if (g > (int64_t)c->sparse_cap) g = c->sparse_cap;
  c->sparse_guess = (uint32_t)g;
  return KT_OK;
}

int kt_debug_compile_tables(const kt_limits* lim, int32_t m, const kt_throttle_cols* cols, const kt_selector_table* sel, int32_t n_ns,
                            const int64_t* ns_labels, int32_t dims[12], uint32_t* table, uint32_t* need, uint32_t* nsmask, int32_t* nsw_off,
                            int32_t* nsw_idx, uint32_t* keydir, uint32_t* valrow, uint32_t* hash) {
  if (!lim || !dims) return KT_ERR_INVALID;
  SelectorSpec spec;
  HostTables ht;
  if (!copy_selector_spec(m, cols, sel, &spec).empty()) return KT_ERR_INVALID;
  if (!compile_tables(*lim, spec, n_ns, ns_labels, &ht).empty()) return KT_ERR_INVALID;
  const int32_t d[12] = {ht.M, ht.W, ht.Wp, ht.TPpad, ht.B, ht.rows, ht.NS, ht.n_keydir, (int32_t)ht.valrow.size(), (int32_t)ht.nsw_idx.size(),
                         ht.max_ns_words, (int32_t)(ht.hash_mask + 1)};
  std::memcpy(dims, d, sizeof d);
  auto put = [](auto* dst, const auto& v) {
    if (dst && !v.empty()) std::memcpy(dst, v.data(), v.size() * sizeof(v[0]));
  };
  put(table, ht.table); put(need, ht.need); put(nsmask, ht.nsmask); put(nsw_off, ht.nsw_off); put(nsw_idx, ht.nsw_idx);
  put(keydir, ht.keydir); put(valrow, ht.valrow); put(hash, ht.hash);
  return KT_OK;
}

int kt_debug_set_pass_plan(kt_ctx* c, const kt_pass_plan* plan) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  kt_pass_plan p{};
  if (plan) {
    p.threads_per_sm = plan->threads_per_sm;
    p.decide = plan->decide;
    p.max_ctas = plan->max_ctas;
  }
  if (p.threads_per_sm != 0 && p.threads_per_sm != kPassThreadsShallow && p.threads_per_sm != kPassThreadsDeep)
    return fail(c, KT_ERR_INVALID, "threads_per_sm %d: expected 0, %d or %d", p.threads_per_sm, kPassThreadsShallow, kPassThreadsDeep);
  if (p.decide < 0 || p.decide > KT_PLAN_DECIDE_PER_POD) return fail(c, KT_ERR_INVALID, "decide %d: expected 0, 1 or 2", p.decide);
  c->plan = p;
  c->plan_forced = p.threads_per_sm != 0 || p.decide != 0 || p.max_ctas != 0;
  return KT_OK;
}

int kt_debug_get_pass_plan(kt_ctx* c, kt_pass_plan* last) {
  if (!c || !last) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->have_ran) return fail(c, KT_ERR_STATE, "kt_debug_get_pass_plan before the first fused pass");
  *last = c->ran;
  return KT_OK;
}

int kt_debug_get_ns_tables(kt_ctx* c, int32_t dims[5], uint32_t* nsmask, int32_t* nsw_off, int32_t* nsw_idx) {
  if (!c || !dims) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_debug_get_ns_tables before kt_upload_throttles");
  int rc = set_device(c);
  if (rc) return rc;
  const size_t NS = (size_t)c->ht.NS;
  dims[0] = c->ht.NS; dims[1] = c->nsw_total; dims[2] = c->ht.max_ns_words; dims[3] = c->ht.W; dims[4] = c->ht.TPpad;
  if (nsmask && NS) KT_CUDA(c, cudaMemcpyAsync(nsmask, c->d_nsmask.p, NS * c->ht.W * c->ht.TPpad * 4, cudaMemcpyDeviceToHost, c->stream));
  if (nsw_off) KT_CUDA(c, cudaMemcpyAsync(nsw_off, c->d_nsw_off.p, (NS + 1) * 4, cudaMemcpyDeviceToHost, c->stream));
  if (nsw_idx && c->nsw_total) KT_CUDA(c, cudaMemcpyAsync(nsw_idx, c->d_nsw_idx.p, (size_t)c->nsw_total * 4, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  return KT_OK;
}

int kt_debug_set_row_order(kt_ctx* c, int kind, int mode) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (int rc = check_kind(c, __func__, kind)) return rc;
  if (mode < KT_ROW_ORDER_AUTO || mode > KT_ROW_ORDER_BY_NAMESPACE) return fail(c, KT_ERR_INVALID, "row order %d: expected 0, 1 or 2", mode);
  c->pods[kind].order_mode = mode;
  return KT_OK;
}

int kt_debug_get_row_order(kt_ctx* c, int kind, int64_t* dev_row, int32_t* clustered) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (int rc = check_kind(c, __func__, kind)) return rc;
  const PodStore& s = c->pods[kind];
  if (clustered) *clustered = s.clustered ? 1 : 0;
  if (!dev_row || s.n == 0) return KT_OK;
  if (!s.clustered) {
    for (int64_t i = 0; i < s.n; ++i) dev_row[i] = i;
    return KT_OK;
  }
  int rc = set_device(c);
  if (rc) return rc;
  std::vector<uint32_t> map((size_t)s.n);
  KT_CUDA(c, cudaMemcpyAsync(map.data(), s.o_dev.p, (size_t)s.n * 4, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  for (int64_t i = 0; i < s.n; ++i) dev_row[i] = map[(size_t)i];
  return KT_OK;
}

int kt_comm_unique_id(uint8_t uid[128]) {
  if (!uid) return KT_ERR_INVALID;
  if (load_nccl()) return KT_ERR_NCCL;
  return g_nccl.GetUniqueId(uid) == 0 ? KT_OK : KT_ERR_NCCL;
}

int kt_comm_init(kt_ctx* c, const uint8_t uid[128], int nranks, int rank) {
  if (!c || !uid || nranks < 1 || rank < 0 || rank >= nranks) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (const char* e = load_nccl()) return fail(c, KT_ERR_NCCL, "%s", e);
  int rc = set_device(c);
  if (rc) return rc;
  Uid128 id;
  std::memcpy(id.internal, uid, 128);
  int e = g_nccl.CommInitRank(&c->comm, nranks, id, rank);
  if (e != 0) return fail(c, KT_ERR_NCCL, "ncclCommInitRank: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(e) : "error");
  c->nranks = nranks;
  c->rank = rank;
  return KT_OK;
}

int kt_comm_destroy(kt_ctx* c) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (set_device(c) == KT_OK) {
    cudaStreamSynchronize(c->stream);
    release_window(c);
  }
  if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
  c->comm = nullptr;
  c->nranks = 1;
  c->rank = 0;
  c->p2p_failed = false;
  return KT_OK;
}

}  // extern "C"
