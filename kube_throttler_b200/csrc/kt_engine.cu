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
#include <mutex>
#include <string>
#include <vector>

#include "../../include/kt_b200.h"
#include "kt_kernels.cuh"
#include "kt_admit.cuh"
#include "kt_tables.h"

namespace {

using namespace kt;

// ---- grow-only device buffer ---------------------------------------------------------------------
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;  // slack so row appends do not reallocate every time
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct PodStore {
  int64_t n = 0;
  DevBuf labels, req, present, flags, ns;
  DevBuf roff;              // [Lpad][n] u32: the labels as row offsets into the current selector tables (k_translate_rows)
  DevBuf winfo;             // [n] u32: the words that can apply to the row's namespace (winfo_pack), same life cycle as roff
  bool roff_valid = false;  // false after a full upload or a table compile; row deltas translate their own rows
  DevBuf c_labels, c_req, c_meta;  // staging of the compact transfer format (kt_upload_pods_compact)
  DevBuf c_pairs;                  // label-pair dictionary of the packed transfer format (kt_upload_pods_packed)
  DevBuf c_dict;                   // request-value dictionaries of the same format
  DevBuf t_rows, t_labels, t_req, t_present, t_flags, t_ns, t_words;  // grow-only staging of row deltas / row gathers
  DevBuf bitmap;  // [n][Wp]
  // The passes MAINTAIN the bitmap (and, for pending rows, the check codes): they store the words of each row's namespace list
  // and nothing else.  Whatever can leave a stale non-zero word outside those lists -- new rows, a row delta, new tables, a
  // buffer that was just allocated -- clears this flag; the next pass zeroes the buffers once before it runs.
  bool bitmap_clean = false;
  void release() {
    labels.release(); req.release(); present.release(); flags.release(); ns.release(); bitmap.release(); roff.release(); winfo.release();
    roff_valid = false;
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
  DevBuf d_kind, d_tflags, d_thr, d_thr_present, d_thr_cnt, d_ovr_off, d_ovr_begin, d_ovr_end, d_ovr_flags, d_ovr_thr,
      d_ovr_present, d_ovr_cnt;
  bool have_status = false;
  DevBuf d_st_calculated, d_st_calc_thr, d_st_calc_present, d_st_calc_cnt, d_st_used, d_st_used_present, d_st_used_cnt,
      d_st_throttled;
  bool have_reserved = false;
  DevBuf d_reserved, d_reserved_present, d_reserved_cnt;
  // pass state / outputs
  DevBuf d_part;   // 2 x [2R+1][M] u64 by pass parity: a reconciling pass adds into one half and leaves the other zeroed for its successor
  size_t part_stride = 0;  // bytes between the two halves
  unsigned part_parity = 0;  // half that holds the sums of the last reconcile
  DevBuf d_sync;   // PassSync counters of the fused pass (zero between launches)
  DevBuf d_trace;  // optional per-CTA trace rows of the fused pass
  bool trace = false;
  uint32_t trace_roles[4] = {0, 0, 0, 0};
  PassSync* last_sync = nullptr;  // counters of the last fused pass: its error flag is checked when results are fetched
  bool fused = true;  // one-launch pass (k_pass) when the whole pass is asked for; three PDL-chained kernels otherwise
  DevBuf d_changed;  // device-side status diff: {count[2] u32 by pass parity, pad to 16 B, idx[M] i32, flag[M] u8}
  unsigned diff_parity = 0;
  bool have_diff = false;  // the last pass produced a diff (an observed status was uploaded)
  DevBuf d_adm_cnt2, d_adm_off, d_adm_pod, d_adm_state, d_adm_fail, d_adm_counters;  // kt_admit_queue (kt_admit.cuh)
  DevBuf d_pre;    // [M] pre-records, finalize tiles -> decide tiles (kt_kernels.cuh pre_record_bytes)
  // per-throttle outputs of the reconcile half: ONE device block (and one pinned host mirror) so that kt_get_reconcile
  // is a single D2H copy; o_off[i] = byte offset of {used, used_cnt, calc_thr, calc_cnt, used_present, throttled,
  // calc_present, override_active}
  DevBuf d_out;
  void* h_out = nullptr;
  size_t h_out_cap = 0, out_bytes = 0;
  size_t o_off[8] = {};
  bool async_uploads = false;  // kt_set_async_uploads
  // kt_step_submit / kt_step_wait: one pinned result block, one event
  void* h_step = nullptr;
  size_t h_step_cap = 0, step_off[3] = {};
  cudaEvent_t ev_step = nullptr;
  int64_t step_first = 0;
  bool step_pending = false;
  DevBuf d_codes, d_admit;
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

#ifndef KT_WIDE_TILES  // 1: ClusterThrottle-heavy tables run the pass with 256-pod tiles
#define KT_WIDE_TILES 1
#endif
#ifndef KT_PASS_PDL  // 1: k_pass is launched with programmatic stream serialization (its launch overlaps the previous kernel's tail)
#define KT_PASS_PDL 1
#endif

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

int set_device(kt_ctx* c) {
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
template <class... KArgs, class... Args>
cudaError_t launch(kt_ctx* c, void (*kern)(KArgs...), unsigned blocks, unsigned threads, size_t smem, bool pdl, Args... args) {
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

// Kernel variant dispatch.  Fast family (label rows in registers): L <= 8 and counter bits B = 2, with the
// register accumulators sized for R <= 4 / R <= 8.  General family (rows in shared memory, shared-memory
// accumulation): any L <= 32, R <= 31, B in {2, 6}.  Both come for 1 or 2 term planes per table entry.
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
                (const unsigned char*)c->d_pre.as<unsigned char>(), px, c->pods[KT_PODS_PENDING].bitmap.as<uint32_t>(),
                c->d_codes.as<uint32_t>(), c->d_admit.as<unsigned char>(), sparse_view(c));
}
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
  a.n_status = (a.n_fin + kStatusBatch - 1) / kStatusBatch;
  // Does the whole grid fit on the device at once?  Then the match CTAs stay on as the decide tiles (k_pass, "resident").
  int per_sm = 0;
  cudaError_t e = cudaFuncSetAttribute((const void*)k_pass<TPC, B, RT, REG, TILE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pass<TPC, B, RT, REG, TILE>, TILE, smem);
  if (e != cudaSuccess) return e;
  const unsigned capacity = (unsigned)per_sm * (unsigned)c->sm_count;
  // (the status CTAs come last and are waited for by nobody on this GPU -- with peers only by decide tiles, after every
  // reconcile tile has left -- so they do not count)
  a.resident = (KT_PASS_RESIDENT != 0 && a.n_chk + a.n_rec <= capacity) ? 1u : 0u;
  if (a.resident && KT_PASS_RESIDENT == 2) {
    // shared second phase: the CTAs draw the decide sub-tiles and the status tiles from a ticket counter once their own tile
    // is done; the grid is the match and reconcile tiles only
    a.resident = 2u;
    a.n_sub = (unsigned)((a.pend.n + TILE / 4 - 1) / (TILE / 4));
    a.n_status = 0;
  }
  if (c->trace) { c->trace_roles[0] = a.n_chk; c->trace_roles[1] = a.n_rec; c->trace_roles[2] = a.n_status; c->trace_roles[3] = a.resident ? 0 : a.n_chk; }
  return launch(c, k_pass<TPC, B, RT, REG, TILE>, (a.resident ? 1u : 2u) * a.n_chk + a.n_rec + a.n_status, TILE, smem, /*pdl=*/KT_PASS_PDL != 0, a);
}
cudaError_t dispatch_pass(kt_ctx* c, const PassArgs& a) {
  const bool t1 = c->ht.TPpad == 1, b2 = c->ht.B <= 2;
  const int R = c->lim.n_resources;
  const bool fast = c->lim.label_slots <= 8 && b2 && R <= 8;
  // ClusterThrottle-heavy tables (a namespace's word list is long): 256 pods share a CTA's accumulator slots
  const bool wide = KT_WIDE_TILES != 0 && a.S >= 8 && kTileReconcile == 128;
  if (fast) {
    if (wide) {
      if (t1) return R <= 4 ? launch_pass<1, 2, 4, true, 256>(c, a) : launch_pass<1, 2, 8, true, 256>(c, a);
      return R <= 4 ? launch_pass<2, 2, 4, true, 256>(c, a) : launch_pass<2, 2, 8, true, 256>(c, a);
    }
    if (t1) return R <= 4 ? launch_pass<1, 2, 4, true, kTileReconcile>(c, a) : launch_pass<1, 2, 8, true, kTileReconcile>(c, a);
    return R <= 4 ? launch_pass<2, 2, 4, true, kTileReconcile>(c, a) : launch_pass<2, 2, 8, true, kTileReconcile>(c, a);
  }
  if (t1 && b2) return launch_pass<1, 2, 0, false, kTileReconcile>(c, a);
  if (t1) return launch_pass<1, 6, 0, false, kTileReconcile>(c, a);
  if (b2) return launch_pass<2, 2, 0, false, kTileReconcile>(c, a);
  return launch_pass<2, 6, 0, false, kTileReconcile>(c, a);
}
cudaError_t dispatch_reconcile(kt_ctx* c, const PodView& pv, const TableView& tb, unsigned long long* part, unsigned blocks) {
  const bool t1 = c->ht.TPpad == 1, b2 = c->ht.B <= 2;
  const int R = c->lim.n_resources;
  const bool fast = c->lim.label_slots <= 8 && b2 && R <= 8;
  if (fast) {
    if (t1) return R <= 4 ? launch_reconcile<1, 2, 4, true>(c, pv, tb, part, blocks) : launch_reconcile<1, 2, 8, true>(c, pv, tb, part, blocks);
    return R <= 4 ? launch_reconcile<2, 2, 4, true>(c, pv, tb, part, blocks) : launch_reconcile<2, 2, 8, true>(c, pv, tb, part, blocks);
  }
  if (t1 && b2) return launch_reconcile<1, 2, 0, false>(c, pv, tb, part, blocks);
  if (t1) return launch_reconcile<1, 6, 0, false>(c, pv, tb, part, blocks);
  if (b2) return launch_reconcile<2, 2, 0, false>(c, pv, tb, part, blocks);
  return launch_reconcile<2, 6, 0, false>(c, pv, tb, part, blocks);
}
cudaError_t dispatch_check(kt_ctx* c, const PodView& pv, const TableView& tb, const PartExchange& px, unsigned blocks, bool pdl) {
  const bool t1 = c->ht.TPpad == 1, b2 = c->ht.B <= 2;
  if (c->lim.label_slots <= 8 && b2) return t1 ? launch_check<1, 2, true>(c, pv, tb, px, blocks, pdl) : launch_check<2, 2, true>(c, pv, tb, px, blocks, pdl);
  if (t1 && b2) return launch_check<1, 2, false>(c, pv, tb, px, blocks, pdl);
  if (t1) return launch_check<1, 6, false>(c, pv, tb, px, blocks, pdl);
  if (b2) return launch_check<2, 2, false>(c, pv, tb, px, blocks, pdl);
  return launch_check<2, 6, false>(c, pv, tb, px, blocks, pdl);
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
  if (c->d_sync.reserve(sizeof(PassSync)) != cudaSuccess || cudaMemset(c->d_sync.p, 0, sizeof(PassSync)) != cudaSuccess) { kt_destroy(c); return KT_ERR_CUDA; }
  *out = c;
  return KT_OK;
}

void kt_destroy(kt_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  release_window(c);
  if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
  for (auto& s : c->pods) s.release();
  DevBuf* all[] = {&c->d_hash, &c->d_keydir, &c->d_valrow, &c->d_table, &c->d_need, &c->d_nsmask, &c->d_nsw_off, &c->d_nsw_idx, &c->d_kind, &c->d_tflags, &c->d_thr,
                   &c->d_thr_present, &c->d_thr_cnt, &c->d_ovr_off, &c->d_ovr_begin, &c->d_ovr_end, &c->d_ovr_flags, &c->d_ovr_thr,
                   &c->d_ovr_present, &c->d_ovr_cnt, &c->d_st_calculated, &c->d_st_calc_thr, &c->d_st_calc_present, &c->d_st_calc_cnt,
                   &c->d_st_used, &c->d_st_used_present, &c->d_st_used_cnt, &c->d_st_throttled, &c->d_reserved, &c->d_reserved_present,
                   &c->d_reserved_cnt, &c->d_part, &c->d_sync, &c->d_trace, &c->d_pre, &c->d_changed, &c->d_adm_cnt2, &c->d_adm_off, &c->d_adm_pod,
                   &c->d_adm_state, &c->d_adm_fail, &c->d_adm_counters, &c->d_out, &c->d_codes, &c->d_admit};
  if (c->h_out) cudaFreeHost(c->h_out);
  if (c->h_step) cudaFreeHost(c->h_step);
  if (c->ev_step) cudaEventDestroy(c->ev_step);
  if (c->h_sparse_count) cudaFreeHost(c->h_sparse_count);
  c->d_sparse.release();
  for (DevBuf* b : all) b->release();
  for (auto& e : c->ev)
    if (e) cudaEventDestroy(e);
  if (c->own_stream) cudaStreamDestroy(c->own_stream);
  delete c;
}

int kt_set_stream(kt_ctx* c, void* cuda_stream) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  c->stream = cuda_stream ? (cudaStream_t)cuda_stream : c->own_stream;
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
  const int64_t total = (int64_t)c->trace_roles[0] + c->trace_roles[1] + c->trace_roles[2] + c->trace_roles[3];
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

void* kt_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) return nullptr;
  return p;
}
void* kt_host_alloc_upload(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocWriteCombined) != cudaSuccess) return nullptr;
  return p;
}
void kt_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

int kt_upload_pods(kt_ctx* c, int kind, int64_t n, const int64_t* labels, const int64_t* req, const uint32_t* present,
                   const uint32_t* flags, const int32_t* ns_id) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (kind != KT_PODS_RUNNING && kind != KT_PODS_PENDING) return fail(c, KT_ERR_INVALID, "bad pod kind %d", kind);
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
  s.n = n;
  s.roff_valid = s.bitmap_clean = false;
  c->evaluated = false;
  if (!c->async_uploads) KT_CUDA(c, cudaStreamSynchronize(c->stream));  // the caller may reuse its buffers as soon as we return
  return KT_OK;
}

int kt_upload_pods_compact(kt_ctx* c, int kind, int64_t n, int32_t val_bits, const uint32_t* labels32, const int32_t* req32, const int32_t* req_shift,
                           const uint32_t* present, const uint32_t* meta) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (kind != KT_PODS_RUNNING && kind != KT_PODS_PENDING) return fail(c, KT_ERR_INVALID, "bad pod kind %d", kind);
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
  s.n = n;
  s.roff_valid = s.bitmap_clean = false;
  c->evaluated = false;
  if (!c->async_uploads) KT_CUDA(c, cudaStreamSynchronize(c->stream));  // the caller may reuse its buffers as soon as we return
  return KT_OK;
}

static int upload_pods_packed_locked(kt_ctx* c, int kind, int64_t n, const kt_packed_pods* pk);
int kt_upload_pods_packed(kt_ctx* c, int kind, int64_t n, const kt_packed_pods* pk) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  return upload_pods_packed_locked(c, kind, n, pk);
}
static int upload_pods_packed_locked(kt_ctx* c, int kind, int64_t n, const kt_packed_pods* pk) {
  if (kind != KT_PODS_RUNNING && kind != KT_PODS_PENDING) return fail(c, KT_ERR_INVALID, "bad pod kind %d", kind);
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
  KT_CUDA(c, s.labels.reserve((size_t)Lpad * n * 8 + 16));
  KT_CUDA(c, s.req.reserve((size_t)R * n * 8 + 16));
  KT_CUDA(c, s.present.reserve((size_t)n * 4 + 16));
  KT_CUDA(c, s.flags.reserve((size_t)n * 4 + 16));
  KT_CUDA(c, s.ns.reserve((size_t)n * 4 + 16));
  // The columns a caller carved out of ONE pinned block (bench.py, a Go packer with one arena per snapshot) cross the link as
  // one transfer: five copies of a few hundred KB each cost more in per-copy latency than their bytes.  Detected, not declared:
  // the device-bound arrays span little more than their own size.
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
  const bool one_block = n > 0 && sum > 0 && (lo & 15) == 0 && hi - lo <= sum + 2048;
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
    // with tables in place the rows are translated (labels -> table row offsets, namespace -> word info) in the same kernel:
    // one launch and one read of the labels less per upload
    const bool fuse = c->have_throttles;
    if (fuse) {
      KT_CUDA(c, s.roff.reserve((size_t)Lpad * n * 4 + 16));
      KT_CUDA(c, s.winfo.reserve((size_t)n * 4 + 16));
    }
    k_unpack_packed<<<(unsigned)((n + 255) / 256), 256, 0, c->stream>>>(n, L, Lpad, R, pk->ns_bits, pk->n_pairs, d_pairs, d_labels16,
                                                                        (const int32_t*)d_req, sh, rc, d_meta, s.labels.as<int64_t>(),
                                                                        s.req.as<int64_t>(), s.present.as<uint32_t>(), s.flags.as<uint32_t>(), s.ns.as<int32_t>(),
                                                                        fuse ? 1 : 0, fuse ? table_view(c) : TableView{}, s.roff.as<uint32_t>(), s.winfo.as<uint32_t>());
    KT_CUDA(c, cudaGetLastError());
    s.n = n;
    s.roff_valid = fuse;
    s.bitmap_clean = false;
  } else {
    s.n = n;
    s.roff_valid = s.bitmap_clean = false;
  }
  c->evaluated = false;
  if (!c->async_uploads) KT_CUDA(c, cudaStreamSynchronize(c->stream));  // the caller may reuse its buffers as soon as we return
  return KT_OK;
}

int kt_update_pod_rows(kt_ctx* c, int kind, int64_t k, const int64_t* rows, const int64_t* labels, const int64_t* req,
                       const uint32_t* present, const uint32_t* flags, const int32_t* ns_id) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (kind != KT_PODS_RUNNING && kind != KT_PODS_PENDING) return fail(c, KT_ERR_INVALID, "bad pod kind %d", kind);
  if (k < 0 || (k > 0 && (!rows || !labels || !req || !present || !flags || !ns_id))) return fail(c, KT_ERR_INVALID, "null delta columns");
  if (k == 0) return KT_OK;
  PodStore& s = c->pods[kind];
  for (int64_t i = 0; i < k; ++i)
    if (rows[i] < 0 || rows[i] >= s.n) return fail(c, KT_ERR_INVALID, "delta row %lld out of range [0,%lld)", (long long)rows[i], (long long)s.n);
  int rc = set_device(c);
  if (rc) return rc;
  const int L = c->lim.label_slots, R = c->lim.n_resources;
  // grow-only staging buffers: an informer event must not cost a cudaMalloc/cudaFree pair
  if ((rc = upload(c, s.t_rows, rows, (size_t)k)) || (rc = upload(c, s.t_labels, labels, (size_t)L * k)) || (rc = upload(c, s.t_req, req, (size_t)R * k)) ||
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
  KT_CUDA(c, c->d_pre.reserve((size_t)((m + 31) & ~31) * pre_record_bytes(R) + 16));  // whole 32-throttle words: a decide slot is staged as one block
  KT_CUDA(c, c->d_changed.reserve(16 + (size_t)m * 5 + 16));
  KT_CUDA(c, cudaMemsetAsync(c->d_changed.p, 0, 16, c->stream));
  c->have_diff = false;
  {
    const size_t sizes[8] = {(size_t)R * m * 8, (size_t)m * 8, (size_t)R * m * 8, (size_t)m * 8, (size_t)m * 4, (size_t)m * 4, (size_t)m * 4, (size_t)m};
    size_t at = 0;
    for (int i = 0; i < 8; ++i) { c->o_off[i] = at; at += (sizes[i] + 15) & ~(size_t)15; }
    c->out_bytes = at;
    KT_CUDA(c, c->d_out.reserve(at + 16));
    if (c->h_out_cap < at) {
      if (c->h_out) cudaFreeHost(c->h_out);
      c->h_out = nullptr;
      c->h_out_cap = 0;
      KT_CUDA(c, cudaHostAlloc(&c->h_out, at + 16, cudaHostAllocDefault));
      c->h_out_cap = at;
    }
  }
  c->have_throttles = true;
  c->have_status = false;
  c->have_reserved = false;
  c->evaluated = false;
  return recompile_tables(c);
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
  int rc = set_device(c);
  if (rc) return rc;
  const int R = c->lim.n_resources, M = c->M, Wp = c->ht.Wp;
  PodStore& run = c->pods[KT_PODS_RUNNING];
  PodStore& pend = c->pods[KT_PODS_PENDING];
  {
    const void* b0 = run.bitmap.p; const void* b1 = pend.bitmap.p; const void* b2 = c->d_codes.p;
    KT_CUDA(c, run.bitmap.reserve((size_t)run.n * Wp * 4 + 16));
    KT_CUDA(c, pend.bitmap.reserve((size_t)pend.n * Wp * 4 + 16));
    KT_CUDA(c, c->d_codes.reserve((size_t)pend.n * 2 * Wp * 4 + 16));
    if (run.bitmap.p != b0) run.bitmap_clean = false;
    if (pend.bitmap.p != b1 || c->d_codes.p != b2) pend.bitmap_clean = false;
  }
  KT_CUDA(c, c->d_admit.reserve((size_t)pend.n + 16));
  if (do_rec && (rc = ensure_roff(c, run))) return rc;   // no-ops unless rows or tables changed since the last pass
  if (do_chk && (rc = ensure_roff(c, pend))) return rc;
  const TableView tb = table_view(c);
  int launches = 0;
  const bool tm = c->timing;

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
  unsigned char* ob = c->d_out.as<unsigned char>();
  ReconcileView ov{reinterpret_cast<int64_t*>(ob + c->o_off[0]), reinterpret_cast<uint32_t*>(ob + c->o_off[4]), reinterpret_cast<int64_t*>(ob + c->o_off[1]),
                   reinterpret_cast<uint32_t*>(ob + c->o_off[5]), reinterpret_cast<int64_t*>(ob + c->o_off[2]), reinterpret_cast<uint32_t*>(ob + c->o_off[6]),
                   reinterpret_cast<int64_t*>(ob + c->o_off[3]), reinterpret_cast<uint8_t*>(ob + c->o_off[7]), nullptr, nullptr, nullptr, nullptr};
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
  PartExchange px{};
  px.mine = px.total = reinterpret_cast<unsigned long long*>(c->d_part.as<unsigned char>() + (size_t)c->part_parity * c->part_stride);
  px.zero_mine = reinterpret_cast<unsigned long long*>(c->d_part.as<unsigned char>() + (size_t)(c->part_parity ^ 1u) * c->part_stride);
  px.sync = c->d_sync.as<PassSync>();
  px.rank = c->rank;

  // ---- the whole pass in one launch (k_pass), both halves asked for.  With several ranks the all-reduce happens
  // inside it: finalize tiles add this rank's partial sums into every rank's totals over NVLink (exchange windows). ----
  const bool multi = c->comm && c->nranks > 1;
  const bool whole = c->fused && !tm && do_rec && do_chk && M > 0 && run.n > 0 && pend.n > 0;
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
    PassArgs a{};
    a.run = pod_view(run); a.pend = pod_view(pend); a.tb = tb; a.tv = tv; a.out = ov; a.px = px;
    a.run_bitmap = run.bitmap.as<uint32_t>(); a.pend_bitmap = pend.bitmap.as<uint32_t>(); a.codes = c->d_codes.as<uint32_t>();
    a.admit = c->d_admit.as<unsigned char>(); a.pre = c->d_pre.as<unsigned char>(); a.sync = px.sync;
    a.sparse = sparse_view(c);
    a.now = (long long)now; a.eval_flags = flags; a.L = c->lim.label_slots; a.R = R; a.S = reconcile_slots(c); a.G = G;
    a.n_rec = (unsigned)((run.n + kTileReconcile - 1) / kTileReconcile);
    a.n_fin = (unsigned)(((long long)M * G + kTileReconcile - 1) / kTileReconcile);
    a.n_chk = (unsigned)((pend.n + kTileReconcile - 1) / kTileReconcile);
    if (c->trace) {
      const size_t rows = (size_t)2 * a.n_chk + a.n_rec + a.n_fin;  // (an upper bound of the grid: resident passes launch fewer CTAs)
      KT_CUDA(c, c->d_trace.reserve(rows * kTraceRow * 8));
      KT_CUDA(c, cudaMemsetAsync(c->d_trace.p, 0, rows * kTraceRow * 8, c->stream));
      a.trace = c->d_trace.as<unsigned long long>();
      c->trace_roles[0] = a.n_chk; c->trace_roles[1] = a.n_rec; c->trace_roles[2] = a.n_fin; c->trace_roles[3] = a.n_chk;  // (prep tiles are counted with the match tiles)
    }
    KT_CUDA(c, dispatch_pass(c, a));
    run.bitmap_clean = pend.bitmap_clean = true;  // zero-filled (if need be) and written by this pass: maintained from here on
    c->last_sync = (multi && !c->p2p_failed) ? a.sync : nullptr;  // only a pass that waits for OTHER ranks can time out
    c->last = kt_timing{};
    c->last.launches = 1;
    c->evaluated = true;
    return KT_OK;
  }

  // ---- separate kernels, PDL-chained: partial passes (SKIP_*), per-kernel timing, NCCL all-reduce in between ----
  if (px.npeers > 0) {  // the window was set up but the one-launch pass is not taken after all: this rank's own buffers
    px = PartExchange{};
    px.mine = px.total = reinterpret_cast<unsigned long long*>(c->d_part.as<unsigned char>() + (size_t)c->part_parity * c->part_stride);
    px.zero_mine = reinterpret_cast<unsigned long long*>(c->d_part.as<unsigned char>() + (size_t)(c->part_parity ^ 1u) * c->part_stride);
    px.sync = c->d_sync.as<PassSync>();
    px.rank = c->rank;
  }
  if (tm) KT_CUDA(c, cudaEventRecord(c->ev[0], c->stream));
  if (do_rec && run.n > 0 && M > 0) {
    const PodView pv = pod_view(run);
    const unsigned blocks = (unsigned)((run.n + kTileReconcile - 1) / kTileReconcile);
    KT_CUDA(c, dispatch_reconcile(c, pv, tb, px.mine, blocks));
    run.bitmap_clean = true;
    ++launches;
  }
  if (tm) KT_CUDA(c, cudaEventRecord(c->ev[1], c->stream));
  if (do_rec && multi && M > 0) {
    // the single exchange of the pass: int64 sum of the per-throttle partials over NVLink
    int e = g_nccl.AllReduce(px.mine, px.mine, (size_t)(2 * R + 1) * M, kNcclInt64, kNcclSum, c->comm, c->stream);
    if (e != 0) return fail(c, KT_ERR_NCCL, "ncclAllReduce: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(e) : "error");
  }
  if (tm) KT_CUDA(c, cudaEventRecord(c->ev[2], c->stream));
  if (M > 0) {
    // PDL: overlaps its launch + override merge with the tail of k_reconcile (or of the all-reduce kernel)
    const long long lanes = (long long)M * G;
    KT_CUDA(c, launch(c, k_finalize, (unsigned)((lanes + 127) / 128), 128, 0, /*pdl=*/!tm, tv, M, R, G, (long long)now, flags, px, ov,
                      c->d_pre.as<unsigned char>()));
    ++launches;
  }
  if (tm) KT_CUDA(c, cudaEventRecord(c->ev[3], c->stream));
  if (do_chk && pend.n > 0) {
    const PodView pv = pod_view(pend);
    const unsigned blocks = (unsigned)((pend.n + kTileCheck - 1) / kTileCheck);
    if (c->sparse_cap) KT_CUDA(c, cudaMemsetAsync(c->d_sparse.p, 0, 4, c->stream));  // k_check appends; nobody in it can clear first
    KT_CUDA(c, dispatch_check(c, pv, tb, px, blocks, /*pdl=*/!tm && M > 0));
    pend.bitmap_clean = true;
    ++launches;
  }
  if (tm) KT_CUDA(c, cudaEventRecord(c->ev[4], c->stream));
  c->last = kt_timing{};
  c->last.launches = launches;
  c->evaluated = true;
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
  a.n = pend.n; a.Wp = c->ht.Wp; a.W = c->ht.W; a.M = M; a.R = R; a.pre = c->d_pre.as<unsigned char>();
  a.nblk = (int)((count + kAdmitBlock - 1) / kAdmitBlock);
  KT_CUDA(c, c->d_adm_cnt2.reserve((size_t)a.nblk * M * 4 + 16));
  KT_CUDA(c, c->d_adm_off.reserve((size_t)(M + 1) * 4 + 16));
  KT_CUDA(c, c->d_adm_state.reserve((size_t)count + 16));
  KT_CUDA(c, c->d_adm_fail.reserve((size_t)count * 4 + 16));
  KT_CUDA(c, c->d_adm_counters.reserve(16));
  a.cnt2 = c->d_adm_cnt2.as<int32_t>(); a.tl_off = c->d_adm_off.as<int32_t>(); a.state = c->d_adm_state.as<uint8_t>();
  a.fail = c->d_adm_fail.as<uint32_t>(); a.counters = c->d_adm_counters.as<uint32_t>();
  a.codes = c->d_codes.as<uint32_t>(); a.admit = c->d_admit.as<unsigned char>();
  // 2. every throttle's toucher list (CSR over the queue, built once)
  const unsigned warps = (unsigned)a.nblk * (unsigned)a.W;
  k_admit_count<<<(warps + 3) / 4, 128, 0, c->stream>>>(a);
  k_admit_lengths<<<(unsigned)((M + 255) / 256), 256, 0, c->stream>>>(a);
  k_admit_starts<<<1, 1024, 0, c->stream>>>(a);
  KT_CUDA(c, cudaGetLastError());
  int32_t nnz = 0;
  KT_CUDA(c, cudaMemcpyAsync(&nnz, a.tl_off + M, 4, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  KT_CUDA(c, c->d_adm_pod.reserve((size_t)nnz * 4 + 16));
  a.tl_pod = c->d_adm_pod.as<int32_t>();
  k_admit_fill<<<(warps + 3) / 4, 128, 0, c->stream>>>(a);
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
  // results -> ONE pinned block: [status block | admit | sparse count | first entries]
  const int64_t P = c->pods[KT_PODS_PENDING].n;
  const size_t off_admit = (c->out_bytes + 63) & ~(size_t)63, off_cnt = (off_admit + (size_t)P + 63) & ~(size_t)63, off_ent = off_cnt + 16;
  const size_t need = off_ent + (size_t)c->sparse_cap * 12 + 64;
  if (c->h_step_cap < need) {
    if (c->h_step) cudaFreeHost(c->h_step);
    c->h_step = nullptr;
    c->h_step_cap = 0;
    KT_CUDA(c, cudaHostAlloc(&c->h_step, need, cudaHostAllocDefault));
    c->h_step_cap = need;
  }
  if (!c->ev_step) KT_CUDA(c, cudaEventCreateWithFlags(&c->ev_step, cudaEventDisableTiming));
  unsigned char* hb = reinterpret_cast<unsigned char*>(c->h_step);
  if (c->out_bytes) KT_CUDA(c, cudaMemcpyAsync(hb, c->d_out.p, c->out_bytes, cudaMemcpyDeviceToHost, c->stream));
  if (P > 0) KT_CUDA(c, cudaMemcpyAsync(hb + off_admit, c->d_admit.p, (size_t)P, cudaMemcpyDeviceToHost, c->stream));
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
  unsigned char* hb = reinterpret_cast<unsigned char*>(c->h_step);
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
  out->status.used = reinterpret_cast<int64_t*>(hb + c->o_off[0]);
  out->status.used_cnt = reinterpret_cast<int64_t*>(hb + c->o_off[1]);
  out->status.calc_thr = reinterpret_cast<int64_t*>(hb + c->o_off[2]);
  out->status.calc_cnt = reinterpret_cast<int64_t*>(hb + c->o_off[3]);
  out->status.used_present = reinterpret_cast<uint32_t*>(hb + c->o_off[4]);
  out->status.throttled = reinterpret_cast<uint32_t*>(hb + c->o_off[5]);
  out->status.calc_present = reinterpret_cast<uint32_t*>(hb + c->o_off[6]);
  out->status.override_active = reinterpret_cast<uint8_t*>(hb + c->o_off[7]);
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
  int rc = set_device(c);
  if (rc) return rc;
  if ((rc = check_pass_error(c))) return rc;
  const size_t m = (size_t)c->M, R = (size_t)c->lim.n_resources;
  // one copy of the whole block into the pinned mirror, then plain host copies into the caller's columns
  if (c->out_bytes) KT_CUDA(c, cudaMemcpyAsync(c->h_out, c->d_out.p, c->out_bytes, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  const unsigned char* hb = reinterpret_cast<const unsigned char*>(c->h_out);
  auto put = [&](void* dst, int i, size_t bytes) {
    if (dst && bytes) std::memcpy(dst, hb + c->o_off[i], bytes);
  };
  put(o->used, 0, R * m * 8);
  put(o->used_cnt, 1, m * 8);
  put(o->calc_thr, 2, R * m * 8);
  put(o->calc_cnt, 3, m * 8);
  put(o->used_present, 4, m * 4);
  put(o->throttled, 5, m * 4);
  put(o->calc_present, 6, m * 4);
  put(o->override_active, 7, m);
  return KT_OK;
}

int kt_get_changed(kt_ctx* c, int32_t* idx, int64_t cap, int64_t* count, uint8_t* flags) {
  if (!c || !count || cap < 0 || (cap > 0 && !idx)) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_changed before kt_evaluate");
  if (!c->have_diff) return fail(c, KT_ERR_STATE, "kt_get_changed: the last pass had no observed status to diff against (kt_upload_status) or did not reconcile");
  int rc = set_device(c);
  if (rc) return rc;
  if ((rc = check_pass_error(c))) return rc;
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
  const int R = c->lim.n_resources, M = c->M;
  for (int64_t i = 0; i < k; ++i)
    if (idx[i] < 0 || idx[i] >= M) return fail(c, KT_ERR_INVALID, "throttle %d out of range [0,%d)", idx[i], M);
  int rc = set_device(c);
  if (rc) return rc;
  if ((rc = check_pass_error(c))) return rc;
  // one packed block per call: {used[R][k], calc_thr[R][k], used_cnt[k], calc_cnt[k], used_present[k], throttled[k], calc_present[k], override_active[k]}
  const size_t bytes = (size_t)k * ((size_t)2 * R * 8 + 16 + 12 + 1);
  PodStore& s = c->pods[KT_PODS_RUNNING];  // its grow-only staging buffers serve small gathers
  KT_CUDA(c, s.t_rows.reserve((size_t)k * 4 + 16));
  KT_CUDA(c, s.t_words.reserve(bytes + 64));
  if (c->h_out_cap < bytes + 64) {
    if (c->h_out) cudaFreeHost(c->h_out);
    c->h_out = nullptr;
    c->h_out_cap = 0;
    KT_CUDA(c, cudaHostAlloc(&c->h_out, bytes + 64, cudaHostAllocDefault));
    c->h_out_cap = bytes + 64;
  }
  KT_CUDA(c, cudaMemcpyAsync(s.t_rows.p, idx, (size_t)k * 4, cudaMemcpyHostToDevice, c->stream));
  unsigned char* ob = c->d_out.as<unsigned char>();
  const ReconcileView ov{reinterpret_cast<int64_t*>(ob + c->o_off[0]), reinterpret_cast<uint32_t*>(ob + c->o_off[4]), reinterpret_cast<int64_t*>(ob + c->o_off[1]),
                         reinterpret_cast<uint32_t*>(ob + c->o_off[5]), reinterpret_cast<int64_t*>(ob + c->o_off[2]), reinterpret_cast<uint32_t*>(ob + c->o_off[6]),
                         reinterpret_cast<int64_t*>(ob + c->o_off[3]), reinterpret_cast<uint8_t*>(ob + c->o_off[7]), nullptr, nullptr, nullptr, nullptr};
  k_gather_status<<<(unsigned)((k + 127) / 128), 128, 0, c->stream>>>(k, s.t_rows.as<int32_t>(), R, M, ov, s.t_words.as<unsigned char>());
  KT_CUDA(c, cudaGetLastError());
  KT_CUDA(c, cudaMemcpyAsync(c->h_out, s.t_words.p, bytes, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  const unsigned char* hb = reinterpret_cast<const unsigned char*>(c->h_out);
  size_t at = 0;
  auto take = [&](void* dst, size_t n) {
    if (dst) std::memcpy(dst, hb + at, n);
    at += n;
  };
  take(o->used, (size_t)R * k * 8); take(o->calc_thr, (size_t)R * k * 8); take(o->used_cnt, (size_t)k * 8); take(o->calc_cnt, (size_t)k * 8);
  take(o->used_present, (size_t)k * 4); take(o->throttled, (size_t)k * 4); take(o->calc_present, (size_t)k * 4); take(o->override_active, (size_t)k);
  return KT_OK;
}

int kt_get_check_rows(kt_ctx* c, int64_t k, const int64_t* rows, uint32_t* codes, uint8_t* admit) {
  if (!c || k < 0 || (k > 0 && !rows)) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_check_rows before kt_evaluate");
  if (k == 0) return KT_OK;
  PodStore& s = c->pods[KT_PODS_PENDING];
  for (int64_t i = 0; i < k; ++i)
    if (rows[i] < 0 || rows[i] >= s.n) return fail(c, KT_ERR_INVALID, "row %lld out of range [0,%lld)", (long long)rows[i], (long long)s.n);
  int rc = set_device(c);
  if (rc) return rc;
  if ((rc = check_pass_error(c))) return rc;
  const int Wc = 2 * c->ht.Wp;
  KT_CUDA(c, s.t_rows.reserve((size_t)k * 8));
  KT_CUDA(c, s.t_words.reserve((size_t)k * Wc * 4 + (size_t)k + 64));
  KT_CUDA(c, cudaMemcpyAsync(s.t_rows.p, rows, (size_t)k * 8, cudaMemcpyHostToDevice, c->stream));
  unsigned char* adm = s.t_words.as<unsigned char>() + (size_t)k * Wc * 4;
  k_gather_rows<<<(unsigned)((k + 7) / 8), 256, 0, c->stream>>>(k, s.t_rows.as<int64_t>(), Wc, c->d_codes.as<uint32_t>(), s.t_words.as<uint32_t>());
  k_gather_bytes<<<(unsigned)((k + 255) / 256), 256, 0, c->stream>>>(k, s.t_rows.as<int64_t>(), c->d_admit.as<unsigned char>(), adm);
  KT_CUDA(c, cudaGetLastError());
  if (codes) KT_CUDA(c, cudaMemcpyAsync(codes, s.t_words.p, (size_t)k * Wc * 4, cudaMemcpyDeviceToHost, c->stream));
  if (admit) KT_CUDA(c, cudaMemcpyAsync(admit, adm, (size_t)k, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  return KT_OK;
}

int kt_get_match_bitmap(kt_ctx* c, int kind, uint32_t* words) {
  if (!c || !words) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (kind != KT_PODS_RUNNING && kind != KT_PODS_PENDING) return fail(c, KT_ERR_INVALID, "bad pod kind %d", kind);
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_match_bitmap before kt_evaluate");
  int rc = set_device(c);
  if (rc) return rc;
  PodStore& s = c->pods[kind];
  if (s.n > 0) KT_CUDA(c, cudaMemcpyAsync(words, s.bitmap.p, (size_t)s.n * c->ht.Wp * 4, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  return KT_OK;
}

int kt_get_match_rows(kt_ctx* c, int kind, int64_t k, const int64_t* rows, uint32_t* words) {
  if (!c || k < 0 || (k > 0 && (!rows || !words))) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (kind != KT_PODS_RUNNING && kind != KT_PODS_PENDING) return fail(c, KT_ERR_INVALID, "bad pod kind %d", kind);
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_match_rows before kt_evaluate");
  if (k == 0) return KT_OK;
  PodStore& s = c->pods[kind];
  for (int64_t i = 0; i < k; ++i)
    if (rows[i] < 0 || rows[i] >= s.n) return fail(c, KT_ERR_INVALID, "row %lld out of range [0,%lld)", (long long)rows[i], (long long)s.n);
  int rc = set_device(c);
  if (rc) return rc;
  const int Wp = c->ht.Wp;
  KT_CUDA(c, s.t_rows.reserve((size_t)k * 8));
  KT_CUDA(c, s.t_words.reserve((size_t)k * Wp * 4));
  KT_CUDA(c, cudaMemcpyAsync(s.t_rows.p, rows, (size_t)k * 8, cudaMemcpyHostToDevice, c->stream));
  k_gather_rows<<<(unsigned)((k + 7) / 8), 256, 0, c->stream>>>(k, s.t_rows.as<int64_t>(), Wp, s.bitmap.as<uint32_t>(), s.t_words.as<uint32_t>());
  KT_CUDA(c, cudaGetLastError());
  KT_CUDA(c, cudaMemcpyAsync(words, s.t_words.p, (size_t)k * Wp * 4, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
  return KT_OK;
}

int kt_get_check(kt_ctx* c, uint32_t* codes, uint8_t* admit) {
  if (!c) return KT_ERR_INVALID;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_check before kt_evaluate");
  int rc = set_device(c);
  if (rc) return rc;
  if ((rc = check_pass_error(c))) return rc;
  const int64_t P = c->pods[KT_PODS_PENDING].n;
  if (codes && P > 0) KT_CUDA(c, cudaMemcpyAsync(codes, c->d_codes.p, (size_t)P * 2 * c->ht.Wp * 4, cudaMemcpyDeviceToHost, c->stream));
  if (admit && P > 0) KT_CUDA(c, cudaMemcpyAsync(admit, c->d_admit.p, (size_t)P, cudaMemcpyDeviceToHost, c->stream));
  KT_CUDA(c, cudaStreamSynchronize(c->stream));
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
  int rc = set_device(c);
  if (rc) return rc;
  if ((rc = check_pass_error(c))) return rc;
  const int64_t P = c->pods[KT_PODS_PENDING].n;
  const int64_t room = cap < (int64_t)c->sparse_cap ? cap : (int64_t)c->sparse_cap;
  // one round trip in the common case: the count and as many entries as the last pass produced (plus slack) together
  int64_t first = c->sparse_guess < room ? c->sparse_guess : room;
  if (P == 0) first = 0;
  if (admit && P > 0) KT_CUDA(c, cudaMemcpyAsync(admit, c->d_admit.p, (size_t)P, cudaMemcpyDeviceToHost, c->stream));
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
