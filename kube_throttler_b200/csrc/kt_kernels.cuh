// kt_kernels.cuh -- sm_90a kernels of the throttle-admission pass (hand-written CUDA, no libraries).
//
//   k_reconcile   running pods  -> affectedPods bitmap + per-throttle partial sums
//                 (replaces throttle_controller.go:221-246 affectedPods + :116-119 used-sum,
//                  clusterthrottle_controller.go:224-270, for EVERY throttle at once)
//   k_finalize    per throttle  -> CalculateThreshold(now), status.throttled, check constants
//                 (throttle_types.go:65-106, resource_amount.go:127-159, throttle_controller.go:122-133)
//   k_check       pending pods  -> affectedThrottles bitmap + 2-bit CheckThrottleStatus + admit
//                 (throttle_controller.go:248-269,349-397; throttle_types.go:128-153;
//                  clusterthrottle_types.go:30-55; plugin.go:177-180)
//
// HBM-bound integer work: no tensor cores.  One lane = one pod row for the selector match, which is
// word-parallel (32 throttles per LOP3) over the bit-sliced tables built by kt_tables.cc, so a pod costs
// O(label slots x non-zero namespace words) instead of O(throttles x terms x requirements).
// The segmented sum then flips the roles inside the warp: the 32x32 match bits are transposed with five
// shuffles so that one lane = one THROTTLE, which adds up its pods' requests from shared memory without
// any atomics; warps meet in per-CTA shared-memory accumulators and only those reach HBM (RED.ADD.64).
//
// A whole pass is ONE launch, k_pass: a grid no larger than the device holds at once, whose CTAs draw tickets from one counter
// until none is left -- pending-match tiles (which also write the per-throttle pre-records), reconcile tiles, then the second
// phase: status tiles and decide sub-tiles (TILE/4 pods, four lanes per pod, pre-records staged with cp.async.bulk on
// mbarriers, check_decide_quad); hand-offs are counters in L2.  Partial passes, per-kernel timing and the NCCL fallback run the same tile functions as the three
// kernels above, chained with programmatic dependent launch (griddepcontrol): k_check matches the pending pods while k_reconcile
// is still summing, and only its 4-step compare waits for k_finalize.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/kt_b200.h"
#include "kt_tables.h"

namespace kt {

// Resident threads per SM the fused pass is compiled for (register cap = 65536 / this).  Both are built; launch_pass picks one from
// the shape: 512 (128 registers, no spills) for passes whose tiles are a few rounds of the grid, where the chain after the last
// reconcile tile is the time; 768 (80 registers) for passes many rounds deep, whose reconcile tiles stream better with 24 warps
// per SM than with 16 (C5).
constexpr int kPassThreadsShallow = 512, kPassThreadsDeep = 768;
constexpr int kTileReconcile = 128;  // running pods per CTA (one lane per pod)
constexpr int kTileCheck = 64;       // pending pods per CTA
constexpr int kMaxSlots = 32;        // upper bound on the per-CTA accumulator slots (one per distinct 32-throttle word)
constexpr uint32_t kFull = 0xffffffffu;
constexpr int kStageChunk = 4;       // resources whose pre-record values and sums a decide lane requests together
constexpr int kPropose = 4;          // words a warp of a decide tile may propose to its CTA's staging table per round
constexpr int kTraceRow = 32;        // u64 per traced tile of the optional in-kernel trace: {ticket, sm, t_start, t_end, 12 stage stamps (globaltimer ns),
                                     // 12 cycle counts, CTA, CTA exit}

// Word info of a pod row (k_translate_rows; valid for the tables it was computed with): the words whose namespace mask is
// non-zero for the pod's namespace are the only ones the pod can match anything in.  Namespace-scoped Throttles give 1-3 of
// them, so the first two travel INLINE with the row -- the pass starts gathering table rows as soon as the row has landed,
// instead of two dependent hops (namespace -> list offsets -> word indices) later.
//   bits 0..11 first word, 12..23 second word, 24..31 count: 0..2 everything is inline; 3..254 the rest comes from the
//   namespace's list (nsw_off / nsw_idx); kWinfoList: tables with more than 4096 words, nothing is inline
constexpr uint32_t kWinfoList = 0xffu;
__host__ __device__ inline uint32_t winfo_pack(int cnt, int w0, int w1, int W) {
  if (W > 4096) return kWinfoList << 24;
  return (uint32_t)(w0 & 0xfff) | ((uint32_t)(w1 & 0xfff) << 12) | ((uint32_t)(cnt > 254 ? 254 : cnt) << 24);
}
constexpr int kHeavyPods = 6;        // a throttle matching more pods of a warp than this is summed by the whole warp

struct PodView {
  const int64_t* labels;    // [Lpad][n] keyId<<32 | valId (the snapshot as uploaded; re-translated when the tables change)
  const uint32_t* roff;     // [Lpad][n] the same labels as row offsets into the CURRENT selector tables (k_translate_rows)
  const uint32_t* winfo;    // [n] the 32-throttle words that can apply to the pod's namespace: first two inline + count (k_translate_rows)
  const int64_t* req;       // [R][n]
  const uint32_t* present;  // [n]
  const uint32_t* flags;    // [n]
  const int32_t* ns;        // [n]
  int64_t n;
  int zero_fill;            // 1: this pass zeroes the rows' bitmap (and code) rows itself -- the rows or the tables changed since the last
                            // pass, stale words may sit outside the namespaces' word lists; 0: the rows are maintained word by word
};

struct TableView {
  const uint4* hash;        // {keyId, valId, row, 0}; empty = {~0,~0,..}   (fallback for sparse ids)
  uint32_t hash_mask;
  const uint4* keydir;      // [n_keydir + 1] {other roff, vmin, vcnt, off (~0: hashed values)}; [n_keydir] = unmentioned key
  const uint32_t* valrow;   // roff or kOtherRoff; [0] = kOtherRoff
  uint32_t n_keydir;        // 0: no direct table, every label is hashed
  const uint32_t* table;    // [W][rows][TPpad][2]
  const uint32_t* need;     // [W][TPpad][B]
  const uint32_t* nsmask;   // [NS][W][TPpad]
  const int32_t* nsw_off;   // [NS+1]
  const int32_t* nsw_idx;
  int32_t M, W, Wp, TPpad, B, rows, NS;
};

// A lane's walk over its namespace's words in ascending order.
struct WordCursor {
  int cnt, inl, lo, w0, w1;
  __device__ __forceinline__ void init(const TableView& tb, uint32_t winfo, int ns, bool on) {
    const int c8 = on ? (int)(winfo >> 24) : 0;
    w0 = (int)(winfo & 0xfffu);
    w1 = (int)((winfo >> 12) & 0xfffu);
    cnt = c8;
    inl = c8 == (int)kWinfoList ? 0 : (c8 < 2 ? c8 : 2);
    lo = 0;
    if (c8 > 2) {  // rare with namespaced Throttles: the list itself
      lo = __ldg(&tb.nsw_off[ns]);
      cnt = __ldg(&tb.nsw_off[ns + 1]) - lo;
    }
  }
  __device__ __forceinline__ int at(const TableView& tb, int k) const {
    if (k >= cnt) return 0x7fffffff;
    if (k < inl) return k == 0 ? w0 : w1;
    return __ldg(&tb.nsw_idx[lo + k]);
  }
};

// Per-throttle constants of the 4-step check, produced by k_finalize, gathered per matched pair.
// Followed in memory by int64 thrv[R] (S1 thresholds) and int64 head[R] (S4: threshold - used - reserved).
struct __align__(16) CheckHdr {
  uint32_t thr_has;   // threshold has resource r
  uint32_t m2;        // status.throttled.resourceRequests[r] == true          (S2)
  uint32_t m3;        // threshold.IsThrottled(used+reserved, E3)[r]           (S3)
  uint32_t cntbits;   // bit0 S1 count, bit1 S2 count, bit2 S3 count, bit3 S4 count, bit4 S4 uses >= instead of >
};

struct ThrottleView {  // device copies of kt_throttle_cols / kt_status_cols / reserved
  const uint8_t* kind;
  const uint8_t* flags;
  const int64_t* thr;          // [R][M]
  const uint32_t* thr_present;
  const int64_t* thr_cnt;
  const int32_t* ovr_off;
  const int64_t* ovr_begin;
  const int64_t* ovr_end;
  const uint8_t* ovr_flags;
  const int64_t* ovr_thr;      // [R][n_ovr]
  const uint32_t* ovr_present;
  const int64_t* ovr_cnt;
  int32_t n_ovr;
  // observed status (GIVEN_STATUS); null otherwise
  const uint8_t* st_calculated;
  const int64_t* st_calc_thr;
  const uint32_t* st_calc_present;
  const int64_t* st_calc_cnt;
  const int64_t* st_used;
  const uint32_t* st_used_present;
  const int64_t* st_used_cnt;
  const uint32_t* st_throttled;
  // reservations (null => nothing reserved)
  const int64_t* reserved;
  const uint32_t* reserved_present;
  const int64_t* reserved_cnt;
};

struct ReconcileView {  // device-resident kt_reconcile_out
  int64_t* used;
  uint32_t* used_present;
  int64_t* used_cnt;
  uint32_t* throttled;
  int64_t* calc_thr;
  uint32_t* calc_present;
  int64_t* calc_cnt;
  uint8_t* override_active;
  // device-side status diff (SURVEY 8f.3; throttle_controller.go:157-173 only writes a status that differs from the informer
  // copy): with an observed status uploaded, every responsible throttle whose used / throttled / calculated threshold of THIS
  // pass differs from it is appended to a list (unordered) and flagged; null: no diff
  uint32_t* changed_count;       // this pass's counter
  uint32_t* changed_count_next;  // the other parity's: left zeroed for the next pass
  int32_t* changed_idx;          // [M]
  uint8_t* changed_flag;         // [M]
};

// ---- programmatic dependent launch (PTX griddepcontrol; both are no-ops in a plain launch) -------
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait_primary() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- in-kernel hand-off between the roles of the fused pass (k_pass) ----------------------------------
// Work is handed out by ONE ticket counter: pending-match tiles, reconcile tiles, then the second phase (status tiles and
// decide sub-tiles).  First-phase tiles never wait.  A second-phase piece waits only for pieces with smaller tickets, which
// running CTAs have already drawn (a CTA draws its next ticket only once its previous piece is done), or for other GPUs,
// whose pieces follow the same order -- so the waits cannot deadlock whatever the residency, and correctness does not depend
// on the grid fitting the device (k_pass sizes it to the device for speed only).  A CTA publishes its finished first-phase tiles
// in runs, when it draws its first ticket past them: match_done at its first reconcile ticket or when it leaves the phase,
// rec_done when it leaves the phase.  First-phase tiles never wait, so every one of them is published without anything having to
// wait for it, and before its CTA starts a piece that can wait.  prep_done and tot_done are signalled piece by piece.  Signals are
// fence + relaxed add (release pattern) by thread 0 after a CTA barrier; waits are relaxed polls + one acquire by thread 0 + a CTA barrier.
struct PassSync {
  // counters of ONE pass, re-armed by its last CTA (everything before `error`).  A context keeps one set per pass parity: an
  // early k_pass draws tickets while its predecessor still runs on the other set.
  unsigned ticket;      // next piece of work
  unsigned rec_done;    // reconcile tiles finished and published (their REDs are performed at L2)
  unsigned prep_done;   // finalize tiles that have written their throttles' pre-records (nothing to wait for: early)
  unsigned match_done;  // pending-match tiles finished (affectedThrottles rows written)
  unsigned tot_done;    // multi-GPU: finalize tiles of this rank that have written the all-rank totals of their throttles
  unsigned exited;      // CTAs that are done with everything; the last one re-arms the counters
  unsigned spare[2];    // unused: `error` stays at index kPassSyncRearm
  unsigned error;       // a wait gave up (kSpinTimeoutNs): a peer never arrived; the host reports it, the results are void
  unsigned pad[3];
};
constexpr int kPassSyncRearm = 8;  // leading counters the last CTA out (or the host, after a timed-out pass) zeroes
// Polling loads are RELAXED (performed at L2 / at the peer, no side effects on this SM); the acquire comes once, as one
// acquire load of the same counter after the awaited value has been seen.  An acquire load per poll would invalidate the
// SM's L1 on every iteration (CCTL.IVALL) and take the table rows of the tiles still working on that SM with it; an
// acquire FENCE instead of the final load also waits for the thread's own outstanding memory operations.
__device__ __forceinline__ unsigned ld_relaxed_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fence_acquire_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void cta_signal(unsigned* counter) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
  }
}
// No wait spins forever: a rank that died (or a bug) must not wedge the GPU.  After kSpinTimeoutNs the waiter records the
// failure and goes on; the pass's results are then meaningless and the host says so (KT_ERR_STATE).
constexpr unsigned long long kSpinTimeoutNs = 2000000000ull;
__device__ __forceinline__ unsigned long long spin_clock_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
template <class Done>
__device__ __forceinline__ void spin_until(Done done, unsigned* error_flag, unsigned sleep_ns) {
  unsigned long long t0 = 0;
  for (unsigned polls = 0; !done(); ++polls) {
    __nanosleep(sleep_ns);
    if ((polls & 255u) == 255u) {  // the clock is only consulted now and then: the common wait is a few polls long
      const unsigned long long t = spin_clock_ns();
      if (t0 == 0) t0 = t;
      else if (t - t0 > kSpinTimeoutNs) {
        *reinterpret_cast<volatile unsigned*>(error_flag) = 1u;
        return;
      }
    }
  }
}
__device__ __forceinline__ void cta_wait_at_least(const unsigned* counter, unsigned target, unsigned* error_flag) {
  if (threadIdx.x == 0) {
    spin_until([&] { return ld_relaxed_gpu(counter) >= target; }, error_flag, 40);
    (void)ld_acquire_gpu(counter);  // the counter only grows within a pass: an acquire load here reads a value >= target
  }
  __syncthreads();
}

// Where the per-throttle partial sums of a pass live.  Buffers come in pairs indexed by pass parity: the pass that follows
// may start adding into the other buffer while readers of this one are still at work, and every pass leaves the OTHER
// parity's buffers zeroed for its successor (they were last read one whole pass ago).
// Single GPU / NCCL path: total == mine (NCCL all-reduces in place), no peers.
// Peer path: the all-reduce happens inside the pass, in the finalize tiles, without a single fence on the wire.  Once this
// rank's reconcile tiles are done, the lane that owns (throttle, field) SENDS its 64-bit partial sum to every peer as two
// 8-byte words {low half | pass number << 32} {high half | pass number << 32} into the slot that peer keeps for (this rank,
// throttle, field) -- plain posted stores over NVLink, each word atomic, each carrying its own "valid" tag -- then polls, in
// its OWN memory, the slots the peers write for the same (throttle, field), adds up, and stores the total locally.  The
// decide tiles wait for a local counter of finished finalize tiles.  (The low-latency protocol of collective libraries:
// data and flag travel in the same word, so neither side needs a system-scope fence or a round trip.)
struct PartExchange {
  unsigned long long* mine;        // this rank's partial sums of this pass (reconcile tiles RED here)
  unsigned long long* total;       // sums over all ranks (what decide / status read)
  unsigned long long* zero_mine;   // other parity: left zeroed for the next pass
  unsigned long long* slots;       // [nranks][len][2] what the peers send THIS rank for this pass parity (slot of rank r at r * len * 2)
  unsigned long long* peer_slots[7];  // the same array of peer i (mapped over NVLink)
  int peer_rank[7];
  PassSync* sync;                  // this rank's counters
  int npeers, rank;
  unsigned len;                    // (2R+1) * M values per rank
  unsigned epoch;                  // this pass's number (never 0)
};

__device__ __forceinline__ void st_relaxed_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// one 64-bit value as two self-validating words
__device__ __forceinline__ void ll_send(unsigned long long* slot, unsigned long long v, unsigned epoch) {
  const unsigned long long tag = (unsigned long long)epoch << 32;
  st_relaxed_sys_u64(slot, (v & 0xffffffffull) | tag);
  st_relaxed_sys_u64(slot + 1, (v >> 32) | tag);
}
__device__ __forceinline__ unsigned long long ll_recv(const unsigned long long* slot, unsigned epoch, unsigned* error_flag) {
  unsigned long long w0 = 0, w1 = 0;
  spin_until([&] {
    w0 = ld_relaxed_sys_u64(slot);
    w1 = ld_relaxed_sys_u64(slot + 1);
    return (unsigned)(w0 >> 32) == epoch && (unsigned)(w1 >> 32) == epoch;
  }, error_flag, 20);
  return (w0 & 0xffffffffull) | (w1 << 32);
}

// How a dependent role waits for its producer: programmatic dependent launch between separate kernels ...
struct PdlSync {
  __device__ __forceinline__ void wait_reconciled() const { pdl_wait_primary(); }
  __device__ __forceinline__ void wait_totals(const PartExchange&) const { pdl_wait_primary(); }  // k_finalize is complete: so is everything before it
  __device__ __forceinline__ void wait_matched() const {}   // same CTA: a barrier already ordered the rows
  __device__ __forceinline__ void wait_prepped() const { pdl_wait_primary(); }  // k_check's primary is k_finalize: complete, and everything before it
  __device__ __forceinline__ void signal_prepped() const {}
  __device__ __forceinline__ void signal_totals() const {}
  __device__ __forceinline__ unsigned* error_flag() const { return nullptr; }
};
// ... or counters inside the one fused kernel
struct FlagSync {
  PassSync* s;
  unsigned n_rec, n_fin, n_match;
  __device__ __forceinline__ void wait_reconciled() const { cta_wait_at_least(&s->rec_done, n_rec, &s->error); }
  // the sums of every rank are in px.total
  __device__ __forceinline__ void wait_totals(const PartExchange& px) const {
    if (px.npeers == 0) wait_reconciled();
    else cta_wait_at_least(&s->tot_done, n_fin, &s->error);
  }
  __device__ __forceinline__ void wait_matched() const { cta_wait_at_least(&s->match_done, n_match, &s->error); }
  __device__ __forceinline__ void wait_prepped() const { cta_wait_at_least(&s->prep_done, n_fin, &s->error); }
  __device__ __forceinline__ void signal_prepped() const { cta_signal(&s->prep_done); }
  __device__ __forceinline__ void signal_totals() const { cta_signal(&s->tot_done); }
  __device__ __forceinline__ unsigned* error_flag() const { return &s->error; }
};

// ---- label -> table row ---------------------------------------------------------------------------
// Exact (key,value) row, else the key's "other value" row, else the neutral row.
// Fast path: two-level direct dictionary (keydir -> valrow), two dependent loads and no probing.
// Fallback for sparse ids: open-addressing hash (label_hash() shared with kt_tables.cc), probed serially.
__device__ __noinline__ int32_t hash_lookup(const uint4* __restrict__ hash, uint32_t hash_mask, int32_t neutral, uint32_t key, uint32_t val) {
#pragma unroll 1
  for (int pass = 0; pass < 2; ++pass) {
    uint32_t slot = label_hash(key, val) & hash_mask;
#pragma unroll 1
    while (true) {
      const uint4 e = __ldg(&hash[slot]);
      if (e.x == key && e.y == val) return (int32_t)e.z;
      if ((e.x & e.y) == 0xffffffffu) break;
      slot = (slot + 1) & hash_mask;
    }
    val = 0xffffffffu;  // second pass: the key's "other value" row
  }
  return neutral;
}

// Table rows travel as BYTE offsets inside one 32-throttle word slice of the match table ("roff").
// keydir / valrow hold roffs too; kOtherRoff in valrow means "a value no requirement mentions".
constexpr uint32_t kOtherRoff = 0xfffffffeu;

// Where a lane keeps the roffs of its pod's labels: registers when L <= 8 (the common shape), else a
// shared-memory column.
template <bool REG>
struct PodRows;
template <>
struct PodRows<true> {
  uint32_t off[8];
  __device__ __forceinline__ void init(int32_t*, int, int) {}
};
template <>
struct PodRows<false> {
  uint32_t* col;  // this lane's column: col[i * stride]
  int stride;
  __device__ __forceinline__ void init(int32_t* base, int tid, int tile) { col = reinterpret_cast<uint32_t*>(base) + tid; stride = tile; }
};

template <bool REG>
__device__ __forceinline__ uint32_t rows_touch(const PodRows<REG>& r) {
  if constexpr (REG) return r.off[0] ^ r.off[7];
  else return r.col[0];
}

// Translate eight label slots (one chunk) of a pod row.  No predicates: the device label columns are
// padded to a multiple of eight slots with KT_LABEL_EMPTY, keydir has a sentinel entry at [n_keydir]
// and valrow a sentinel at [0], so every load is unconditional and the addresses are one IMAD.WIDE each.
__device__ __forceinline__ void load_labels8(const int64_t* __restrict__ lp, int64_t n, int64_t (&lab)[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    lab[k] = __ldg(lp);
    lp += n;
  }
}
// first hop: the key directory entries {other roff, vmin, vcnt, off (~0: hashed values)}
__device__ __forceinline__ void translate8_keys(const TableView& tb, const int64_t (&lab)[8], uint4 (&ke)[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint32_t key = (uint32_t)((uint64_t)lab[k] >> 32);
    ke[k] = __ldg(&tb.keydir[min(key, tb.n_keydir)]);
  }
}
// second hop: the value rows, then the (rare, serial) hashed fallback for sparse dictionary ids
__device__ __forceinline__ void translate8_rows(const TableView& tb, const int64_t (&lab)[8], const uint4 (&ke)[8], uint32_t (&out)[8]) {
  uint32_t vr[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint32_t d = (uint32_t)lab[k] - ke[k].y;
    vr[k] = __ldg(&tb.valrow[d < ke[k].z ? ke[k].w + d : 0u]);  // valrow[0] == kOtherRoff
  }
  uint32_t hashed = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    out[k] = vr[k] != kOtherRoff ? vr[k] : ke[k].x;
    hashed |= ke[k].w;
  }
  if (tb.n_keydir == 0 || (hashed >> 31)) {  // offsets never reach 2^31; the hashed flag is off = ~0
    const uint32_t row_bytes = (uint32_t)tb.TPpad * 8u;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint32_t key = (uint32_t)((uint64_t)lab[k] >> 32), val = (uint32_t)lab[k];
      if (lab[k] != KT_LABEL_EMPTY && (tb.n_keydir == 0 || ke[k].w == 0xffffffffu))
        out[k] = (uint32_t)hash_lookup(tb.hash, tb.hash_mask, tb.rows - 1, key, val) * row_bytes;
    }
  }
}
__device__ __forceinline__ void translate8(const TableView& tb, const int64_t* __restrict__ lp, int64_t n, uint32_t (&out)[8]) {
  int64_t lab[8];
  uint4 ke[8];
  load_labels8(lp, n, lab);
  translate8_keys(tb, lab, ke);
  translate8_rows(tb, lab, ke, out);
}

// labels: device columns [Lpad][n] with Lpad = L rounded up to 8.
template <bool REG>
__device__ __forceinline__ void stage_rows(const TableView& tb, const int64_t* __restrict__ labels, int64_t n, int64_t p, int L, PodRows<REG>& rows) {
  if constexpr (REG) {
    translate8(tb, labels + p, n, rows.off);
  } else {
#pragma unroll 1
    for (int i0 = 0; i0 < L; i0 += 8) {
      uint32_t o[8];
      translate8(tb, labels + (int64_t)i0 * n + p, n, o);
#pragma unroll
      for (int k = 0; k < 8; ++k) rows.col[(i0 + k) * rows.stride] = o[k];  // the column has Lpad entries
    }
  }
}

// The pass does not translate: label -> row offset is done once per (pod row, table version) by k_translate_rows, at
// upload / update / table-compile time, and the pass reads the [Lpad][n] u32 offsets (half the bytes of the label column and
// no dependent dictionary hops on the tile's critical path).
template <bool REG>
__device__ __forceinline__ void load_rows(const uint32_t* __restrict__ roff, int64_t n, int64_t p, int L, PodRows<REG>& rows) {
  const uint32_t* rp = roff + p;
  if constexpr (REG) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      rows.off[k] = __ldg(rp);
      rp += n;
    }
  } else {
    const int Lpad = (L + 7) & ~7;
#pragma unroll 4
    for (int i = 0; i < Lpad; ++i) {
      rows.col[i * rows.stride] = __ldg(rp);
      rp += n;
    }
  }
}

// Match word w (32 throttles) of one pod: OR over term planes of
//   AND_labels sat  &  (count of positive keys present == need)  &  namespace mask.
// Unmentioned / empty labels point at the neutral row (sat = ~0, pos = 0): no branches.
template <int TPC, int B, bool REG>
__device__ __forceinline__ uint32_t eval_word(const TableView& tb, const PodRows<REG>& rows, int Lpad, int ns, int w) {
  uint32_t result = 0;
  const uint32_t row_bytes = (uint32_t)tb.TPpad * 8u;
  const unsigned char* wbase = reinterpret_cast<const unsigned char*>(tb.table) + (size_t)w * tb.rows * row_bytes;
  const uint32_t* nsm = tb.nsmask + ((size_t)ns * tb.W + w) * tb.TPpad;
  const uint32_t* need = tb.need + (size_t)w * tb.TPpad * B;
#pragma unroll 1
  for (int s0 = 0; s0 < tb.TPpad; s0 += TPC) {
    uint32_t sat[TPC], cnt[TPC][B];
#pragma unroll
    for (int s = 0; s < TPC; ++s) {
      sat[s] = __ldg(&nsm[s0 + s]);
#pragma unroll
      for (int b = 0; b < B; ++b) cnt[s][b] = 0;
    }
    auto fold = [&](uint32_t off) {
      const unsigned char* e = wbase + off + s0 * 8;
      uint32_t v[TPC * 2];
      if constexpr (TPC == 2) {
        const uint4 q = __ldg(reinterpret_cast<const uint4*>(e));
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
      } else {
        const uint2 q = __ldg(reinterpret_cast<const uint2*>(e));
        v[0] = q.x; v[1] = q.y;
      }
#pragma unroll
      for (int s = 0; s < TPC; ++s) {
        sat[s] &= v[2 * s];
        uint32_t carry = v[2 * s + 1];  // ripple-add one bit into the bit-sliced counter
#pragma unroll
        for (int b = 0; b < B; ++b) {
          const uint32_t t = cnt[s][b] & carry;
          cnt[s][b] ^= carry;
          carry = t;
        }
      }
    };
    if constexpr (REG) {
#pragma unroll
      for (int i = 0; i < 8; ++i) fold(rows.off[i]);
    } else {
#pragma unroll 4
      for (int i = 0; i < Lpad; ++i) fold(rows.col[i * rows.stride]);
    }
#pragma unroll
    for (int s = 0; s < TPC; ++s) {
      uint32_t m = sat[s];
#pragma unroll
      for (int b = 0; b < B; ++b) m &= ~(cnt[s][b] ^ __ldg(&need[(s0 + s) * B + b]));
      result |= m;
    }
  }
  return result;
}

// 32x32 bit-matrix transpose across the warp: in = lane l holds row l; out = lane b holds column b.
__device__ __forceinline__ uint32_t warp_transpose32(uint32_t x, int lane) {
  uint32_t m = 0x0000ffffu;
#pragma unroll
  for (int j = 16; j >= 1; j >>= 1) {
    const uint32_t o = __shfl_xor_sync(kFull, x, j);
    x = (lane & j) ? ((x & ~m) | ((o >> j) & m)) : ((x & m) | ((o & m) << j));
    m ^= m << (j >> 1);
  }
  return x;
}

// Sum of one 64-bit value per lane (mod 2^64) with three 32-bit REDUX: 22+22+20-bit limbs cannot overflow
// when 32 lanes are added.
__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
  const uint32_t lo = __reduce_add_sync(kFull, (uint32_t)v & 0x3fffffu);
  const uint32_t mi = __reduce_add_sync(kFull, (uint32_t)(v >> 22) & 0x3fffffu);
  const uint32_t hi = __reduce_add_sync(kFull, (uint32_t)(v >> 44));
  return (unsigned long long)lo + ((unsigned long long)mi << 22) + ((unsigned long long)hi << 44);
}

// ---- bulk asynchronous copies (TMA engine, no tensor map: cp.async.bulk) completing on an mbarrier --------------------------
// One elected lane arms the barrier with the byte count and issues the copies; the data lands in shared memory without passing
// through anybody's registers and the consumers sleep on the barrier's phase instead of a scoreboard.  SASS: UBLKCP / SYNCS.
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy accesses to shared memory (earlier ST / LD of the same bytes) are ordered before the async-proxy copy that follows
__device__ __forceinline__ void proxy_fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(dst_smem)), "l"(src_gmem), "r"(bytes),
               "r"(smem_addr(bar))
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, unsigned parity) {
  unsigned done;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(done)
      : "r"(smem_addr(bar)), "r"(parity)
      : "memory");
  return done != 0;
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  while (!mbar_try_wait(bar, parity)) {}  // try_wait suspends the thread for a hardware-chosen interval by itself
}
constexpr int kMaxWarps = 8;  // of a pass CTA (TILE <= 256)

// 64-bit add into a shared-memory accumulator.  atomicAdd(unsigned long long*) on shared memory compiles to a compare-and-swap
// loop (ATOMS.CAST.SPIN); two native 32-bit adds do the same mod 2^64: the low add returns the old low word, which tells
// whether THIS add carried, and the carry travels with the high word.  (The halves are only read together after a barrier.)
__device__ __forceinline__ void smem_add_u64(unsigned long long* acc, unsigned long long v) {
  unsigned* w = reinterpret_cast<unsigned*>(acc);
  const unsigned lo = (unsigned)v;
  unsigned hi = (unsigned)(v >> 32);
  if (lo) {
    const unsigned old = atomicAdd(w, lo);
    hi += (old + lo) < old ? 1u : 0u;
  }
  if (hi) atomicAdd(w + 1, hi);
}

// Shared-memory carve-up of k_reconcile (host and device must agree).  S = accumulator slots.
__host__ __device__ inline size_t reconcile_smem_bytes(int L, int R, int S, bool reg_rows, int tile) {
  const size_t b = (size_t)R * tile * 8 + (size_t)S * R * 32 * 8 + (reg_rows ? 0 : (size_t)((L + 7) & ~7) * tile * 4) + (size_t)tile * 4 + (size_t)S * 32 * 4 * 2 +
                   (size_t)S * 4;
  return (b + 15) & ~(size_t)15;
}

// ------------------------------------------------------------------------------------------------
// k_reconcile: one lane per RUNNING pod.
//   RT  compile-time bound on R for the register accumulators (0: any R, accumulate in shared memory)
//   REG label rows in registers (L <= 8) or in a shared-memory column (any L)
//   S   per-CTA accumulator slots, one per distinct 32-throttle word the tile touches (host: from the
//       largest per-namespace word list); words beyond S go straight to HBM
// ------------------------------------------------------------------------------------------------
template <int TPC, int B, int RT, bool REG, int TILE = kTileReconcile>
__device__ __forceinline__ void reconcile_tile(const PodView& pods, const TableView& tb, int L, int R, int S, uint32_t* __restrict__ bitmap,
                                               unsigned long long* __restrict__ part /* [2R+1][M]: used, present, cnt */,
                                               unsigned char* smem_raw, int64_t tile_index, unsigned long long* trace_row = nullptr) {
  // optional stage stamps of warp 0 (kt_enable_trace): [4] the pod rows have landed, [5] first two words evaluated, [6] barrier
  // passed, [7] words + sums done, [8] sweep done
  auto stamp = [&](int k) {
    if (trace_row && threadIdx.x == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      trace_row[k] = t;
    }
  };
  long long* s_req = reinterpret_cast<long long*>(smem_raw);                                     // [R][TILE], 0 where absent
  unsigned long long* s_used = reinterpret_cast<unsigned long long*>(s_req + (size_t)R * TILE);  // [S][R][32]
  int32_t* s_rowid = reinterpret_cast<int32_t*>(s_used + (size_t)S * R * 32);                    // [L][TILE] (!REG)
  uint32_t* s_present = reinterpret_cast<uint32_t*>(s_rowid + (REG ? 0 : (size_t)((L + 7) & ~7) * TILE));     // [TILE]
  uint32_t* s_cnt = s_present + TILE;                                                            // [S][32]
  uint32_t* s_pres = s_cnt + S * 32;                                                             // [S][32]
  int* s_key = reinterpret_cast<int*>(s_pres + S * 32);                                          // [S] word index or -1

  const int tid = threadIdx.x, lane = tid & 31, wbase_pod = tid & ~31;
  const int64_t tile0 = tile_index * TILE;
  const int Wp = tb.Wp;
  const int Lpad = (L + 7) & ~7;
  const int64_t p = tile0 + tid;
  const bool valid = p < pods.n;
  const int64_t pc = valid ? p : pods.n - 1;  // clamped: every lane loads, invalid lanes are masked below
  // ---- everything the tile needs of its pod rows is requested at once: ONE trip to HBM, and nothing else is waited for
  // before the table gathers of the first two words go out
  const uint32_t winfo = __ldg(&pods.winfo[pc]);
  const uint32_t flags = valid ? __ldg(&pods.flags[pc]) : 0u;
  const int ns = __ldg(&pods.ns[pc]);
  const uint32_t present = __ldg(&pods.present[pc]);
  PodRows<REG> rows;
  rows.init(s_rowid, tid, TILE);
  load_rows<REG>(pods.roff, pods.n, pc, L, rows);
  long long rq[RT > 0 ? RT : 1];
  if constexpr (RT > 0) {
    const int64_t* rp = pods.req + pc;
#pragma unroll
    for (int r = 0; r < RT; ++r) {
      rq[r] = r < R ? __ldg(rp) : 0;
      rp += pods.n;
    }
  }
  // The match bitmap is maintained, not rebuilt: a row can only ever be non-zero in the words of its namespace's list, so a
  // pass stores exactly those words (zero or not) and never touches the rest of the row -- which the engine zeroed when the
  // rows or the tables last changed (kt_engine.cu bitmap_clean).  Half of the pass's memory traffic used to be that zero-fill.
  {  // the CTA accumulators are zeroed while the loads are in flight
    if (pods.zero_fill) {  // first pass over new rows / new tables: the tile's bitmap rows (contiguous: pod-major) as well
      const int64_t rows_here = pods.n - tile0 < TILE ? pods.n - tile0 : TILE;
      uint4* dst = reinterpret_cast<uint4*>(bitmap + tile0 * Wp);
      const int nvec = (int)rows_here * (Wp / 4);
      for (int i = tid; i < nvec; i += TILE) dst[i] = make_uint4(0, 0, 0, 0);
    }
    for (int i = tid; i < S * R * 32; i += TILE) s_used[i] = 0ull;
    for (int i = tid; i < S * 32; i += TILE) { s_cnt[i] = 0u; s_pres[i] = 0u; }
    if (tid < S) s_key[tid] = -1;
  }
  // shouldCountIn (throttle_controller.go:217-219): schedulerName == target && nodeName != ""
  const bool counted = (flags & (KT_POD_SCHEDULER_MATCH | KT_POD_SCHEDULED)) == (KT_POD_SCHEDULER_MATCH | KT_POD_SCHEDULED) &&
                       (unsigned)ns < (unsigned)tb.NS;
  const bool alive = counted && (flags & KT_POD_NOT_FINISHED);  // isNotFinished (pod_util.go:26-28)
  WordCursor wc;
  wc.init(tb, winfo, ns, counted);
  if (trace_row && threadIdx.x == 0 && (rows_touch(rows) | winfo) == 0x12345u) trace_row[4] = 1;  // forces the loads to have landed
  stamp(4);
  // phase 1 -- the lane's first two words, back to back and independent of the other lanes (a match word only needs the
  // lane's own row): their 2 x Lpad table gathers are all in flight together
  uint32_t m0 = 0, m1 = 0;
  if (wc.inl > 0) m0 = eval_word<TPC, B, REG>(tb, rows, Lpad, ns, wc.w0);
  if (wc.inl > 1) m1 = eval_word<TPC, B, REG>(tb, rows, Lpad, ns, wc.w1);
  // ResourceAmountOfPod(p) columns -> shared memory (absent keys read as 0; presence kept separately)
  if constexpr (RT > 0) {
#pragma unroll
    for (int r = 0; r < RT; ++r)
      if (r < R) s_req[r * TILE + tid] = ((present >> r) & 1) ? rq[r] : 0;
  } else {
    const int64_t* rp = pods.req + pc;
    for (int r = 0; r < R; ++r) {
      const long long v = __ldg(rp);
      rp += pods.n;
      s_req[r * TILE + tid] = ((present >> r) & 1) ? v : 0;
    }
  }
  s_present[tid] = present & ~KT_COUNT_BIT;
  stamp(5);
  __syncthreads();  // accumulators initialised
  stamp(6);
  if (valid && wc.inl > 0) bitmap[p * Wp + wc.w0] = m0;
  if (valid && wc.inl > 1) bitmap[p * Wp + wc.w1] = m1;

  unsigned long long* part_used = part;
  unsigned long long* part_pres = part + (size_t)R * tb.M;
  unsigned long long* part_cnt = part + (size_t)2 * R * tb.M;

  // phase 2 -- the segmented sums, word by word in ascending order, warp-uniform: lanes whose namespace has word w bring
  // their match word (already known for their first two), the others idle.  Namespace-clustered rows (the reference's pod
  // informer is namespace-indexed) make this 1-3 rounds.
  int k = 0;
  int cur = wc.at(tb, 0);
#pragma unroll 1
  while (true) {
    const int w = __reduce_min_sync(kFull, cur);
    if (w == 0x7fffffff) break;
    uint32_t word = 0;
    if (cur == w) {
      if (k < wc.inl) {
        word = k == 0 ? m0 : m1;
      } else {
        word = eval_word<TPC, B, REG>(tb, rows, Lpad, ns, w);
        bitmap[p * Wp + w] = word;
      }
      ++k;
      cur = wc.at(tb, k);
    }
    const uint32_t aword = alive ? word : 0u;
    if (!__any_sync(kFull, aword != 0u)) continue;
    // used = used.Add(ResourceAmountOfPod(p)) for every matched throttle (throttle_controller.go:116-119):
    // lane b now owns throttle w*32+b and the set of this warp's pods that matched it.
    uint32_t T = warp_transpose32(aword, lane);
    int slot = -1;
    if (lane == 0) {  // open addressing from w mod S: one probe in the common case, at most S
      int s = (int)((unsigned)w % (unsigned)S);
#pragma unroll 1
      for (int probes = 0; probes < S; ++probes) {
        int k = *reinterpret_cast<volatile int*>(&s_key[s]);
        if (k == -1) k = atomicCAS(&s_key[s], -1, w);
        if (k == -1 || k == w) { slot = s; break; }
        s = s + 1 == S ? 0 : s + 1;
      }
    }
    slot = __shfl_sync(kFull, slot, 0);
    const int t = w * 32 + lane;
    if constexpr (RT > 0) {
      unsigned long long acc[RT];
#pragma unroll
      for (int r = 0; r < RT; ++r) acc[r] = 0ull;
      uint32_t cnt = 0, pres = 0;
      // Throttles that matched many of the warp's pods ("everything in the namespace", NotIn, DoesNotExist)
      // would make one lane walk up to 32 pods while the others idle: those are summed by the whole warp
      // (lane = pod again, REDUX tree), the sparse rest by their owning lane.
      const bool is_heavy = __popc(T) > kHeavyPods;
      uint32_t heavy = __ballot_sync(kFull, is_heavy);
      if (heavy) {
        unsigned long long mine[RT];
#pragma unroll
        for (int r = 0; r < RT; ++r) mine[r] = r < R ? (unsigned long long)s_req[r * TILE + tid] : 0ull;
        const uint32_t mypres = s_present[tid];
        while (heavy) {
          const int b = __ffs(heavy) - 1;
          heavy &= heavy - 1;
          const uint32_t mask = __shfl_sync(kFull, T, b);  // the pods (lanes) matched by throttle w*32+b
          const bool in = (mask >> lane) & 1;
          const uint32_t pr = __reduce_or_sync(kFull, in ? mypres : 0u);
          if (lane == b) { cnt = __popc(mask); pres = pr; }
#pragma unroll
          for (int r = 0; r < RT; ++r)
            if (r < R) {
              const unsigned long long v = in ? mine[r] : 0ull;
              const unsigned long long sum = warp_sum_u64(v);
              if (lane == b) acc[r] = sum;
            }
        }
      }
      if (!is_heavy) {
        while (T) {
          const int i = wbase_pod + __ffs(T) - 1;
          T &= T - 1;
          ++cnt;
          pres |= s_present[i];
#pragma unroll
          for (int r = 0; r < RT; ++r)
            if (r < R) acc[r] += (unsigned long long)s_req[r * TILE + i];
        }
      }
      if (cnt == 0) continue;
      if (slot >= 0) {
        atomicAdd(&s_cnt[slot * 32 + lane], cnt);
        atomicOr(&s_pres[slot * 32 + lane], pres);
#pragma unroll
        for (int r = 0; r < RT; ++r)
          if (r < R && acc[r]) smem_add_u64(&s_used[(slot * R + r) * 32 + lane], acc[r]);
      } else {  // more distinct words in this CTA than slots: straight to HBM
        atomicAdd(&part_cnt[t], (unsigned long long)cnt);
#pragma unroll
        for (int r = 0; r < RT; ++r)
          if (r < R) {
            if (acc[r]) atomicAdd(&part_used[(size_t)r * tb.M + t], acc[r]);
            if ((pres >> r) & 1) part_pres[(size_t)r * tb.M + t] = 1ull;
          }
      }
    } else {
      while (T) {
        const int i = wbase_pod + __ffs(T) - 1;
        T &= T - 1;
        const uint32_t pres = s_present[i];
        if (slot >= 0) {
          atomicAdd(&s_cnt[slot * 32 + lane], 1u);
          atomicOr(&s_pres[slot * 32 + lane], pres);
        } else {
          atomicAdd(&part_cnt[t], 1ull);
        }
        for (int r = 0; r < R; ++r) {
          const unsigned long long v = (unsigned long long)s_req[r * TILE + i];
          if (slot >= 0) {
            if (v) smem_add_u64(&s_used[(slot * R + r) * 32 + lane], v);
          } else {
            if (v) atomicAdd(&part_used[(size_t)r * tb.M + t], v);
            if ((pres >> r) & 1) part_pres[(size_t)r * tb.M + t] = 1ull;
          }
        }
      }
    }
  }
  stamp(7);
  __syncthreads();
  // CTA accumulators -> HBM partials: one RED per (throttle, resource) the tile touched.
  for (int idx = tid; idx < S * 32; idx += TILE) {
    const int slot = idx >> 5, b = idx & 31;
    const int w = s_key[slot];
    const uint32_t cnt = s_cnt[idx];
    if (w < 0 || cnt == 0) continue;
    const int t = w * 32 + b;
    atomicAdd(&part_cnt[t], (unsigned long long)cnt);
    const uint32_t pres = s_pres[idx];
    for (int r = 0; r < R; ++r) {
      const unsigned long long u = s_used[(slot * R + r) * 32 + b];
      if (u) atomicAdd(&part_used[(size_t)r * tb.M + t], u);
      if ((pres >> r) & 1) part_pres[(size_t)r * tb.M + t] = 1ull;  // idempotent flag
    }
  }
  stamp(8);
}

template <int TPC, int B, int RT, bool REG>
__global__ void __launch_bounds__(kTileReconcile, 768 / kTileReconcile) k_reconcile(PodView pods, TableView tb, int L, int R, int S, uint32_t* __restrict__ bitmap,
                                                                                    unsigned long long* __restrict__ part) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  pdl_launch_dependents();  // k_finalize / k_check may be scheduled; they wait for our completion where they need it
  reconcile_tile<TPC, B, RT, REG>(pods, tb, L, R, S, bitmap, part, smem_raw, blockIdx.x);
}

// ------------------------------------------------------------------------------------------------
// Finalize tiles: a group of G = 2^g >= R+1 lanes per throttle; lane r < R owns resource r, lane R owns the pod count.
// Two halves:
//   prep    (no dependency on the running pods, done and signalled at once) CalculateThreshold(now), the threshold
//           CheckThrottledFor uses, what is already used before this pass's sums (observed status.used in GIVEN_STATUS mode,
//           the reservations) -> one PRE-RECORD per throttle.  The decide tiles turn it into the 4-step check's constants
//           themselves, adding this pass's sums: finalize is NOT a stage of the pass's critical path.
//   status  (after the reconcile tiles) used / throttled / calculated threshold columns for the host; with peers, the
//           all-reduce: this rank's sums are ADDED into every rank's totals over NVLink (push), then the flags go up.
// ------------------------------------------------------------------------------------------------
// Pre-record of one throttle: PreHdr, int64 thrv[R] (thresholds), int64 base[R] (given used + reserved), thr_cnt, base_cnt.
struct __align__(16) PreHdr {
  uint32_t thr_has;   // threshold has resource r / KT_COUNT_BIT: has resourceCounts
  uint32_t base_has;  // `base` is present (Go map has the key / Counts != nil)
  uint32_t st_thr;    // GIVEN_STATUS: the observed status.throttled
  uint32_t flags;     // kPre*
};
constexpr uint32_t kPreLive = 1u, kPreE3 = 2u, kPreOnEqual = 4u, kPreGiven = 8u;
__host__ __device__ inline size_t pre_record_bytes(int R) { return 16 + 16 * (size_t)R + 16; }

constexpr int kFinPrep = 1, kFinStatus = 2;  // the halves of a finalize tile: the fused pass runs them as separate tiles (prep first, so
                                             // that nobody ever waits for pre-records), the chained k_finalize runs both
constexpr int kFinZero = 4;  // with kFinStatus: also zero the other parity's partial sums (k_finalize; k_pass zeroes them after its wait)

// CalculateThreshold(now) of throttle t for resource r (is_res) or the pod count: merged active overrides REPLACE
// spec.threshold; per resource name the first active override wins (throttle_types.go:65-106).  mybit is r's presence bit
// (KT_COUNT_BIT for the count), col = r * M + t.  The finalize tiles and the keyed reconcile (kt_keyed.cuh) share it.
struct CalcThreshold {
  bool spec_has, calc_has, active;
  long long spec_val, calc_val;
};
__device__ __forceinline__ CalcThreshold calculate_threshold(const ThrottleView& tv, int t, int r, bool is_res, uint32_t mybit, size_t col, long long now) {
  CalcThreshold ct;
  ct.spec_has = tv.thr_present[t] & mybit;
  ct.spec_val = is_res ? tv.thr[col] : tv.thr_cnt[t];
  ct.active = false;
  bool ov_has = false;
  long long ov_val = 0;
  const int o_lo = tv.ovr_off[t], o_hi = tv.ovr_off[t + 1];
  for (int i = o_lo; i < o_hi; ++i) {
    if (tv.ovr_flags[i] & KT_OVR_PARSE_ERROR) continue;               // skipped, reported in Messages by the host
    if (!(tv.ovr_begin[i] <= now && now <= tv.ovr_end[i])) continue;  // IsActive: inclusive both ends
    ct.active = true;
    if (!ov_has && (tv.ovr_present[i] & mybit)) {
      ov_has = true;
      ov_val = is_res ? tv.ovr_thr[(size_t)r * tv.n_ovr + i] : tv.ovr_cnt[i];
    }
  }
  ct.calc_has = ct.active ? ov_has : ct.spec_has;
  ct.calc_val = ct.active ? ov_val : ct.spec_val;
  return ct;
}

template <class Sync>
__device__ __forceinline__ void finalize_tile(const ThrottleView& tv, int M, int R, int G, long long now, uint32_t eval_flags, const PartExchange& px,
                                              const ReconcileView& out, unsigned char* __restrict__ pre /* [M][pre_record_bytes(R)] */, int tile_index,
                                              const Sync& sync, unsigned long long* trace_row = nullptr, int halves = kFinPrep | kFinStatus | kFinZero) {
  // optional stage stamps (kt_enable_trace): [4] pre-records written; [5] this rank's reconcile tiles done; [6] sums of every
  // rank read; [7] status columns written
  auto stamp = [&](int k) {
    if (trace_row && threadIdx.x == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      trace_row[k] = t;
    }
  };
  const int gid = tile_index * (int)blockDim.x + (int)threadIdx.x;
  const int lane = threadIdx.x & 31;
  const int t = gid / G, r = gid % G;  // G divides 32: a group never straddles a warp
  const int gbase = lane - r;          // first lane of this group inside the warp
  const bool given = eval_flags & KT_EVAL_GIVEN_STATUS;
  const bool on_equal = eval_flags & KT_EVAL_ON_EQUAL;
  const bool in_range = t < M;
  const bool is_res = in_range && r < R, is_cnt = in_range && r == R;
  const uint32_t mybit = r < R ? (1u << r) : KT_COUNT_BIT;
  const size_t col = (size_t)r * M + t;  // resource lanes: index into [R][M] columns
  const size_t i_val = is_res ? col : (size_t)2 * R * M + t;  // this lane's sum in a partial-sum buffer
  const size_t i_has = (size_t)(R + r) * M + t;               // resource lanes: its presence flag

  // the other parity's buffers are left zeroed for the next pass
  if (halves & kFinZero) {
    if (is_res) {
      px.zero_mine[col] = 0ull;
      px.zero_mine[i_has] = 0ull;
    } else if (is_cnt) {
      px.zero_mine[i_val] = 0ull;
    }
  }

  uint32_t tflags = 0;
  bool spec_has = false, calc_has = false, active_found = false;
  long long spec_val = 0, calc_val = 0;
  if (is_res || is_cnt) {
    tflags = tv.flags[t];
    const CalcThreshold ct = calculate_threshold(tv, t, r, is_res, mybit, col, now);
    spec_has = ct.spec_has; spec_val = ct.spec_val; calc_has = ct.calc_has; calc_val = ct.calc_val; active_found = ct.active;
  }
  // the threshold CheckThrottledFor compares with (throttle_types.go:128-132): this pass's, or -- GIVEN_STATUS, what
  // PreFilter sees -- the informer copy's status.calculatedThreshold when calculatedAt is set, else spec.threshold
  bool thr_has = calc_has, base_has = false, g_st_thr = false;
  long long thr = calc_val, base = 0;
  if (given && (is_res || is_cnt)) {
    if (tv.st_calculated[t]) {
      thr_has = tv.st_calc_present[t] & mybit;
      thr = is_res ? tv.st_calc_thr[col] : tv.st_calc_cnt[t];
    } else {
      thr_has = spec_has;
      thr = spec_val;
    }
    if (tv.st_used_present[t] & mybit) {  // alreadyUsed starts from status.used ...
      base_has = true;
      base = is_res ? tv.st_used[col] : tv.st_used_cnt[t];
    }
    g_st_thr = tv.st_throttled[t] & mybit;
  }
  if ((is_res || is_cnt) && tv.reserved_present && (tv.reserved_present[t] & mybit)) {  // ... + reserved: presence is the union
    base_has = true;
    base += is_res ? (tv.reserved ? tv.reserved[col] : 0) : (tv.reserved_cnt ? tv.reserved_cnt[t] : 0);
  }
  const bool is_throttle_kind = in_range ? tv.kind[t] == KT_KIND_THROTTLE : true;
  const bool live = (tflags & KT_THR_RESPONSIBLE) && !(tflags & KT_THR_SELECTOR_ERROR);

  // ---- per-throttle masks: one ballot each, bit (lane - gbase) = resource r, bit R = count ----
  const uint32_t gmask = G == 32 ? 0xffffffffu : ((1u << G) - 1u);
  const uint32_t rmask = (R == 32 ? 0xffffffffu : ((1u << R) - 1u));
  auto group_mask = [&](bool pred) -> uint32_t {
    const uint32_t g = (__ballot_sync(kFull, pred) >> gbase) & gmask;
    return (g & rmask) | (((g >> R) & 1u) ? KT_COUNT_BIT : 0u);
  };
  if (halves & kFinPrep) {
    const uint32_t m_thr = group_mask(thr_has), m_base = group_mask(base_has), m_st = group_mask(g_st_thr);
    unsigned char* rec = pre + (size_t)t * pre_record_bytes(R);
    long long* vals = reinterpret_cast<long long*>(rec + 16);  // thrv[R], base[R], thr_cnt, base_cnt
    if (is_res) {
      vals[r] = thr;
      vals[R + r] = base;
    } else if (is_cnt) {
      PreHdr h;
      h.thr_has = m_thr;
      h.base_has = m_base;
      h.st_thr = m_st;
      // Q1: S3 compares with >= for a Throttle whatever the caller says (throttle_types.go:143), a ClusterThrottle passes
      // isThrottledOnEqual on (clusterthrottle_types.go:45)
      h.flags = (live ? kPreLive : 0u) | ((is_throttle_kind || on_equal) ? kPreE3 : 0u) | (on_equal ? kPreOnEqual : 0u) | (given ? kPreGiven : 0u);
      *reinterpret_cast<PreHdr*>(rec) = h;
      vals[2 * R] = thr;
      vals[2 * R + 1] = base;
    }
    sync.signal_prepped();
    stamp(4);
    if (!(halves & kFinStatus)) return;
  }

  sync.wait_reconciled();  // this rank's partial sums are complete and visible
  stamp(5);
  // ---- used (this pass): resource lanes read sum + presence flag, the count lane the pod count.  With peers the
  // all-reduce happens right here, as a push: the lane adds its value into every rank's totals ----
  long long used_val = 0;
  bool used_has = false;
  if (is_res || is_cnt) {
    unsigned long long v = __ldcg(&px.mine[i_val]);
    unsigned long long h = is_res ? __ldcg(&px.mine[i_has]) : 0ull;
    if (px.npeers > 0) {
      // send first (to every peer), then receive: nobody waits for anybody before its own values are on the wire
#pragma unroll 1
      for (int i = 0; i < px.npeers; ++i) {
        unsigned long long* slot = px.peer_slots[i] + ((size_t)px.rank * px.len + i_val) * 2;
        ll_send(slot, v, px.epoch);
        if (is_res) ll_send(px.peer_slots[i] + ((size_t)px.rank * px.len + i_has) * 2, h, px.epoch);
      }
#pragma unroll 1
      for (int i = 0; i < px.npeers; ++i) {
        v += ll_recv(px.slots + ((size_t)px.peer_rank[i] * px.len + i_val) * 2, px.epoch, sync.error_flag());
        if (is_res) h += ll_recv(px.slots + ((size_t)px.peer_rank[i] * px.len + i_has) * 2, px.epoch, sync.error_flag());
      }
      px.total[i_val] = v;
      if (is_res) px.total[i_has] = h;
    }
    used_val = (long long)v;
    used_has = is_res ? h != 0ull : used_val > 0;  // Counts stays nil with zero counted pods (Q3)
  }
  if (px.npeers > 0) sync.signal_totals();  // the decide tiles read px.total
  if (trace_row && threadIdx.x == 0 && used_val == 0x7fffffffffffffffll) trace_row[6] = 1;  // the loads have landed
  stamp(6);
  // status.throttled = calculatedThreshold.IsThrottled(used, onEqual=true) (throttle_controller.go:133)
  const bool throttled = live && calc_has && used_has && used_val >= calc_val;
  const uint32_t m_used = group_mask(used_has);
  const uint32_t m_throttled = group_mask(throttled);
  const uint32_t m_calc = group_mask(calc_has);
  if (is_res) {
    if (out.used) out.used[col] = used_val;
    if (out.calc_thr) out.calc_thr[col] = calc_val;
  } else if (is_cnt) {
    if (out.used_cnt) out.used_cnt[t] = used_val;
    if (out.calc_cnt) out.calc_cnt[t] = calc_val;
    if (out.used_present) out.used_present[t] = m_used;
    if (out.throttled) out.throttled[t] = m_throttled;
    if (out.calc_present) out.calc_present[t] = m_calc;
    if (out.override_active) out.override_active[t] = active_found;
  }
  if (out.changed_count) {  // uniform across the grid
    // what reconcile would write differs from the informer copy?  (Messages / calculatedAt are the host's business.)
    bool diff = false;
    if (live && (is_res || is_cnt)) {
      const bool o_used_has = tv.st_used_present[t] & mybit, o_thr = tv.st_throttled[t] & mybit;
      const long long o_used = is_res ? tv.st_used[col] : tv.st_used_cnt[t];
      diff = used_has != o_used_has || (used_has && used_val != o_used) || throttled != o_thr;
      if (!tv.st_calculated[t]) {
        diff = true;  // calculatedThreshold was never written: this reconcile stamps it
      } else {
        const bool o_calc_has = tv.st_calc_present[t] & mybit;
        const long long o_calc = is_res ? tv.st_calc_thr[col] : tv.st_calc_cnt[t];
        diff = diff || calc_has != o_calc_has || (calc_has && calc_val != o_calc);
      }
    }
    const uint32_t m_diff = group_mask(diff);
    if (is_cnt) {
      out.changed_flag[t] = m_diff != 0u;
      if (m_diff) out.changed_idx[atomicAdd(out.changed_count, 1u)] = t;
    }
    if (tile_index == 0 && threadIdx.x == 0) *out.changed_count_next = 0u;
  }
  stamp(7);
}

__global__ void __launch_bounds__(128) k_finalize(ThrottleView tv, int M, int R, int G, long long now, uint32_t eval_flags, PartExchange px,
                                                  ReconcileView out, unsigned char* __restrict__ pre) {
  pdl_launch_dependents();  // k_check can start matching the pending pods right away
  finalize_tile(tv, M, R, G, now, eval_flags, px, out, pre, blockIdx.x, PdlSync{});
}

// ------------------------------------------------------------------------------------------------
// k_check: one lane per PENDING pod.  Phase 1 (no dependency on the running pods): selector match ->
// affectedThrottles bitmap.  Phase 2 (after k_finalize): 4-step CheckThrottledFor per matched pair; the
// constants of a word's 32 throttles are staged in shared memory by the warp (lane = throttle) so the
// per-pair work is shared-memory compares instead of dependent global gathers.
// ------------------------------------------------------------------------------------------------
// Decide tiles stage the check constants of the words their pods touch ONCE PER CTA: every warp proposes up to KS words per
// round, the CTA's distinct words get one staging slot each (32 throttle records), the slots are spread over the warps.
__host__ __device__ inline size_t decide_record_bytes(int R) { return 16 + 16 * (size_t)R + 16; }  // == pre_record_bytes: staged raw, finished in place
__host__ __device__ inline int decide_stage_words(int R, int tile) {
  return (size_t)(tile / 32) * 2 * 32 * decide_record_bytes(R) <= (48u << 10) ? 2 : 1;
}
__host__ __device__ inline size_t check_smem_bytes(int L, int R, bool reg_rows, int tile) {
  const size_t match = reg_rows ? 0 : (size_t)((L + 7) & ~7) * tile * 4;                                                        // check_match_tile
  const int slots = (tile / 32) * decide_stage_words(R, tile);
  const size_t decide = (size_t)R * tile * 8 + (size_t)slots * 32 * decide_record_bytes(R) + (size_t)slots * 8 + 16;             // check_decide_tile
  return match > decide ? match : decide;
}

// Optional sparse copy of the check result (kt_set_sparse_check): every NON-ZERO 32-bit code word is also appended to a list
// as {pending row, word index within the row's 2*Wp code words, the 16 codes}.  At C2 that is ~10k entries (116 KB) where the
// dense code rows are 2.56 MB, which is what a host that only needs the reasons of the rejected pods wants to download.
// count keeps counting beyond cap (the host then falls back to the dense rows); entries are unordered.
struct SparseOut {
  uint32_t* count;  // nullptr: off
  uint32_t* ent;    // [cap][3]
  uint32_t cap;
};
__device__ __forceinline__ void sparse_append(const SparseOut& sp, uint32_t row, uint32_t widx, uint32_t word) {
  const uint32_t i = atomicAdd(sp.count, 1u);
  if (i < sp.cap) {
    sp.ent[3 * (size_t)i] = row;
    sp.ent[3 * (size_t)i + 1] = widx;
    sp.ent[3 * (size_t)i + 2] = word;
  }
}

// Phase 1 of the pending check, no dependency on the running pods: selector match of TILE pending pods ->
// affectedThrottles bitmap rows (throttle_controller.go:248-269); also clears the tile's code rows.
template <int TPC, int B, bool REG, int TILE>
__device__ __forceinline__ void check_match_tile(const PodView& pods, const TableView& tb, int L, uint32_t* __restrict__ bitmap,
                                                 uint32_t* __restrict__ codes, unsigned char* smem_raw, int64_t tile_index) {
  int32_t* s_rowid = reinterpret_cast<int32_t*>(smem_raw);  // [Lpad][TILE] (!REG)
  const int tid = threadIdx.x;
  const int64_t tile0 = tile_index * TILE;
  const int Wp = tb.Wp;
  const int Lpad = (L + 7) & ~7;
  const int64_t p = tile0 + tid;
  const bool valid = p < pods.n;
  const int64_t pc = valid ? p : pods.n - 1;  // clamped: every lane loads, invalid lanes never store
  const uint32_t winfo = __ldg(&pods.winfo[pc]);
  const int ns = valid ? __ldg(&pods.ns[pc]) : -1;
  PodRows<REG> rows;
  rows.init(s_rowid, tid, TILE);
  load_rows<REG>(pods.roff, pods.n, pc, L, rows);
  // neither the bitmap rows nor the code rows are zero-filled pass after pass: both are maintained word by word (see
  // reconcile_tile) -- except on the first pass over new rows / new tables
  if (pods.zero_fill) {
    const int64_t rows_here = pods.n - tile0 < TILE ? pods.n - tile0 : TILE;
    uint4* d0 = reinterpret_cast<uint4*>(bitmap + tile0 * Wp);
    uint4* d1 = reinterpret_cast<uint4*>(codes + tile0 * 2 * Wp);
    const int nvec = (int)rows_here * (Wp / 4);
    for (int i = tid; i < nvec; i += TILE) d0[i] = make_uint4(0, 0, 0, 0);
    for (int i = tid; i < 2 * nvec; i += TILE) d1[i] = make_uint4(0, 0, 0, 0);
  }
  WordCursor wc;
  wc.init(tb, winfo, ns, valid && (unsigned)ns < (unsigned)tb.NS);
  uint32_t m0 = 0, m1 = 0;  // the first two words: all their table gathers in flight together
  if (wc.inl > 0) m0 = eval_word<TPC, B, REG>(tb, rows, Lpad, ns, wc.w0);
  if (wc.inl > 1) m1 = eval_word<TPC, B, REG>(tb, rows, Lpad, ns, wc.w1);
  if (pods.zero_fill) __syncthreads();  // zero-fill before the word stores (rows of a tile are zeroed by all its lanes)
  if (wc.inl > 0) bitmap[p * Wp + wc.w0] = m0;
  if (wc.inl > 1) bitmap[p * Wp + wc.w1] = m1;
#pragma unroll 1
  for (int k = wc.inl; k < wc.cnt; ++k) {
    const int w = wc.at(tb, k);
    bitmap[p * Wp + w] = eval_word<TPC, B, REG>(tb, rows, Lpad, ns, w);
  }
}

// Phase 2: the 4-step CheckThrottledFor per (pending pod, affected throttle), 2-bit codes and the admit bit.
// Everything that does not depend on the reconcile is done before the wait: the pod's requests and match words, which
// words the CTA needs, and the PRE-RECORDS of those words' throttles (thresholds, observed status, reservations) copied
// into the CTA's staging slots.  After the wait one lane per (slot, throttle) fetches that throttle's sums -- one trip to
// L2 for the whole CTA -- and finishes the record in place (what a finalize stage between reconcile and decide used to
// hand over); then every lane decides its own pairs from shared memory.
//
// The building blocks, shared by the two decide tiles below (lane = pod: check_decide_tile; four lanes per pod, one per word:
// check_decide_quad).

// What a decide lane knows of its pod: the non-zero requests (IsThrottledFor only looks at those, Q5) and where they sit.
struct DecidePod {
  const long long* req;  // &s_req[column of this pod]; resource r at req[r * stride]
  int stride;
  uint32_t nz;
  int64_t p;             // pending row
};

// one lane's verdicts on (some of) the throttles of one word, from the finished records of its slot: 2-bit codes, low / high half
template <int RT>
__device__ __forceinline__ uint2 decide_word_codes(uint32_t word, const unsigned char* recs, size_t rec, int R, const DecidePod& pod) {
  uint32_t c0 = 0, c1 = 0;
  const uint32_t nz = pod.nz;
  while (word) {
    const int b = __ffs(word) - 1;
    word &= word - 1;
    const unsigned char* cb = recs + (size_t)b * rec;
    const uint4 hq = *reinterpret_cast<const uint4*>(cb);
    const long long* thrv = reinterpret_cast<const long long*>(cb + 16);
    const long long* head = thrv + R;
    const uint32_t cand = nz & hq.x;
    uint32_t code;
    bool s1 = hq.w & 1u, s4 = hq.w & 8u;  // the count lane's share of S1 / S4
    const bool ge = hq.w & 16u;
    // S1 threshold.IsThrottled(podAmount, false).IsThrottledFor(pod); S4 used + pod + reserved against the threshold
    for (uint32_t c = cand; c && !s1;) {
      const int r = __ffs(c) - 1;
      c &= c - 1;
      s1 = pod.req[r * pod.stride] > thrv[r];
    }
    for (uint32_t c = cand; c && !s4;) {
      const int r = __ffs(c) - 1;
      c &= c - 1;
      const long long v = pod.req[r * pod.stride];
      const long long hd = head[r];
      s4 = ge ? v >= hd : v > hd;
    }
    if (s1) code = KT_CHECK_POD_REQUESTS_EXCEEDS_THRESHOLD;
    else if ((hq.w & 2u) || (nz & hq.y)) code = KT_CHECK_ACTIVE;   // S2 status.throttled.IsThrottledFor(pod)
    else if ((hq.w & 4u) || (nz & hq.z)) code = KT_CHECK_ACTIVE;   // S3 used+reserved already over
    else code = s4 ? KT_CHECK_INSUFFICIENT : KT_CHECK_NOT_THROTTLED;
    if (b < 16) c0 |= code << (2 * b);
    else c1 |= code << (2 * (b - 16));
  }
  return make_uint2(c0, c1);
}
// the code words of (pending row, word w) go out -- unconditionally: the code rows are maintained word by word, a pair that was
// rejected by the previous pass and is not any more must read 0 again (codes can only be non-zero where match bits are, and
// those do not move between passes)
__device__ __forceinline__ void store_codes(uint2 c, int w, int Wp, int64_t p, uint32_t* __restrict__ codes, const SparseOut& sp, unsigned char& ok) {
  if (c.x | c.y) ok = 0;
  *reinterpret_cast<uint2*>(&codes[p * 2 * Wp + 2 * w]) = c;
  if (sp.count) {
    if (c.x) sparse_append(sp, (uint32_t)p, (uint32_t)(2 * w), c.x);
    if (c.y) sparse_append(sp, (uint32_t)p, (uint32_t)(2 * w + 1), c.y);
  }
}
template <int RT>
__device__ __forceinline__ void decide_word(uint32_t word, int w, const unsigned char* recs, size_t rec, int R, int Wp, const DecidePod& pod,
                                            uint32_t* __restrict__ codes, const SparseOut& sp, unsigned char& ok) {
  store_codes(decide_word_codes<RT>(word, recs, rec, R, pod), w, Wp, pod.p, codes, sp, ok);
}

// lane = throttle of word w: the raw pre-record into the staging slot (nothing here depends on the running pods)
__device__ __forceinline__ void stage_pre_record(const unsigned char* __restrict__ pre, int w, uint32_t any, unsigned char* slot_recs, size_t rec, int R, int lane) {
  if (w < 0 || !((any >> lane) & 1)) return;
  const uint4* src = reinterpret_cast<const uint4*>(pre + (size_t)(w * 32 + lane) * rec);  // written earlier in this launch by another SM:
  uint4* dst = reinterpret_cast<uint4*>(slot_recs + (size_t)lane * rec);                   // __ldcg, L2 is the point of coherence
  for (int q = 0; q < R + 2; ++q) dst[q] = __ldcg(&src[q]);
}
// ... and, once the sums exist, the constants of CheckThrottledFor (throttle_types.go:128-153 / clusterthrottle_types.go:30-55)
// in place.  alreadyUsed = status.used + reserved (absent values are 0, presence is the union); in GIVEN_STATUS mode
// status.used and status.throttled are the observed ones and the sums are not looked at.
__device__ __forceinline__ void stage_finish_record(const PartExchange& px, int w, uint32_t any, unsigned char* slot_recs, size_t rec, int R, int M, int lane) {
  if (w < 0 || !((any >> lane) & 1)) return;
  const int t = w * 32 + lane;
  unsigned char* dst = slot_recs + (size_t)lane * rec;
  long long* vals = reinterpret_cast<long long*>(dst + 16);  // thrv[R], base[R] -> head[R], thr_cnt, base_cnt
  const PreHdr ph = *reinterpret_cast<const PreHdr*>(dst);
  const bool live = ph.flags & kPreLive, e3 = ph.flags & kPreE3, on_equal = ph.flags & kPreOnEqual, given = ph.flags & kPreGiven;
  const long long c_used = given ? 0 : (long long)__ldcg(&px.total[(size_t)2 * R * M + t]);
  CheckHdr h;
  h.thr_has = h.m2 = h.m3 = 0;
#pragma unroll 1
  for (int r0 = 0; r0 < R; r0 += kStageChunk) {
    unsigned long long used[kStageChunk], uhas[kStageChunk];
#pragma unroll
    for (int q = 0; q < kStageChunk; ++q) {
      const int r = r0 + q < R ? r0 + q : R - 1;  // clamped: the loads stay unconditional and in flight together
      used[q] = given ? 0ull : __ldcg(&px.total[(size_t)r * M + t]);
      uhas[q] = given ? 0ull : __ldcg(&px.total[(size_t)(R + r) * M + t]);
    }
#pragma unroll
    for (int q = 0; q < kStageChunk; ++q) {
      const int r = r0 + q;
      if (r < R) {
        const long long thr = vals[r];
        long long au = vals[R + r];
        const bool has = (ph.thr_has >> r) & 1;
        bool au_has = (ph.base_has >> r) & 1, m2 = (ph.st_thr >> r) & 1;
        if (!given) {
          const bool used_has = uhas[q] != 0ull;
          au += (long long)used[q];
          au_has = au_has || used_has;
          m2 = has && used_has && (long long)used[q] >= thr;  // status.throttled of THIS pass: IsThrottled(used, onEqual = true)
        }
        const bool s3 = has && au_has && (e3 ? au >= thr : au > thr);
        vals[R + r] = thr - au;  // head: S4 used + reserved + pod (>|>=) threshold  <=>  pod (>|>=) head
        h.thr_has |= (has ? 1u : 0u) << r;
        h.m2 |= (m2 ? 1u : 0u) << r;
        h.m3 |= (s3 ? 1u : 0u) << r;
      }
    }
  }
  {  // the pod count: the pending pod itself counts 1
    const long long thr = vals[2 * R];
    long long au = vals[2 * R + 1];
    const bool has = ph.thr_has & KT_COUNT_BIT;
    bool au_has = ph.base_has & KT_COUNT_BIT, m2 = ph.st_thr & KT_COUNT_BIT;
    if (!given) {
      const bool used_has = c_used > 0;  // Counts stays nil with zero counted pods (Q3)
      au += c_used;
      au_has = au_has || used_has;
      m2 = has && used_has && c_used >= thr;
    }
    const bool s1 = has && 1 > thr;                                           // S1: pod count 1 > threshold (Q4)
    const bool s3 = has && au_has && (e3 ? au >= thr : au > thr);
    const bool s4 = has && (on_equal ? au + 1 >= thr : au + 1 > thr);         // S4 (counts always present: the pod)
    h.cntbits = (on_equal ? 16u : 0u) | (s1 ? 1u : 0u) | (m2 ? 2u : 0u) | (s3 ? 4u : 0u) | (s4 ? 8u : 0u);
  }
  if (!live) { h.thr_has = h.m2 = h.m3 = 0; h.cntbits &= 16u; }
  *reinterpret_cast<CheckHdr*>(dst) = h;
}

// One pair checked straight from L2 (pre-record + sums), no staging: for the pairs whose word found no staging slot (rows in
// ARRIVAL order: a different namespace in every lane).  The same 4 steps.
__device__ __forceinline__ uint32_t decide_pair_direct(const unsigned char* __restrict__ pre, const PartExchange& px, size_t rec, int R, int M, int t,
                                                       const DecidePod& pod) {
  const unsigned char* src = pre + (size_t)t * rec;
  const uint4 phq = __ldcg(reinterpret_cast<const uint4*>(src));
  const long long* pv = reinterpret_cast<const long long*>(src + 16);  // thrv[R], base[R], thr_cnt, base_cnt
  PreHdr ph;
  ph.thr_has = phq.x; ph.base_has = phq.y; ph.st_thr = phq.z; ph.flags = phq.w;
  if (!(ph.flags & kPreLive)) return KT_CHECK_NOT_THROTTLED;
  const bool e3 = ph.flags & kPreE3, on_equal = ph.flags & kPreOnEqual, given = ph.flags & kPreGiven;
  bool s1, s2, s3, s4;
  {  // the pod count: the pending pod itself counts 1
    const long long thr = __ldcg(&pv[2 * R]);
    long long au = __ldcg(&pv[2 * R + 1]);
    const bool has = ph.thr_has & KT_COUNT_BIT;
    bool au_has = ph.base_has & KT_COUNT_BIT, m2 = ph.st_thr & KT_COUNT_BIT;
    if (!given) {
      const long long used = (long long)__ldcg(&px.total[(size_t)2 * R * M + t]);
      const bool used_has = used > 0;
      au += used;
      au_has = au_has || used_has;
      m2 = has && used_has && used >= thr;
    }
    s1 = has && 1 > thr;
    s2 = m2;
    s3 = has && au_has && (e3 ? au >= thr : au > thr);
    s4 = has && (on_equal ? au + 1 >= thr : au + 1 > thr);
  }
  for (uint32_t c = pod.nz; c;) {  // IsThrottledFor only looks at the pod's non-zero requests (Q5)
    const int r = __ffs(c) - 1;
    c &= c - 1;
    const long long thr = __ldcg(&pv[r]);
    long long au = __ldcg(&pv[R + r]);
    const bool has = (ph.thr_has >> r) & 1;
    bool au_has = (ph.base_has >> r) & 1, m2 = (ph.st_thr >> r) & 1;
    if (!given) {
      const long long used = (long long)__ldcg(&px.total[(size_t)r * M + t]);
      const bool used_has = __ldcg(&px.total[(size_t)(R + r) * M + t]) != 0ull;
      au += used;
      au_has = au_has || used_has;
      m2 = has && used_has && used >= thr;
    }
    const long long v = pod.req[r * pod.stride];
    s1 = s1 || (has && v > thr);
    s2 = s2 || m2;
    s3 = s3 || (has && au_has && (e3 ? au >= thr : au > thr));
    s4 = s4 || (has && (on_equal ? v >= thr - au : v > thr - au));
  }
  return s1 ? KT_CHECK_POD_REQUESTS_EXCEEDS_THRESHOLD : ((s2 || s3) ? KT_CHECK_ACTIVE : (s4 ? KT_CHECK_INSUFFICIENT : KT_CHECK_NOT_THROTTLED));
}
// ... a whole word of such pairs
__device__ __forceinline__ uint2 decide_word_direct_codes(uint32_t word, int w, const unsigned char* __restrict__ pre, const PartExchange& px, size_t rec, int R,
                                                          int M, const DecidePod& pod) {
  uint32_t c0 = 0, c1 = 0;
  while (word) {
    const int b = __ffs(word) - 1;
    word &= word - 1;
    const uint32_t code = decide_pair_direct(pre, px, rec, R, M, w * 32 + b, pod);
    if (b < 16) c0 |= code << (2 * b);
    else c1 |= code << (2 * (b - 16));
  }
  return make_uint2(c0, c1);
}

// the same out of line (everything by value: nothing of the caller has to live in local memory for it): the shared decide
// tiles take this path only for words that found no staging slot, and keep their own code short
__device__ __noinline__ uint2 decide_word_direct_far(uint32_t word, int w, const unsigned char* __restrict__ pre, unsigned long long* total, unsigned rec, int R, int M,
                                                     const long long* req, int stride, uint32_t nz) {
  PartExchange px{};
  px.total = total;
  const DecidePod pod{req, stride, nz, 0};
  return decide_word_direct_codes(word, w, pre, px, rec, R, M, pod);
}

template <int TILE, int RT, class Sync>
__device__ __forceinline__ void check_decide_tile(const PodView& pods, const TableView& tb, int R, int KS, const unsigned char* __restrict__ pre,
                                                  const PartExchange& px, const uint32_t* __restrict__ bitmap, uint32_t* __restrict__ codes,
                                                  unsigned char* __restrict__ admit, unsigned char* smem_raw, int64_t tile_index, const Sync& sync,
                                                  const SparseOut sp = SparseOut{nullptr, nullptr, 0}, unsigned long long* trace_row = nullptr) {
  // optional stage stamps (kt_enable_trace): [4] match rows visible, [5] words claimed + pre-records staged, [6] sums of every
  // rank visible, [7] constants finished, [8] decided
  auto stamp = [&](int k) {
    if (trace_row && threadIdx.x == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      trace_row[k] = t;
    }
  };
  constexpr int WARPS = TILE / 32;
  const size_t rec = decide_record_bytes(R);  // per throttle: CheckHdr (PreHdr while raw), thrv[R], head[R] (base[R] while raw), thr_cnt, base_cnt
  const int SLOTS = WARPS * KS;
  long long* s_req = reinterpret_cast<long long*>(smem_raw);                          // [R][TILE]
  unsigned char* s_chk = reinterpret_cast<unsigned char*>(s_req + (size_t)R * TILE);  // [SLOTS][32][rec]
  int* s_key = reinterpret_cast<int*>(s_chk + (size_t)SLOTS * 32 * rec);              // [SLOTS] word index or -1
  uint32_t* s_any = reinterpret_cast<uint32_t*>(s_key + SLOTS);                       // [SLOTS] throttles of the word some lane of the CTA matched
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int Wp = tb.Wp;
  const int M = tb.M;
  const int64_t p = tile_index * TILE + tid;
  const bool valid = p < pods.n;
  const int64_t pc = valid ? p : pods.n - 1;
  const int ns = valid ? __ldg(&pods.ns[pc]) : -1;
  const uint32_t present = __ldg(&pods.present[pc]);
  const uint32_t winfo = __ldg(&pods.winfo[pc]);
  // ResourceAmountOfPod(pod): the non-zero requests are the only ones IsThrottledFor looks at (Q5)
  uint32_t nz = 0;
  {
    const int64_t* rp = pods.req + pc;
    for (int r = 0; r < R; ++r) {
      long long v = __ldg(rp);
      rp += pods.n;
      if (!((present >> r) & 1)) v = 0;
      s_req[r * TILE + tid] = v;
      if (v != 0) nz |= 1u << r;
    }
  }
  const DecidePod pod{s_req + tid, TILE, nz, p};
  if (tid < SLOTS) { s_key[tid] = -1; s_any[tid] = 0u; }
  WordCursor wc;
  wc.init(tb, winfo, ns, valid && (unsigned)ns < (unsigned)tb.NS);
  __syncthreads();  // the slot table is initialised
  sync.wait_matched();
  sync.wait_prepped();  // the pre-records are written (early: they depend on nothing)
  stamp(4);

  unsigned char ok = 1;
  int k = 0;
  int cur = wc.at(tb, 0);
  bool sums_awaited = false;

#pragma unroll 1
  while (true) {
    // 1. every warp's next words in its warp-uniform order -- up to kPropose of them, as long as the CTA's slot table has room
    // (open addressing; a word another warp already claimed costs nothing).  Warps of one namespace share their slots, so a
    // namespace with three or four words is still ONE round.
    int pw[kPropose], pslot[kPropose];
    uint32_t pword[kPropose];
    {
      int tk = k, tcur = cur;
      uint32_t mine = 0;  // rounds q in which this lane's next word is the warp's
#pragma unroll
      for (int q = 0; q < kPropose; ++q) {
        pw[q] = __reduce_min_sync(kFull, tcur);
        pslot[q] = -1;
        pword[q] = 0;
        if (pw[q] != 0x7fffffff && tcur == pw[q]) {
          mine |= 1u << q;
          ++tk;
          tcur = wc.at(tb, tk);
        }
      }
      int nq = 0;
      if (lane == 0) {
        bool open = true;  // (unrolled with a flag instead of a counted loop: pw / pslot stay in registers)
#pragma unroll
        for (int q = 0; q < kPropose; ++q) {
          if (open && pw[q] != 0x7fffffff) {
            int sidx = (int)((unsigned)pw[q] % (unsigned)SLOTS), got = -1;
#pragma unroll 1
            for (int probes = 0; probes < SLOTS; ++probes) {
              int key = *reinterpret_cast<volatile int*>(&s_key[sidx]);
              if (key == -1) key = atomicCAS(&s_key[sidx], -1, pw[q]);
              if (key == -1 || key == pw[q]) { got = sidx; break; }
              sidx = sidx + 1 == SLOTS ? 0 : sidx + 1;
            }
            if (got < 0) {
              open = false;  // table full: the rest waits for the next round
            } else {
              pslot[q] = got;
              nq = q + 1;
            }
          } else {
            open = false;
          }
        }
      }
      nq = __shfl_sync(kFull, nq, 0);
#pragma unroll
      for (int q = 0; q < kPropose; ++q) {
        pslot[q] = __shfl_sync(kFull, pslot[q], 0);
        if (q < nq && ((mine >> q) & 1)) pword[q] = __ldcg(&bitmap[p * Wp + pw[q]]);  // all of the lane's words in flight together
      }
      k += __popc(mine & ((1u << nq) - 1u));
      cur = wc.at(tb, k);
#pragma unroll
      for (int q = 0; q < kPropose; ++q) {
        if (q < nq) {
          const uint32_t any = __reduce_or_sync(kFull, pword[q]);
          if (lane == 0 && any) atomicOr(&s_any[pslot[q]], any);
        }
      }
    }
    __syncthreads();
    // 2. the slots in use are spread over the warps (by rank among the used ones: two words whose slots happen to be four apart
    // must not land on the same warp): pre-records now, the sums after the (first) wait
    int my_slot[2] = {-1, -1};
    {
      uint32_t used = __ballot_sync(kFull, lane < SLOTS && s_key[lane < SLOTS ? lane : 0] >= 0);
      int rank = 0;
      while (used) {
        const int sidx = __ffs(used) - 1;
        used &= used - 1;
        if (rank == warp) my_slot[0] = sidx;
        if (rank == warp + WARPS) my_slot[1] = sidx;
        ++rank;
      }
    }
#pragma unroll
    for (int j = 0; j < 2; ++j)
      if (my_slot[j] >= 0) stage_pre_record(pre, s_key[my_slot[j]], s_any[my_slot[j]], s_chk + (size_t)my_slot[j] * 32 * rec, rec, R, lane);
    stamp(5);
    if (!sums_awaited) {
      sync.wait_totals(px);  // the sums of every running pod (of every rank) are in px.total
      sums_awaited = true;
      stamp(6);
    }
#pragma unroll
    for (int j = 0; j < 2; ++j)
      if (my_slot[j] >= 0) stage_finish_record(px, s_key[my_slot[j]], s_any[my_slot[j]], s_chk + (size_t)my_slot[j] * 32 * rec, rec, R, M, lane);
    __syncthreads();
    stamp(7);
    // 3. every lane decides its own pairs
#pragma unroll
    for (int q = 0; q < kPropose; ++q)
      if (pword[q] && pslot[q] >= 0) decide_word<RT>(pword[q], pw[q], s_chk + (size_t)pslot[q] * 32 * rec, rec, R, Wp, pod, codes, sp, ok);
    const int more = __syncthreads_or(cur != 0x7fffffff);  // pods with more words than fit one round (ClusterThrottle-heavy namespaces)
    if (!more) break;
    if (tid < SLOTS) { s_key[tid] = -1; s_any[tid] = 0u; }
    __syncthreads();
  }
  stamp(8);
  if (valid) admit[p] = ok;
}


// ------------------------------------------------------------------------------------------------
// The SHARED decide tiles of the fused pass.  The decide work is not left to P/TILE CTAs with one lane per pod (walking its
// words and pairs one after the other while every other SM has gone idle): every CTA of k_pass that has run out of match and
// reconcile tiles draws sub-tiles of TILE/4 pending pods from the same ticket counter.  FOUR lanes per pod: lane q
// fetches the pod's q-th word of the round and claims its staging slot (same-word lanes of a warp elect one claimant; a word
// that finds no slot -- rows in arrival order -- is checked pair by pair straight from L2), and the pod's pairs are dealt out
// to its four lanes bit by bit.  Everything before the wait for the sums -- requests, match words, slot claims, the
// pre-records (one bulk copy of 32 records per slot) -- is done while the slowest reconcile tiles are still at work.
//
// KT_QUAD_DRYRUN: the code after the wait (constants, pair checks) runs once per CTA, late in the pass, on SMs that have been
// executing other code: its instructions come from L2, miss by miss.  A tile that has to wait anyway walks that code once
// (1) or over and over (2) on whatever the sums hold so far -- results thrown away, the raw pre-records fetched again -- so
// that the real run finds its instructions in the SM's instruction caches.
// ------------------------------------------------------------------------------------------------
#ifndef KT_QUAD_DRYRUN  // measured: the walk itself costs what it saves -- off.  Not deleted: the compiler keeps the unused dry-run code, and
#define KT_QUAD_DRYRUN 0  // without it the 768-thread k_pass allocates registers differently and C5 is 1.6% slower (DESIGN section 9)
#endif
template <int TILE, int RT>
__device__ __forceinline__ void check_decide_quad(const PodView& pods, const TableView& tb, int R, int KS, const unsigned char* __restrict__ pre,
                                                  const PartExchange& px, const uint32_t* __restrict__ bitmap, uint32_t* __restrict__ codes,
                                                  unsigned char* __restrict__ admit, unsigned char* smem_raw, int64_t sub, const FlagSync& sync,
                                                  const SparseOut sp, unsigned long long* s_mbar /* [WARPS], initialised (count 1) */,
                                                  unsigned& mbar_phase /* this warp's next parity */, unsigned long long* trace_row = nullptr) {
  // optional stage stamps (kt_enable_trace) of the CTA's FIRST sub-tile: [9] match rows + pre-records visible, [10] slots
  // claimed + pre-records requested, [11] sums of every rank visible, [12] constants finished, [13] decided
  auto stamp = [&](int k) {
    if (trace_row && threadIdx.x == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      trace_row[k] = t;
    }
  };
  // ... and SM cycle counts of thread 0's way through its first round ([16 + k], %clock64): 0 entry, 1 requests in shared
  // memory + counters seen, 2 match word loaded + slot claimed, 3 slots ranked + pre-records requested, 4 first dry run done,
  // 5 sums visible, 6 pre-records landed, 7 constants finished, 8 CTA barrier, 9 own pairs decided, 10 round closed;
  // [16 + 11] dry runs made
  auto cyc = [&](int k) {
    if (trace_row && threadIdx.x == 0) {
      long long t;
      asm volatile("mov.u64 %0, %%clock64;" : "=l"(t)::"memory");
      trace_row[16 + k] = (unsigned long long)t;
    }
  };
  cyc(0);
  constexpr int WARPS = TILE / 32, PODS = TILE / 4;
  const size_t rec = decide_record_bytes(R);
  const int SLOTS = WARPS * KS;
  long long* s_req = reinterpret_cast<long long*>(smem_raw);                          // [R][PODS] (carved as [R][TILE], like check_decide_tile)
  unsigned char* s_chk = reinterpret_cast<unsigned char*>(s_req + (size_t)R * TILE);  // [SLOTS][32][rec]
  int* s_key = reinterpret_cast<int*>(s_chk + (size_t)SLOTS * 32 * rec);              // [SLOTS] word index or -1
  uint32_t* s_any = reinterpret_cast<uint32_t*>(s_key + SLOTS);                       // [SLOTS] throttles of the word some lane of the CTA matched
  uint32_t* s_flag = s_any + SLOTS;                                                   // thread 0 -> CTA: the sums are complete
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int j = tid >> 2, q = tid & 3;  // pod of the sub-tile, lane of the pod
  const int Wp = tb.Wp;
  const int M = tb.M;
  const int64_t p = sub * PODS + j;
  const bool valid = p < pods.n;
  const int64_t pc = valid ? p : pods.n - 1;
  // thread 0: what has been signalled already?  Three relaxed loads in flight together with everybody's row loads -- a tile
  // that starts late finds all of it there and pays ONE trip to L2 and one acquire fence instead of three waits in a row.
  const unsigned* sums_counter = px.npeers == 0 ? &sync.s->rec_done : &sync.s->tot_done;
  const unsigned sums_target = px.npeers == 0 ? sync.n_rec : sync.n_fin;
  unsigned seen_match = 0, seen_prep = 0, seen_sums = 0;
  if (tid == 0) {
    seen_match = ld_relaxed_gpu(&sync.s->match_done);
    seen_prep = ld_relaxed_gpu(&sync.s->prep_done);
    seen_sums = ld_relaxed_gpu(sums_counter);
  }
  const int ns = valid ? __ldg(&pods.ns[pc]) : -1;
  const uint32_t present = __ldg(&pods.present[pc]);
  const uint32_t winfo = __ldg(&pods.winfo[pc]);
  // ResourceAmountOfPod(pod): the pod's four lanes fetch every fourth resource each
  uint32_t nz = 0;
  for (int r = q; r < R; r += 4) {
    long long v = __ldg(pods.req + (int64_t)r * pods.n + pc);
    if (!((present >> r) & 1)) v = 0;
    s_req[r * PODS + j] = v;
    if (v != 0) nz |= 1u << r;
  }
  nz |= __shfl_xor_sync(kFull, nz, 1);
  nz |= __shfl_xor_sync(kFull, nz, 2);
  const DecidePod pod{s_req + j, PODS, nz, p};
  if (tid < SLOTS) { s_key[tid] = -1; s_any[tid] = 0u; }
  WordCursor wc;
  wc.init(tb, winfo, ns, valid && (unsigned)ns < (unsigned)tb.NS);
  if (tid == 0) {
    // the match rows of EVERY pending tile (ours came from some other CTA) and the pre-records (early: they depend on nothing)
    if (seen_match < sync.n_match) {
      spin_until([&] { return ld_relaxed_gpu(&sync.s->match_done) >= sync.n_match; }, &sync.s->error, 40);
      (void)ld_acquire_gpu(&sync.s->match_done);
    }
    if (seen_prep < sync.n_fin) {
      spin_until([&] { return ld_relaxed_gpu(&sync.s->prep_done) >= sync.n_fin; }, &sync.s->error, 40);
      (void)ld_acquire_gpu(&sync.s->prep_done);
    }
    *s_flag = seen_sums >= sums_target ? 1u : 0u;
    fence_acquire_gpu();  // ONE acquire for every counter observed so far
  }
  __syncthreads();  // the slot table is initialised, the requests are in shared memory, the counters have been seen
  bool sums_ready = *s_flag != 0u;
  stamp(9);
  cyc(1);

  unsigned char ok = 1;
  unsigned dry_runs = 0;
#pragma unroll 1
  for (int rd = 0;; ++rd) {
    // 1. this lane's word of the round and its match word; lanes with matches need the word's 32 records staged
    const int w = wc.at(tb, rd * 4 + q);  // 0x7fffffff: none left
    const uint32_t mword = w != 0x7fffffff ? __ldcg(&bitmap[p * Wp + w]) : 0u;
    int slot = -1;
    {
      const int key = mword ? w : 0x7fffffff;
      const unsigned grp = __match_any_sync(kFull, key);  // the lanes of this warp that want the same word
      const int leader = __ffs(grp) - 1;
      const uint32_t gor = __reduce_or_sync(grp, mword);
      if (mword && lane == leader) {  // open addressing from w mod SLOTS; full table: the group checks its pairs straight from L2
        int sidx = (int)((unsigned)w % (unsigned)SLOTS);
#pragma unroll 1
        for (int probes = 0; probes < SLOTS; ++probes) {
          int key2 = *reinterpret_cast<volatile int*>(&s_key[sidx]);
          if (key2 == -1) key2 = atomicCAS(&s_key[sidx], -1, w);
          if (key2 == -1 || key2 == w) { slot = sidx; break; }
          sidx = sidx + 1 == SLOTS ? 0 : sidx + 1;
        }
        if (slot >= 0) atomicOr(&s_any[slot], gor);
      }
      slot = __shfl_sync(kFull, slot, leader);
      if (!mword) slot = -1;
    }
    if (rd == 0) cyc(2);
    proxy_fence_async();  // whatever this thread last wrote to the staging slots (generic proxy) is ordered before the bulk copies
    __syncthreads();
    // 2. the slots in use are spread over the warps (by rank among the used ones); one lane per warp asks the copy engine for
    // its slots' pre-records: 32 consecutive records = one contiguous block of 32 * rec bytes per slot
    int slot_a = -1, slot_b = -1;
    {
      uint32_t used = __ballot_sync(kFull, lane < SLOTS && s_key[lane < SLOTS ? lane : 0] >= 0);
      int rank = 0;
      while (used) {
        const int sidx = __ffs(used) - 1;
        used &= used - 1;
        if (rank == warp) slot_a = sidx;
        if (rank == warp + WARPS) slot_b = sidx;
        ++rank;
      }
    }
    const int n_mine = (slot_a >= 0) + (slot_b >= 0);
    auto request_pre = [&]() {
      if (n_mine && lane == 0) {
        mbar_expect_tx(&s_mbar[warp], (unsigned)(n_mine * 32 * rec));
        bulk_copy_g2s(s_chk + (size_t)slot_a * 32 * rec, pre + (size_t)s_key[slot_a] * 32 * rec, (unsigned)(32 * rec), &s_mbar[warp]);
        if (slot_b >= 0) bulk_copy_g2s(s_chk + (size_t)slot_b * 32 * rec, pre + (size_t)s_key[slot_b] * 32 * rec, (unsigned)(32 * rec), &s_mbar[warp]);
      }
    };
    request_pre();
    if (rd == 0) { stamp(10); cyc(3); }
    // 3. sums -> constants -> pairs.  The same instructions serve the dry runs (see above) and the real one.
    int dry_left = KT_QUAD_DRYRUN == 1 ? 1 : (KT_QUAD_DRYRUN >= 2 ? 4096 : 0);
    bool real;
#pragma unroll 1
    do {
      if (!sums_ready) {
        if (dry_left == 0) {
          sync.wait_totals(px);  // the sums of every running pod (of every rank) are in px.total
          sums_ready = true;
        } else {  // look once; not there: one more walk through the code below
          --dry_left;
          if (tid == 0) {
            const bool there = ld_acquire_gpu(sums_counter) >= sums_target;
            *s_flag = there ? 1u : 0u;
          }
          __syncthreads();
          sums_ready = *s_flag != 0u;
        }
      }
      real = sums_ready;
      if (real && rd == 0) { stamp(11); cyc(5); }
      if (n_mine) {  // warp-uniform: the raw records have landed
        mbar_wait(&s_mbar[warp], mbar_phase & 1u);
        mbar_phase ^= 1u;
      }
      if (real && rd == 0) cyc(6);
      if (slot_a >= 0) stage_finish_record(px, s_key[slot_a], s_any[slot_a], s_chk + (size_t)slot_a * 32 * rec, rec, R, M, lane);
      if (slot_b >= 0) stage_finish_record(px, s_key[slot_b], s_any[slot_b], s_chk + (size_t)slot_b * 32 * rec, rec, R, M, lane);
      if (real && rd == 0) cyc(7);
      __syncthreads();
      if (real && rd == 0) { stamp(12); cyc(8); }
      // the pod's pairs, dealt out to its four lanes bit by bit; word i of the round belongs to lane i, which collects its codes
      // (NOT unrolled: this code runs once per CTA, cold -- its instructions come from L2, and four copies are four times the misses)
#pragma unroll 1
      for (int i = 0; i < 4; ++i) {
        const int src = (lane & ~3) | i;
        const int wi = __shfl_sync(kFull, w, src);
        const uint32_t mi = __shfl_sync(kFull, mword, src);
        const int si = __shfl_sync(kFull, slot, src);
        const uint32_t part = mi & (0x11111111u << q);
        uint2 c = make_uint2(0u, 0u);
        if (part) {
          if (si >= 0) c = decide_word_codes<RT>(part, s_chk + (size_t)si * 32 * rec, rec, R, pod);
          else c = decide_word_direct_far(part, wi, pre, px.total, (unsigned)rec, R, M, pod.req, pod.stride, pod.nz);
        }
        c.x |= __shfl_xor_sync(kFull, c.x, 1);
        c.y |= __shfl_xor_sync(kFull, c.y, 1);
        c.x |= __shfl_xor_sync(kFull, c.x, 2);
        c.y |= __shfl_xor_sync(kFull, c.y, 2);
        if (real && q == i && mi) store_codes(c, wi, Wp, p, codes, sp, ok);
      }
      if (real && rd == 0) cyc(9);
      if (!real) {  // a dry run: the records it finished in place are void -- fetch the raw ones again
        ++dry_runs;
        proxy_fence_async();
        __syncthreads();  // everybody is done with the slots
        request_pre();
        if (rd == 0 && dry_runs == 1) cyc(4);
      }
    } while (!real);
    const int more = __syncthreads_or((rd + 1) * 4 < wc.cnt);  // pods with more than four words (ClusterThrottle-heavy namespaces)
    if (rd == 0) cyc(10);
    if (!more) break;
    if (tid < SLOTS) { s_key[tid] = -1; s_any[tid] = 0u; }
    __syncthreads();
  }
  stamp(13);
  if (trace_row && tid == 0) trace_row[16 + 11] = dry_runs;
  unsigned okw = ok;
  okw &= __shfl_xor_sync(kFull, okw, 1);
  okw &= __shfl_xor_sync(kFull, okw, 2);
  if (valid && q == 0) admit[p] = (unsigned char)okw;
}

// k_check: both phases of one tile in one CTA (the PDL-chained path: phase 1 overlaps k_reconcile / k_finalize).
template <int TPC, int B, bool REG>
__global__ void __launch_bounds__(kTileCheck) k_check(PodView pods, TableView tb, int L, int R, const unsigned char* __restrict__ pre, const PartExchange px,
                                                      uint32_t* __restrict__ bitmap, uint32_t* __restrict__ codes,
                                                      unsigned char* __restrict__ admit, SparseOut sparse /* count zeroed by the host before the launch */) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  check_match_tile<TPC, B, REG, kTileCheck>(pods, tb, L, bitmap, codes, smem_raw, blockIdx.x);
  __syncthreads();  // the tile's match rows are written (read back below) and the row staging is free again
  check_decide_tile<kTileCheck, 0>(pods, tb, R, decide_stage_words(R, kTileCheck), pre, px, bitmap, codes, admit, smem_raw, blockIdx.x, PdlSync{}, sparse);
}

// ------------------------------------------------------------------------------------------------
// k_pass: the whole pass in ONE launch of at most as many CTAs as the device holds at once.  Every CTA draws tickets
// until none is left: match tiles (which also write the pre-records), reconcile tiles, then the second phase -- status
// tiles (with peers they perform the all-reduce over NVLink) and decide sub-tiles.  Match tiles hold the first tickets,
// so the pending pods are matched while the reconcile tiles are still summing, and the CTAs that finish those cheap
// tiles first take the reconcile tiles that did not fit the first wave.  One cold start instead of three, and the
// hand-offs cost a poll of an L2 counter instead of a kernel boundary.
// ------------------------------------------------------------------------------------------------
struct PassArgs {
  PodView run, pend;
  TableView tb;
  ThrottleView tv;
  ReconcileView out;
  PartExchange px;
  uint32_t* run_bitmap;
  uint32_t* pend_bitmap;
  uint32_t* codes;
  unsigned char* admit;
  unsigned char* pre;   // [M] pre-records (finalize tiles -> decide tiles)
  SparseOut sparse;
  PassSync* sync;
  long long now;
  uint32_t eval_flags;
  int L, R, S, G;
  unsigned quad;                 // 1: decide sub-tiles of TILE/4 pending pods, four lanes per pod (check_decide_quad); 0: decide tiles of
                                 // TILE pods, one lane per pod (check_decide_tile) -- the host picks (launch_pass)
  unsigned early;                // 1: run the first phase before waiting for the previous grid (the host decides: evaluate_locked)
  unsigned n_chk, n_rec, n_fin;  // tiles per role; tickets: [match (+ prep) n_chk][reconcile n_rec][second phase: n_fin status tiles and n_sub
  unsigned n_sub;                // decide (sub-)tiles -- status first with peers (they carry the exchange the decide
                                 // sub-tiles wait for), last alone (nobody waits for them)]; a piece only ever waits for SMALLER tickets
                                 // (status: reconcile; decide: match + prep, reconcile -- with peers the status tiles' totals) or for other
                                 // GPUs, whose pieces are subject to the same order (PassSync)
  unsigned long long* trace;     // optional (kt_enable_trace): per first-phase ticket, then per status tile, kTraceRow x u64 {ticket, sm, t_start,
                                 // t_end, stage stamps} in globaltimer ns, [28] the CTA that ran it; a CTA's last first-phase tile also
                                 // carries its first decide sub-tile's stamps and [29] the time the CTA exited
};
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// TILE: pods per CTA (= threads).  128 everywhere except ClusterThrottle-heavy tables, where every pod walks a dozen words and a
// CTA's accumulator slots (one per word, 2 KB each at R = 8) are better shared by twice the pods (measured faster at C3).
template <int TPC, int B, int RT, bool REG, int TILE, int THREADS>
__global__ void __launch_bounds__(TILE, THREADS / TILE) k_pass(const __grid_constant__ PassArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ unsigned s_ticket;
  __shared__ unsigned s_last;                 // trace: this CTA's last first-phase ticket (~0u: none yet)
  __shared__ unsigned s_done[2];              // first-phase tiles this CTA has finished and not yet published: match, reconcile
  __shared__ unsigned s_tail;                 // 1: this CTA ran the last first-phase ticket
  __shared__ unsigned long long s_t_start;    // trace: when the current tile began
  __shared__ __align__(8) unsigned long long s_mbar[kMaxWarps];  // transaction barriers: one per warp (bulk copies of the shared decide tiles)
  // Launched with programmatic stream serialization.  The previous grid in the stream is waited for at the top, or -- an EARLY
  // pass -- only once this CTA leaves the first phase.  An early pass is one the host has proven safe (evaluate_locked): its
  // primary is a k_pass of another context, or of this one when neither zero-fills.  Its first phase then writes only what is
  // its own or what the primary's second phase does not read differently:
  //   - PassSync counters and pre-records: one set per pass parity (the host alternates them), re-armed / rewritten only by
  //     the pass two back, which had completed before the primary's CTAs got past their wait and triggered us;
  //   - partial sums: the half of this parity, zeroed by the primary after its wait and before its trigger (below);
  //   - match rows (pending and running bitmaps): rows and tables are unchanged since the primary, so every word is rewritten
  //     with the value the primary stored and reads;
  //   - code words: a match tile writes them only when it zero-fills (never in an early pass); decide rewrites every word
  //     whose match bits are set, and codes are zero elsewhere;
  //   - the sparse list's counter is reset after the wait (s_tail), before anything this pass decides can append.
  // The trigger follows the wait, so at most two passes run at once.  No wait can deadlock: first-phase tiles never wait; a
  // second-phase piece waits for smaller tickets of its own pass, or for the previous grid, all of whose CTAs were placed
  // before it triggered and none of which waits for this one; a CTA of this grid that cannot be placed yet only starts later.
  // Any other kernel that follows with PDL must wait before its first access to shared state, which is why a pass that does
  // not start with k_pass launches k_finalize plainly.
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < kMaxWarps; ++i) mbar_init(&s_mbar[i], 1u);
    mbar_init_fence();
    s_last = ~0u;
    s_done[0] = s_done[1] = 0u;
    s_tail = 0u;
  }
  if (!a.early) pdl_wait_primary();
  const unsigned n_tiles = a.n_chk + a.n_rec;
  auto draw = [&]() -> unsigned {
    __syncthreads();  // everybody has read the previous ticket, and the CTA's shared memory is free again
    if (threadIdx.x == 0) s_ticket = atomicAdd(&a.sync->ticket, 1u);
    __syncthreads();
    return s_ticket;
  };
  // (the trace bookkeeping lives in shared memory: nothing of it stays in registers across a tile, which runs at the register cap)
  auto trace_row = [&](unsigned t) -> unsigned long long* { return a.trace && t != ~0u ? a.trace + (size_t)t * kTraceRow : nullptr; };
  auto open_row = [&](unsigned long long* row) {  // thread 0, before a traced tile stamps anything: the rows are not cleared
    for (int k = 0; k < kTraceRow; ++k) row[k] = 0ull;  // between passes (no memset may come between two queued passes)
    s_t_start = globaltimer_ns();
  };
  auto close_row = [&](unsigned long long* row) {  // thread 0, at the end of a traced tile
    unsigned smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    row[0] = s_ticket; row[1] = smid; row[2] = s_t_start; row[3] = globaltimer_ns(); row[28] = blockIdx.x;
  };
  unsigned ticket;
  // ---- first phase: match and reconcile tiles, none of which waits for anything ----
  // Nothing waits for match_done / rec_done before every first-phase ticket has been drawn, so a CTA publishes the tiles it
  // finished in runs: its match tiles when it draws its first ticket past them (the decide sub-tiles start staging on the match
  // rows while the last reconcile tiles run), its reconcile tiles when it leaves the phase -- no L2 round trip between two
  // reconcile tiles.  Each publish follows the CTA barrier that begins the draw: every thread's tiles are complete.
  while ((ticket = draw()) < n_tiles) {
    if (threadIdx.x == 0 && ticket >= a.n_chk && s_done[0]) {
      __threadfence();
      atomicAdd(&a.sync->match_done, s_done[0]);
      s_done[0] = 0u;
    }
    if (a.trace && threadIdx.x == 0) open_row(trace_row(ticket));
    if (ticket < a.n_chk) {
      const FlagSync sync{a.sync, a.n_rec, a.n_fin, a.n_chk};
      // The match tiles also write the pre-records (the prep half of the finalize tiles, spread over them): they hold the first
      // tickets, so every pre-record exists a few microseconds into the pass and no decide sub-tile ever waits for one.
      for (unsigned ft = ticket; ft < a.n_fin; ft += a.n_chk)
        finalize_tile(a.tv, a.tb.M, a.R, a.G, a.now, a.eval_flags, a.px, a.out, a.pre, (int)ft, sync, nullptr, kFinPrep);
      check_match_tile<TPC, B, REG, TILE>(a.pend, a.tb, a.L, a.pend_bitmap, a.codes, smem_raw, ticket);
    } else {
      reconcile_tile<TPC, B, RT, REG, TILE>(a.run, a.tb, a.L, a.R, a.S, a.run_bitmap, a.px.mine, smem_raw, ticket - a.n_chk, trace_row(ticket));
    }
    if (threadIdx.x == 0) {  // (s_ticket is still this tile's: the next draw begins with a CTA barrier)
      ++s_done[ticket < a.n_chk ? 0 : 1];
      if (ticket == n_tiles - 1) s_tail = 1u;
      if (a.trace) {
        close_row(trace_row(s_ticket));
        s_last = s_ticket;
      }
    }
  }
  if (a.early) pdl_wait_primary();
  // The previous grid has completed.  The CTA that ran the last first-phase ticket clears the sparse list's counter before it
  // publishes that tile: every decide piece waits for it (match_done or rec_done) before it appends.  Then the rest of this
  // CTA's tiles, before it starts anything that can wait (release pattern, as cta_signal).
  if (threadIdx.x == 0) {
    if (s_tail && a.sparse.count) *a.sparse.count = 0u;
    if (s_done[0] | s_done[1]) {
      __threadfence();
      if (s_done[0]) atomicAdd(&a.sync->match_done, s_done[0]);
      if (s_done[1]) atomicAdd(&a.sync->rec_done, s_done[1]);
    }
  }
  // The other parity's partial sums -- the previous pass's, read by nobody now -- are zeroed for the next pass before this CTA
  // lets it start: the next pass adds into them from its first phase on.
  {
    const size_t len = (size_t)(2 * a.R + 1) * a.tb.M, stride = (size_t)gridDim.x * TILE;
    bool wrote = false;
    for (size_t i = (size_t)blockIdx.x * TILE + threadIdx.x; i < len; i += stride) {
      a.px.zero_mine[i] = 0ull;
      wrote = true;
    }
    if (wrote) __threadfence();
  }
  __syncthreads();
  pdl_launch_dependents();
  // ---- second phase: status tiles and decide sub-tiles, until the counter runs past them ----
  unsigned mbar_phase = 0;
  bool first = true;
  const unsigned n_work = a.n_fin + a.n_sub;
  const bool status_first = a.px.npeers > 0;
  for (unsigned work = ticket - n_tiles; work < n_work; work = draw() - n_tiles) {
    const bool is_status = status_first ? work < a.n_fin : work >= a.n_sub;
    const unsigned index = status_first ? (is_status ? work : work - a.n_fin) : (is_status ? work - a.n_sub : work);
    const FlagSync sync{a.sync, a.n_rec, a.n_fin, a.n_chk};
    if (is_status) {  // traced as row n_tiles + index (after the first-phase tickets' rows)
      unsigned long long* trow = trace_row(n_tiles + index);
      if (trow && threadIdx.x == 0) open_row(trow);
      finalize_tile(a.tv, a.tb.M, a.R, a.G, a.now, a.eval_flags, a.px, a.out, a.pre, (int)index, sync, trow, kFinStatus);
      if (trow && threadIdx.x == 0) close_row(trow);
    } else if (a.quad) {
      check_decide_quad<TILE, RT>(a.pend, a.tb, a.R, decide_stage_words(a.R, TILE), a.pre, a.px, a.pend_bitmap, a.codes, a.admit, smem_raw, index, sync,
                                  a.sparse, s_mbar, mbar_phase, first ? trace_row(s_last) : nullptr);
      first = false;
    } else {  // (no trace stamps: they would land on the reconcile tile's)
      check_decide_tile<TILE, RT>(a.pend, a.tb, a.R, decide_stage_words(a.R, TILE), a.pre, a.px, a.pend_bitmap, a.codes, a.admit, smem_raw, index, sync,
                                  a.sparse);
    }
  }
  // the last CTA out re-arms the counters for the next pass of this parity (it starts after this grid has completed)
  __syncthreads();
  if (threadIdx.x == 0) {
    if (unsigned long long* row = trace_row(s_last)) row[29] = globaltimer_ns();
    if (atomicAdd(&a.sync->exited, 1u) == gridDim.x - 1) {
      a.sync->ticket = 0;
      a.sync->rec_done = 0;
      a.sync->prep_done = 0;
      a.sync->match_done = 0;
      a.sync->tot_done = 0;
      a.sync->exited = 0;
    }
  }
}

struct ReqShifts { unsigned char s[32]; };  // per-column left shift of the 32-bit transfer requests (by value, in the launch arguments)

// dictionary-coded request columns of the packed transfer format (by value in the launch arguments; codes == nullptr: not used)
struct ReqCodes {
  const unsigned char* codes;   // the code columns, one after another
  const int64_t* dict;          // the value dictionaries, one after another
  uint32_t col_off[32];         // byte offset of column r inside codes (multiples of 4)
  uint32_t dict_off[32];        // first dictionary entry of column r
  uint32_t dict_len[32];
  unsigned char bytes[32];      // 1 or 2
};

// Packed transfer rows (kt_upload_pods_packed: 16-bit label-pair indices, presence inside the meta word) -> the int64 HBM
// columns.  One lane per pod row, coalesced; the pair dictionary (a few KB) stays in L1.
__global__ void __launch_bounds__(256) k_unpack_packed(int64_t n, int L, int Lpad, int R, int ns_bits, int n_pairs, const int64_t* __restrict__ pairs,
                                                       const uint16_t* __restrict__ labels16, const int32_t* __restrict__ req32, const ReqShifts req_shift,
                                                       const ReqCodes rc, const uint32_t* __restrict__ meta, int64_t* __restrict__ labels, int64_t* __restrict__ req,
                                                       uint32_t* __restrict__ present, uint32_t* __restrict__ flags, int32_t* __restrict__ ns,
                                                       int translate, const TableView tb, uint32_t* __restrict__ roff, uint32_t* __restrict__ winfo) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  // labels in chunks of eight slots; with `translate` the chunk goes through the label dictionary while it is in registers
  // (what k_translate_rows would do in a second launch, re-reading the int64 columns this kernel has just written)
#pragma unroll 1
  for (int s0 = 0; s0 < Lpad; s0 += 8) {
    int64_t lab[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int s = s0 + j;
      lab[j] = KT_LABEL_EMPTY;
      if (s < L) {
        const uint32_t c = __ldg(&labels16[(int64_t)s * n + p]);
        if (c != 0xffffu && (int)c < n_pairs) lab[j] = __ldg(&pairs[c]);
      }
      labels[(int64_t)s * n + p] = lab[j];
    }
    if (translate) {
      uint4 ke[8];
      uint32_t o[8];
      translate8_keys(tb, lab, ke);
      translate8_rows(tb, lab, ke, o);
#pragma unroll
      for (int j = 0; j < 8; ++j) roff[(int64_t)(s0 + j) * n + p] = o[j];
    }
  }
  if (rc.codes) {
    for (int r = 0; r < R; ++r) {
      const unsigned char* col = rc.codes + rc.col_off[r];
      const uint32_t code = rc.bytes[r] == 1 ? (uint32_t)__ldg(&col[p]) : (uint32_t)__ldg(reinterpret_cast<const unsigned short*>(col) + p);
      req[(int64_t)r * n + p] = code < rc.dict_len[r] ? __ldg(&rc.dict[rc.dict_off[r] + code]) : 0;
    }
  } else {
    for (int r = 0; r < R; ++r) req[(int64_t)r * n + p] = (int64_t)__ldg(&req32[(int64_t)r * n + p]) << req_shift.s[r];
  }
  const uint32_t m = __ldg(&meta[p]);
  const int my_ns = (int32_t)(m & ((1u << ns_bits) - 1u));
  ns[p] = my_ns;
  flags[p] = (m >> ns_bits) & 7u;
  present[p] = (m >> (ns_bits + 3)) & (R >= 32 ? 0xffffffffu : ((1u << R) - 1u));
  if (translate) {  // the words that can apply to the row's namespace (see winfo_pack)
    int cnt = 0, w0 = 0, w1 = 0;
    if ((unsigned)my_ns < (unsigned)tb.NS) {
      const int lo = __ldg(&tb.nsw_off[my_ns]);
      cnt = __ldg(&tb.nsw_off[my_ns + 1]) - lo;
      if (cnt > 0) w0 = __ldg(&tb.nsw_idx[lo]);
      if (cnt > 1) w1 = __ldg(&tb.nsw_idx[lo + 1]);
    }
    winfo[p] = cnt == 0 ? 0u : winfo_pack(cnt, w0, w1, tb.W);
  }
}

// Row-level delta: scatter k packed rows into the resident columns (pod informer Add/Update/Delete).
__global__ void __launch_bounds__(256) k_scatter_rows(int64_t k, const int64_t* __restrict__ rows, int L, int R, int64_t n,
                                                      const int64_t* __restrict__ labels, const int64_t* __restrict__ req,
                                                      const uint32_t* __restrict__ present, const uint32_t* __restrict__ flags,
                                                      const int32_t* __restrict__ ns, int64_t* d_labels, int64_t* d_req,
                                                      uint32_t* d_present, uint32_t* d_flags, int32_t* d_ns) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k) return;
  const int64_t row = rows[i];
  if (row < 0 || row >= n) return;
  for (int s = 0; s < L; ++s) d_labels[(int64_t)s * n + row] = labels[(int64_t)s * k + i];
  for (int r = 0; r < R; ++r) d_req[(int64_t)r * n + row] = req[(int64_t)r * k + i];
  d_present[row] = present[i];
  d_flags[row] = flags[i];
  d_ns[row] = ns[i];
}

// Label columns -> row offsets into the CURRENT selector tables: every row (rows == nullptr, k == n) after an upload or a
// table compile, or the k listed rows after a row delta.  One lane per pod row, coalesced column accesses; the two
// dictionary hops per label that used to sit on every pass's critical path are paid here, once per change.
__global__ void __launch_bounds__(256) k_translate_rows(int64_t k, const int64_t* __restrict__ rows, const TableView tb, int Lpad, int64_t n,
                                                        const int64_t* __restrict__ labels, const int32_t* __restrict__ ns_col, uint32_t* __restrict__ roff,
                                                        uint32_t* __restrict__ winfo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k) return;
  const int64_t p = rows ? rows[i] : i;
  if (p < 0 || p >= n) return;
  {  // the words that can apply to the row's namespace (see winfo_pack)
    const int ns = ns_col[p];
    int cnt = 0, w0 = 0, w1 = 0;
    if ((unsigned)ns < (unsigned)tb.NS) {
      const int lo = __ldg(&tb.nsw_off[ns]);
      cnt = __ldg(&tb.nsw_off[ns + 1]) - lo;
      if (cnt > 0) w0 = __ldg(&tb.nsw_idx[lo]);
      if (cnt > 1) w1 = __ldg(&tb.nsw_idx[lo + 1]);
    }
    winfo[p] = cnt == 0 ? 0u : winfo_pack(cnt, w0, w1, tb.W);
  }
#pragma unroll 1
  for (int i0 = 0; i0 < Lpad; i0 += 8) {
    uint32_t o[8];
    translate8(tb, labels + (int64_t)i0 * n + p, n, o);
#pragma unroll
    for (int j = 0; j < 8; ++j) roff[(int64_t)(i0 + j) * n + p] = o[j];
  }
}

// Compact transfer rows -> the int64 HBM columns (kt_upload_pods_compact).  One lane per pod row; every column access is
// coalesced.  Lpad - L padding label rows are filled with KT_LABEL_EMPTY here as well.
__global__ void __launch_bounds__(256) k_unpack_rows(int64_t n, int L, int Lpad, int R, int val_bits, const uint32_t* __restrict__ labels32,
                                                     const int32_t* __restrict__ req32, const ReqShifts req_shift,
                                                     const uint32_t* __restrict__ meta, int64_t* __restrict__ labels, int64_t* __restrict__ req,
                                                     uint32_t* __restrict__ flags, int32_t* __restrict__ ns) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint32_t vmask = (1u << val_bits) - 1u;
  for (int s = 0; s < Lpad; ++s) {
    int64_t lab = KT_LABEL_EMPTY;
    if (s < L) {
      const uint32_t c = __ldg(&labels32[(int64_t)s * n + p]);
      if (c != 0xffffffffu) lab = (int64_t)(((uint64_t)(c >> val_bits) << 32) | (uint64_t)(c & vmask));
    }
    labels[(int64_t)s * n + p] = lab;
  }
  for (int r = 0; r < R; ++r) req[(int64_t)r * n + p] = (int64_t)__ldg(&req32[(int64_t)r * n + p]) << req_shift.s[r];
  const uint32_t m = __ldg(&meta[p]);
  ns[p] = (int32_t)(m & 0x1fffffffu);
  flags[p] = m >> 29;
}

// Status columns of k listed throttles: column idx[i] of the pass's M columns (src) -> column i of k (dst), so that
// kt_get_reconcile_rows downloads in proportion to what changed, not to M.
__global__ void __launch_bounds__(128) k_gather_status(int64_t k, const int32_t* __restrict__ idx, int R, int M, const ReconcileView src,
                                                       const ReconcileView dst) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k) return;
  const int t = idx[i];
  for (int r = 0; r < R; ++r) {
    dst.used[(size_t)r * k + i] = src.used[(size_t)r * M + t];
    dst.calc_thr[(size_t)r * k + i] = src.calc_thr[(size_t)r * M + t];
  }
  dst.used_cnt[i] = src.used_cnt[t];
  dst.calc_cnt[i] = src.calc_cnt[t];
  dst.used_present[i] = src.used_present[t];
  dst.throttled[i] = src.throttled[t];
  dst.calc_present[i] = src.calc_present[t];
  dst.override_active[i] = src.override_active[t];
}
__global__ void __launch_bounds__(256) k_gather_bytes(int64_t k, const int64_t* __restrict__ rows, const unsigned char* __restrict__ src, unsigned char* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < k) out[i] = src[rows[i]];
}

// Gather k bitmap rows (one warp-wide strided copy per row).
__global__ void __launch_bounds__(256) k_gather_rows(int64_t k, const int64_t* __restrict__ rows, int Wp, const uint32_t* __restrict__ bitmap,
                                                     uint32_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (i >= k) return;
  const int64_t row = rows[i];
  for (int w = threadIdx.x & 31; w < Wp; w += 32) out[i * Wp + w] = bitmap[row * Wp + w];
}

}  // namespace kt
