// kt_keyed.cuh -- reconcile(key) for k listed throttles on the device (kt_reconcile_throttles), PreFilter for k listed
// pending rows (kt_check_pending_rows), the affected throttles of k pods given by value (kt_match_pods), PreFilter of k pods given
// by value (kt_check_pods) and the scheduling queue summarised per throttle (kt_get_check_summary), the last four at the end of
// this file.
//
// The reference reconciles one key at a time (throttle_controller.go:84-211, clusterthrottle_controller.go:87-214): a key costs
// the pods of the namespaces its throttle reaches (affectedPods, :221-246), not the whole snapshot.  Here the listed throttles'
// 32-throttle words ("listed words", with a mask of the listed bits of each) are evaluated for the running rows whose namespace
// can reach a listed bit, and for nothing else:
//   1. k_keyed_reach     namespace -> which listed words it reaches (the tables' nsmask AND the listed bits), one bit per word
//   2. k_keyed_rows      a warp reads ns / flags of 32 rows (the only O(N) traffic, 8 B per row); rows that are not counted or
//                        whose namespace reaches nothing listed stop there.  The others evaluate the words they reach with the
//                        pass's own word evaluation (eval_word), AND the listed mask, store the non-zero words in a compact
//                        scratch [n][nw] and add the not-finished rows' requests into per-CTA accumulators (one warp reduction
//                        per matched throttle, one global add per CTA and throttle)
//   3. ColumnView        the scratch transposed into the CSR of matched rows (kt_admit.cuh: count, offsets, scan, fill)
//   4. k_keyed_status    per listed entry: CalculateThreshold(now) (the finalize tiles' code), IsThrottled(used, true)
// Nothing here writes a buffer another call reads: the match bitmaps, their clean flags, the partial-sum halves and the status
// block of the last pass are left as they are.
#pragma once
#include "kt_kernels.cuh"

namespace kt {

constexpr int kKeyedTile = 128;            // rows per CTA iteration (one lane per row)
constexpr size_t kKeyedSmemAcc = 96 * 1024;  // per-CTA accumulators up to this size; beyond it the warps add into HBM directly

struct KeyedArgs {
  PodView pods;              // the running rows (roff current)
  TableView tb;
  int L, R;
  int nw;                    // listed words
  const int32_t* words;      // [nw] word index of listed word j
  const uint32_t* masks;     // [nw] listed bits of word j
  const uint32_t* reach;     // [NS][NC] bit j%32 of reach[ns * NC + j/32]: namespace ns reaches a listed bit of word j
  int NC;                    // (nw + 31) / 32
  uint32_t* scratch;         // [n][nw] the listed bits each row matches (zeroed before the launch; counted rows only)
  unsigned long long* used;  // [R][nw * 32] sums of the not-finished matched rows (compact throttle j * 32 + b)
  unsigned long long* cnt;   // [nw * 32]
  uint32_t* pres;            // [nw * 32] presence bits of those rows' requests
  int smem_acc;              // 1: per-CTA accumulators in shared memory
};

__host__ __device__ inline size_t keyed_smem_acc_bytes(int nw, int R) { return (size_t)nw * 32 * ((size_t)R * 8 + 8 + 4); }
__host__ __device__ inline size_t keyed_smem_bytes(int nw, int R, int L, bool reg_rows, bool smem_acc) {
  const size_t b = (smem_acc ? keyed_smem_acc_bytes(nw, R) : 0) + (reg_rows ? 0 : (size_t)((L + 7) & ~7) * kKeyedTile * 4);
  return (b + 15) & ~(size_t)15;
}

__global__ void __launch_bounds__(256) k_keyed_reach(const TableView tb, int nw, const int32_t* __restrict__ words, const uint32_t* __restrict__ masks,
                                                     int NC, uint32_t* __restrict__ reach) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)tb.NS * NC) return;
  const int ns = (int)(i / NC), c = (int)(i % NC);
  uint32_t bits = 0;
  for (int jj = 0; jj < 32 && c * 32 + jj < nw; ++jj) {
    const int j = c * 32 + jj;
    const uint32_t* nsm = tb.nsmask + ((size_t)ns * tb.W + words[j]) * tb.TPpad;
    uint32_t any = 0;
    for (int s = 0; s < tb.TPpad; ++s) any |= nsm[s];
    if (any & masks[j]) bits |= 1u << jj;
  }
  reach[i] = bits;
}

template <int TPC, int B, int RT, bool REG>
__global__ void __launch_bounds__(kKeyedTile) k_keyed_rows(const KeyedArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x, lane = tid & 31;
  const int R = a.R, NJ = a.nw * 32;
  const int Lpad = (a.L + 7) & ~7;
  const PodView& pods = a.pods;
  unsigned long long* s_used = reinterpret_cast<unsigned long long*>(smem_raw);  // [R][NJ]
  unsigned long long* s_cnt = s_used + (size_t)R * NJ;                           // [NJ]
  uint32_t* s_pres = reinterpret_cast<uint32_t*>(s_cnt + NJ);                    // [NJ]
  int32_t* s_rowid = reinterpret_cast<int32_t*>(smem_raw + (a.smem_acc ? keyed_smem_acc_bytes(a.nw, R) : 0));  // [Lpad][TILE] (!REG)
  if (a.smem_acc) {
    for (int i = tid; i < R * NJ; i += kKeyedTile) s_used[i] = 0ull;
    for (int i = tid; i < NJ; i += kKeyedTile) { s_cnt[i] = 0ull; s_pres[i] = 0u; }
    __syncthreads();
  }
  PodRows<REG> rows;
  rows.init(s_rowid, tid, kKeyedTile);
  const int64_t tiles = (pods.n + kKeyedTile - 1) / kKeyedTile;
#pragma unroll 1
  for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int64_t p = tile * kKeyedTile + tid;
    const bool valid = p < pods.n;
    const int64_t pc = valid ? p : pods.n - 1;
    const uint32_t flags = valid ? __ldg(&pods.flags[pc]) : 0u;
    const int ns = __ldg(&pods.ns[pc]);
    // shouldCountIn (throttle_controller.go:217-219), and a namespace that reaches a listed throttle at all
    const bool counted = (flags & (KT_POD_SCHEDULER_MATCH | KT_POD_SCHEDULED)) == (KT_POD_SCHEDULER_MATCH | KT_POD_SCHEDULED) &&
                         (unsigned)ns < (unsigned)a.tb.NS;
    const uint32_t* my_reach = a.reach + (size_t)(counted ? ns : 0) * a.NC;
    uint32_t any_reach = 0;
    if (counted)
      for (int c = 0; c < a.NC; ++c) any_reach |= __ldg(&my_reach[c]);
    const bool on = counted && any_reach != 0u;
    if (!__any_sync(kFull, on)) continue;
    const bool alive = on && (flags & KT_POD_NOT_FINISHED);  // isNotFinished (pod_util.go:26-28)
    const uint32_t present = on ? __ldg(&pods.present[pc]) & ~KT_COUNT_BIT : 0u;
    long long rq[RT > 0 ? RT : 1];
    if constexpr (RT > 0) {
#pragma unroll
      for (int r = 0; r < RT; ++r) rq[r] = (alive && r < R && ((present >> r) & 1)) ? __ldg(&pods.req[(int64_t)r * pods.n + pc]) : 0;
    }
    if (on) load_rows<REG>(pods.roff, pods.n, pc, a.L, rows);
#pragma unroll 1
    for (int c = 0; c < a.NC; ++c) {
      const uint32_t bits = on ? __ldg(&my_reach[c]) : 0u;
      uint32_t u = __reduce_or_sync(kFull, bits);
#pragma unroll 1
      while (u) {
        const int j = c * 32 + __ffs(u) - 1;
        u &= u - 1;
        uint32_t word = 0;
        if ((bits >> (j & 31)) & 1u) {
          word = eval_word<TPC, B, REG>(a.tb, rows, Lpad, ns, __ldg(&a.words[j])) & __ldg(&a.masks[j]);
          if (word) a.scratch[p * a.nw + j] = word;
        }
        // used = used.Add(ResourceAmountOfPod(p)) over the not-finished matched rows: lane b owns throttle (j, b) and the
        // set of this warp's rows that matched it; each matched throttle is summed by the whole warp
        const uint32_t T = warp_transpose32(alive ? word : 0u, lane);
        uint32_t hit = __ballot_sync(kFull, T != 0u);
#pragma unroll 1
        while (hit) {
          const int b = __ffs(hit) - 1;
          hit &= hit - 1;
          const uint32_t m = __shfl_sync(kFull, T, b);
          const bool in = (m >> lane) & 1u;
          const uint32_t pr = __reduce_or_sync(kFull, in ? present : 0u);
          const int cj = j * 32 + b;
          if (lane == 0) {
            if (a.smem_acc) {
              smem_add_u64(&s_cnt[cj], (unsigned long long)__popc(m));
              atomicOr(&s_pres[cj], pr);
            } else {
              atomicAdd(&a.cnt[cj], (unsigned long long)__popc(m));
              atomicOr(&a.pres[cj], pr);
            }
          }
          for (int r = 0; r < R; ++r) {
            long long v;
            if constexpr (RT > 0) {
              v = 0;
#pragma unroll
              for (int q = 0; q < RT; ++q)
                if (q == r) v = rq[q];
            } else {
              v = (alive && ((present >> r) & 1)) ? __ldg(&pods.req[(int64_t)r * pods.n + pc]) : 0;
            }
            const unsigned long long s = warp_sum_u64(in ? (unsigned long long)v : 0ull);
            if (lane == (r & 31) && s) {
              if (a.smem_acc) smem_add_u64(&s_used[(size_t)r * NJ + cj], s);
              else atomicAdd(&a.used[(size_t)r * NJ + cj], s);
            }
          }
        }
      }
    }
  }
  if (a.smem_acc) {  // CTA accumulators -> HBM: one add per (throttle, resource) this CTA touched
    __syncthreads();
    for (int i = tid; i < NJ; i += kKeyedTile) {
      if (s_cnt[i] == 0ull) continue;
      atomicAdd(&a.cnt[i], s_cnt[i]);
      atomicOr(&a.pres[i], s_pres[i]);
      for (int r = 0; r < R; ++r)
        if (s_used[(size_t)r * NJ + i]) atomicAdd(&a.used[(size_t)r * NJ + i], s_used[(size_t)r * NJ + i]);
    }
  }
}

// Status of listed entry e (throttle idx[e], compact accumulator cidx[e]): what a FRESH_STATUS pass reports for that column,
// written into column e of the k columns of `out`, as kt_get_reconcile_rows gathers them from the pass's.
__global__ void __launch_bounds__(128) k_keyed_status(int64_t k, const int32_t* __restrict__ idx, const int32_t* __restrict__ cidx, int R, int M, int NJ,
                                                      const ThrottleView tv, long long now, const unsigned long long* __restrict__ used,
                                                      const unsigned long long* __restrict__ cnt, const uint32_t* __restrict__ pres, const ReconcileView out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= k) return;
  const int t = idx[e], cj = cidx[e];
  const uint32_t tflags = tv.flags[t];
  const bool live = (tflags & KT_THR_RESPONSIBLE) && !(tflags & KT_THR_SELECTOR_ERROR);
  const uint32_t p = pres[cj];
  uint32_t m_used = 0, m_thr = 0, m_calc = 0;
  bool active = false;
  for (int r = 0; r <= R; ++r) {  // r == R: the pod count
    const bool is_res = r < R;
    const uint32_t mybit = is_res ? (1u << r) : KT_COUNT_BIT;
    const CalcThreshold ct = calculate_threshold(tv, t, r, is_res, mybit, (size_t)r * M + t, now);
    const long long used_val = (long long)(is_res ? used[(size_t)r * NJ + cj] : cnt[cj]);
    const bool used_has = is_res ? ((p >> r) & 1u) != 0u : used_val > 0;  // Counts stays nil with zero counted pods (Q3)
    // status.throttled = calculatedThreshold.IsThrottled(used, onEqual=true) (throttle_controller.go:133)
    const bool throttled = live && ct.calc_has && used_has && used_val >= ct.calc_val;
    if (used_has) m_used |= mybit;
    if (throttled) m_thr |= mybit;
    if (ct.calc_has) m_calc |= mybit;
    active = ct.active;
    if (is_res) {
      out.used[(size_t)r * k + e] = used_val;
      out.calc_thr[(size_t)r * k + e] = ct.calc_val;
    } else {
      out.used_cnt[e] = used_val;
      out.calc_cnt[e] = ct.calc_val;
    }
  }
  out.used_present[e] = m_used;
  out.throttled[e] = m_thr;
  out.calc_present[e] = m_calc;
  out.override_active[e] = active;
}

// ------------------------------------------------------------------------------------------------
// PreFilter by key: the GIVEN_STATUS check of k listed pending rows (kt_check_pending_rows).
//
// PreFilter sees the informer copy of .status plus the reservations (plugin.go:148-215), so nothing it decides depends on the
// running rows: the check of one pod costs the words of its own namespace, not a pass over the queue.
//   1. k_rows_prep   the pass's finalize tile, prep half only (kFinPrep), into this call's own pre-records [M]: the threshold
//                    CheckThrottledFor compares with and the given used + reserved.  In GIVEN_STATUS mode the prep half reads
//                    no clock (status.calculatedThreshold or spec.threshold), so `now` is 0 as in the host's queue passes.
//   2. k_check_rows  one lane per listed row (listed rows share no namespace locality): its row offsets, the words of its
//                    namespace's list with the pass's eval_word, and each non-zero word decided pair by pair from the
//                    pre-records (decide_word_direct_codes; in GIVEN_STATUS mode it reads no sums).
// Outputs go to the call's own block [k] admit | [k][2 Wp] codes | [k][Wp] words, zeroed before the launch, so that every word
// outside the row's namespace list reads 0 as in the pass's maintained rows.
// ------------------------------------------------------------------------------------------------
struct NoSync {  // finalize_tile's prep half signals nobody: the rows kernel is the next launch in the stream
  __device__ __forceinline__ void wait_reconciled() const {}
  __device__ __forceinline__ void wait_totals(const PartExchange&) const {}
  __device__ __forceinline__ void wait_matched() const {}
  __device__ __forceinline__ void wait_prepped() const {}
  __device__ __forceinline__ void signal_prepped() const {}
  __device__ __forceinline__ void signal_totals() const {}
  __device__ __forceinline__ unsigned* error_flag() const { return nullptr; }
};

__global__ void __launch_bounds__(128) k_rows_prep(const ThrottleView tv, int M, int R, int G, uint32_t eval_flags, unsigned char* __restrict__ pre) {
  finalize_tile(tv, M, R, G, 0, eval_flags, PartExchange{}, ReconcileView{}, pre, blockIdx.x, NoSync{}, nullptr, kFinPrep);
}

constexpr int kRowsTile = 64;  // listed rows per CTA (one lane per row)

struct RowsArgs {
  PodView pods;                  // the pending rows (roff / winfo current)
  TableView tb;
  int L, R;
  int64_t k;
  const int64_t* rows;           // [k] caller rows
  const uint32_t* dev_of;        // caller row -> device row, or null (rows stored as given)
  const unsigned char* pre;      // [M][pre_record_bytes(R)] from k_rows_prep
  uint32_t* words;               // [k][Wp]
  uint32_t* codes;               // [k][2 Wp]
  unsigned char* admit;          // [k]
};

__host__ __device__ inline size_t rows_smem_bytes(int L, int R, bool reg_rows) {
  return (size_t)R * kRowsTile * 8 + (reg_rows ? 0 : (size_t)((L + 7) & ~7) * kRowsTile * 4);
}

// ResourceAmountOfPod(pod) of the column `p` of req [R][n] into s_req[r * stride]: the non-zero requests are the only ones
// IsThrottledFor looks at (Q5), so their bits are returned
__device__ __forceinline__ uint32_t stage_requests(const int64_t* req, int64_t n, int64_t p, uint32_t present, int R, long long* s_req, int stride) {
  uint32_t nz = 0;
  for (int r = 0; r < R; ++r) {
    long long v = __ldg(&req[(int64_t)r * n + p]);
    if (!((present >> r) & 1)) v = 0;
    s_req[r * stride] = v;
    if (v != 0) nz |= 1u << r;
  }
  return nz;
}

// The check of one pending pod, one lane: the words of its namespace's list (winfo) evaluated with the pass's eval_word, each
// non-zero word stored and decided pair by pair from the pre-records (decide_word_direct_codes; GIVEN_STATUS reads no sums).
// wrow [Wp] / crow [2 Wp] must be zero: only the non-zero words are written.  Returns the admit byte.
template <int TPC, int B, bool REG>
__device__ __forceinline__ unsigned char check_words(const TableView& tb, const PodRows<REG>& rows, int Lpad, int ns, uint32_t winfo,
                                                     const unsigned char* pre, int R, const DecidePod& pod, uint32_t* wrow, uint32_t* crow) {
  WordCursor wc;
  wc.init(tb, winfo, ns, (unsigned)ns < (unsigned)tb.NS);  // a namespace out of range affects nothing
  const PartExchange px{};  // GIVEN_STATUS: the pre-records carry everything, no sums are read
  const size_t rec = pre_record_bytes(R);
  unsigned char ok = 1;
#pragma unroll 1
  for (int q = 0; q < wc.cnt; ++q) {
    const int w = wc.at(tb, q);
    const uint32_t word = eval_word<TPC, B, REG>(tb, rows, Lpad, ns, w);
    if (!word) continue;
    wrow[w] = word;
    const uint2 c = decide_word_direct_codes(word, w, pre, px, rec, R, tb.M, pod);
    *reinterpret_cast<uint2*>(&crow[2 * w]) = c;
    if (c.x | c.y) ok = 0;
  }
  return ok;
}

template <int TPC, int B, bool REG>
__global__ void __launch_bounds__(kRowsTile) k_check_rows(const RowsArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x;
  const int64_t i = (int64_t)blockIdx.x * kRowsTile + tid;
  if (i >= a.k) return;  // (no barrier and no warp collective below: each lane works alone)
  const int R = a.R, Wp = a.tb.Wp, Lpad = (a.L + 7) & ~7;
  const PodView& pods = a.pods;
  long long* s_req = reinterpret_cast<long long*>(smem_raw);                                   // [R][TILE]
  int32_t* s_rowid = reinterpret_cast<int32_t*>(smem_raw + (size_t)R * kRowsTile * 8);        // [Lpad][TILE] (!REG)
  const int64_t cr = __ldg(&a.rows[i]);
  const int64_t p = a.dev_of ? (int64_t)__ldg(&a.dev_of[cr]) : cr;
  const int ns = __ldg(&pods.ns[p]);
  const uint32_t present = __ldg(&pods.present[p]);
  const uint32_t winfo = __ldg(&pods.winfo[p]);
  const uint32_t nz = stage_requests(pods.req, pods.n, p, present, R, s_req + tid, kRowsTile);
  const DecidePod pod{s_req + tid, kRowsTile, nz, p};
  PodRows<REG> rows;
  rows.init(s_rowid, tid, kRowsTile);
  load_rows<REG>(pods.roff, pods.n, p, a.L, rows);
  a.admit[i] = check_words<TPC, B, REG>(a.tb, rows, Lpad, ns, winfo, a.pre, R, pod, a.words + i * Wp, a.codes + i * 2 * Wp);
}

// ------------------------------------------------------------------------------------------------
// affectedThrottles of k pods that live only in this call (kt_match_pods): the selector relation of pod versions an informer
// event carries (throttle_controller.go:248-269, clusterthrottle_controller.go:272-298), with no resident row read or written.
// One lane per listed pod, as in k_check_rows: its label slots become table row offsets in registers (translate8, the chunk
// k_unpack_packed translates while it is in registers), its namespace's words come from the list k_translate_rows packs
// (winfo_pack), and each word is evaluated with the pass's eval_word.  The CTA zeroes its [kRowsTile][Wp] block of the output
// first, so the words outside the namespace's list read 0 as in the pass's rows; the lanes then store their non-zero words.
// ------------------------------------------------------------------------------------------------
struct MatchArgs {
  TableView tb;
  int L;
  int64_t k;
  const int64_t* labels;  // [L][k] label codes (keyId << 32 | valId, KT_LABEL_EMPTY)
  const int32_t* ns;      // [k]
  uint32_t* words;        // [k][Wp]
};

// The label codes of column i of labels [L][k] as row offsets into the current tables, in the lane's rows (translate8, the chunk
// k_unpack_packed translates while it is in registers); slots L..Lpad read empty as the resident rows' padding does.
template <bool REG>
__device__ __forceinline__ void translate_labels(const TableView& tb, const int64_t* labels, int64_t k, int64_t i, int L, PodRows<REG>& rows) {
  const int Lpad = (L + 7) & ~7;
#pragma unroll 1
  for (int s0 = 0; s0 < Lpad; s0 += 8) {
    int64_t lab[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) lab[j] = s0 + j < L ? __ldg(&labels[(int64_t)(s0 + j) * k + i]) : KT_LABEL_EMPTY;
    uint4 ke[8];
    uint32_t o[8];
    translate8_keys(tb, lab, ke);
    translate8_rows(tb, lab, ke, o);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if constexpr (REG) rows.off[j] = o[j];  // (REG: L <= 8, one chunk)
      else rows.col[(s0 + j) * rows.stride] = o[j];
    }
  }
}

// The words that can apply to namespace ns, as k_translate_rows packs them for a resident row (0 for a namespace out of range)
__device__ __forceinline__ uint32_t ns_winfo(const TableView& tb, int ns) {
  if ((unsigned)ns >= (unsigned)tb.NS) return 0u;
  const int lo = __ldg(&tb.nsw_off[ns]);
  const int cnt = __ldg(&tb.nsw_off[ns + 1]) - lo;
  return cnt == 0 ? 0u : winfo_pack(cnt, __ldg(&tb.nsw_idx[lo]), cnt > 1 ? __ldg(&tb.nsw_idx[lo + 1]) : 0, tb.W);
}

__host__ __device__ inline size_t match_smem_bytes(int L, bool reg_rows) { return reg_rows ? 0 : (size_t)((L + 7) & ~7) * kRowsTile * 4; }

template <int TPC, int B, bool REG>
__global__ void __launch_bounds__(kRowsTile) k_match_pods(const MatchArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x;
  const int Wp = a.tb.Wp, Lpad = (a.L + 7) & ~7;
  const int64_t row0 = (int64_t)blockIdx.x * kRowsTile;
  {  // the block's output rows, coalesced (Wp is a multiple of 4)
    const int64_t rows_here = a.k - row0 < kRowsTile ? a.k - row0 : kRowsTile;
    uint4* d = reinterpret_cast<uint4*>(a.words + row0 * Wp);
    const int64_t nvec = rows_here * (Wp / 4);
    for (int64_t v = tid; v < nvec; v += kRowsTile) d[v] = make_uint4(0, 0, 0, 0);
  }
  __syncthreads();
  const int64_t i = row0 + tid;
  if (i >= a.k) return;  // (no barrier and no warp collective below: each lane works alone)
  const int ns = __ldg(&a.ns[i]);
  if ((unsigned)ns >= (unsigned)a.tb.NS) return;  // a namespace out of range affects nothing
  PodRows<REG> rows;
  rows.init(reinterpret_cast<int32_t*>(smem_raw), tid, kRowsTile);
  translate_labels<REG>(a.tb, a.labels, a.k, i, a.L, rows);
  const uint32_t winfo = ns_winfo(a.tb, ns);
  WordCursor wc;
  wc.init(a.tb, winfo, ns, true);
  uint32_t* wrow = a.words + i * Wp;
#pragma unroll 1
  for (int q = 0; q < wc.cnt; ++q) {
    const int w = wc.at(a.tb, q);
    const uint32_t word = eval_word<TPC, B, REG>(a.tb, rows, Lpad, ns, w);
    if (word) wrow[w] = word;
  }
}

// ------------------------------------------------------------------------------------------------
// PreFilter of k pods given by value (kt_check_pods): a manifest PreFilter, Reserve or Unreserve costs the words of the pod's
// namespace, with no row of the pending table read or written.  The front half is k_match_pods' (the label slots translated in
// the lane's rows, the namespace's word list from winfo_pack), the back half k_check_rows' (the requests in shared memory, each
// non-zero word decided from the pre-records k_rows_prep wrote for this call).  The pass reads no flags of a pending row, so the
// pods carry none.  Outputs go to the call's own block, zeroed before the launch, as in k_check_rows.
// ------------------------------------------------------------------------------------------------
struct PodsArgs {
  TableView tb;
  int L, R;
  int64_t k;
  const int64_t* labels;     // [L][k] label codes
  const int64_t* req;        // [R][k]
  const uint32_t* present;   // [k]
  const int32_t* ns;         // [k]
  const unsigned char* pre;  // [M][pre_record_bytes(R)] from k_rows_prep
  uint32_t* words;           // [k][Wp]
  uint32_t* codes;           // [k][2 Wp]
  unsigned char* admit;      // [k]
};

template <int TPC, int B, bool REG>
__global__ void __launch_bounds__(kRowsTile) k_check_pods(const PodsArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x;
  const int64_t i = (int64_t)blockIdx.x * kRowsTile + tid;
  if (i >= a.k) return;  // (no barrier and no warp collective below: each lane works alone)
  const int R = a.R, Wp = a.tb.Wp, Lpad = (a.L + 7) & ~7;
  long long* s_req = reinterpret_cast<long long*>(smem_raw);                              // [R][TILE]
  int32_t* s_rowid = reinterpret_cast<int32_t*>(smem_raw + (size_t)R * kRowsTile * 8);   // [Lpad][TILE] (!REG)
  const int ns = __ldg(&a.ns[i]);
  const uint32_t nz = stage_requests(a.req, a.k, i, __ldg(&a.present[i]), R, s_req + tid, kRowsTile);
  const DecidePod pod{s_req + tid, kRowsTile, nz, i};
  PodRows<REG> rows;
  rows.init(s_rowid, tid, kRowsTile);
  translate_labels<REG>(a.tb, a.labels, a.k, i, a.L, rows);
  a.admit[i] = check_words<TPC, B, REG>(a.tb, rows, Lpad, ns, ns_winfo(a.tb, ns), a.pre, R, pod, a.words + i * Wp, a.codes + i * 2 * Wp);
}

// ------------------------------------------------------------------------------------------------
// The scheduling queue summarised per throttle (kt_get_check_summary): what the last checking pass left in the dense codes,
// reduced over the rejected rows for every throttle at once.
// A warp takes 32 consecutive DEVICE rows (the per-throttle results do not depend on row order, so the rows stay where the layout
// put them; only the caller's row classes are read through the row map).  A row that is admitted, outside the range or of class 0
// costs its admit byte.  A rejected row reads its code words twice: once to count its non-zero codes (one alone makes its throttle
// the only blocker), once in warp lockstep to credit them.  A code's word and position name the throttle, so the lanes holding a
// non-zero code at the same place form the warp's group for that throttle: ballots give the counts per status, warp sums the
// requests, and one lane adds each into HBM -- one atomic per warp and throttle however many rows the throttle rejects.
// ------------------------------------------------------------------------------------------------
constexpr int kSummaryThreads = 256;

struct SummaryArgs {
  int64_t first, count;            // caller rows [first, first + count)
  int64_t n;                       // pending rows
  int Wc, R, M;                    // code words per row (2 Wp), resources, throttles
  const uint32_t* codes;           // [n][Wc] by device row
  const unsigned char* admit;      // [n]
  const int64_t* req;              // [R][n]
  const uint32_t* present;         // [n]
  const uint32_t* caller_of;       // device row -> caller row, or null (rows stored as given)
  const unsigned char* row_class;  // [count] by caller row - first, or null (every row class 1)
  unsigned long long* status_cnt;  // [3][M]
  unsigned long long* sole_cnt;    // [M]
  unsigned long long* held;        // [R][M]
  uint32_t* held_present;          // [M]
};

__global__ void __launch_bounds__(kSummaryThreads) k_check_summary(const SummaryArgs a) {
  const int lane = threadIdx.x & 31;
  // the device rows the range occupies: itself when rows are stored as given, anywhere when they are laid out by namespace
  const int64_t lo = a.caller_of ? 0 : a.first, rows = a.caller_of ? a.n : a.count;
  const int64_t stride = (int64_t)gridDim.x * kSummaryThreads;
#pragma unroll 1
  for (int64_t base = (int64_t)blockIdx.x * kSummaryThreads + (threadIdx.x & ~31); base < rows; base += stride) {
    const int64_t d = lo + base + lane;
    int cls = 0;
    if (base + lane < rows && !__ldg(&a.admit[d])) {
      const int64_t c = a.caller_of ? (int64_t)__ldg(&a.caller_of[d]) : d;
      if (c >= a.first && c < a.first + a.count) cls = a.row_class ? __ldg(&a.row_class[c - a.first]) : 1;
    }
    if (!__any_sync(kFull, cls != 0)) continue;
    const uint32_t* crow = a.codes + (cls ? d : 0) * a.Wc;
    int nz = 0;
    if (cls)
      for (int j = 0; j < a.Wc; ++j) {
        const uint32_t w = __ldg(&crow[j]);
        nz += __popc((w | w >> 1) & 0x55555555u);
      }
    const bool sole = cls == 1 && nz == 1;
    const uint32_t present = cls ? __ldg(&a.present[d]) & ~KT_COUNT_BIT : 0u;
#pragma unroll 1
    for (int j = 0; j < a.Wc; ++j) {
      const uint32_t w = cls ? __ldg(&crow[j]) : 0u;
      uint32_t u = __reduce_or_sync(kFull, (w | w >> 1) & 0x55555555u);  // the even bit of each position some lane has non-zero
#pragma unroll 1
      while (u) {
        const int q = __ffs(u) - 1;
        u &= u - 1;
        const int t = j * 16 + (q >> 1);
        if (t >= a.M) break;  // (warp-uniform; no code names a column beyond the throttles)
        const uint32_t code = (w >> q) & 3u;
        const uint32_t b1 = __ballot_sync(kFull, code == KT_CHECK_ACTIVE), b2 = __ballot_sync(kFull, code == KT_CHECK_INSUFFICIENT);
        const uint32_t b3 = __ballot_sync(kFull, code == KT_CHECK_POD_REQUESTS_EXCEEDS_THRESHOLD);
        const uint32_t bs = __ballot_sync(kFull, code != 0u && sole);
        const uint32_t pr = __reduce_or_sync(kFull, code ? present : 0u);
        if (lane == 0) {
          if (a.status_cnt) {
            if (b1) atomicAdd(&a.status_cnt[t], (unsigned long long)__popc(b1));
            if (b2) atomicAdd(&a.status_cnt[(size_t)a.M + t], (unsigned long long)__popc(b2));
            if (b3) atomicAdd(&a.status_cnt[(size_t)2 * a.M + t], (unsigned long long)__popc(b3));
          }
          if (a.sole_cnt && bs) atomicAdd(&a.sole_cnt[t], (unsigned long long)__popc(bs));
          if (a.held_present) atomicOr(&a.held_present[t], pr | KT_COUNT_BIT);
        }
        if (a.held)
          for (int r = 0; r < a.R; ++r) {
            const long long v = (code && ((present >> r) & 1u)) ? __ldg(&a.req[(int64_t)r * a.n + d]) : 0;
            const unsigned long long s = warp_sum_u64((unsigned long long)v);  // two's complement: exact modulo 2^64
            if (lane == (r & 31) && s) atomicAdd(&a.held[(size_t)r * a.M + t], s);
          }
      }
    }
  }
}

}  // namespace kt
