// kt_nsrows.cuh -- namespace row deltas on the device (kt_update_namespace_rows), and the namespace side of selector column
// deltas (kt_update_selector_rows).
//
// A namespace's labels feed two things of the compiled tables: its own nsmask row ([W][TPpad], which throttle terms can apply to
// its pods) and its entry in the per-namespace word lists (nsw_off / nsw_idx).  The pod-label tables (table, need, keydir, valrow,
// hash) do not depend on namespaces.  So a Namespace event re-evaluates the listed rows here, from a device copy of the namespace
// side of the selector spec (NsSpecView, staged by kt_upload_throttles), and rebuilds the word lists from the nsmask rows:
//   1. k_ns_rows     one warp per (listed namespace, 32-throttle word), one lane per throttle: its terms in order, as
//                    compile_tables (kt_tables.cc) builds the row -- a ClusterThrottle term's namespaceSelector over the row's
//                    labels, a Throttle term's namespace equality, a KT_TERM_POD_INVALID term switching the later terms off
//                    where it applies -- one ballot per term plane
//   2. k_ns_count    one warp per namespace: how many of its words have a non-zero plane
//   3. k_ns_scan     one CTA: the counts -> nsw_off, plus the total and the longest list (brought back to the host)
//   4. k_ns_fill     one warp per namespace: the non-zero words in ascending order into nsw_idx
//   5. k_ns_winfo    one lane per resident pod row: the words inlined with the row (winfo_pack), from the new lists
// A selector column delta changes the other axis: k_ns_cols re-evaluates the listed 32-throttle words for every namespace with
// the same per-lane walk as k_ns_rows (ns_word_planes), then steps 2-5 follow.  k_scatter_words / k_scatter_kind_flags land the
// host-recompiled table and need slices of those words and the listed columns' kind and flags.
// A column append (kt_append_throttle_rows) grows M: k_widen_cols restrides the resident per-throttle arrays (and nsmask when W
// grows) in one launch, filling in the staged new columns, then k_ns_cols takes the touched words and steps 2-5 follow.
// A column move (kt_move_throttle_columns) renumbers the columns: every per-column bit is column-local, so k_gather_bits gathers
// table, need and nsmask by column in one launch, k_widen_cols restrides the per-throttle arrays through the same column map, and
// steps 2-5 follow -- no namespace is evaluated again.
#pragma once
#include "kt_keyed.cuh"

namespace kt {

constexpr uint8_t kTermUnsat = 0x80u;  // staged term flag: the podSelector needs more keys than a pod row holds (HostTables::term_unsat)
constexpr int kNsScanThreads = 1024;

// What compile_tables reads to build the namespace masks, on the device
struct NsSpecView {
  const int32_t* term_off;     // [M+1]
  const int32_t* ns_req_off;   // [n_terms+1]
  const uint8_t* term_flags;   // [n_terms] KT_TERM_NS_INVALID | KT_TERM_POD_INVALID | kTermUnsat
  const uint32_t* req_key;     // [n_reqs]
  const uint8_t* req_op;       // [n_reqs]
  const int32_t* req_val_off;  // [n_reqs+1]
  const uint32_t* req_vals;    // [n_vals]
  const int32_t* ns_id;        // [M]
  const uint8_t* kind;         // [M] (the throttle columns)
  const uint8_t* flags;        // [M]
  int32_t M, W, TPpad;
};

// The namespaceSelector of one term over one namespace row (labels[s * stride], LN slots): kt_tables.cc ns_term_matches
__device__ __forceinline__ bool ns_term_holds(const NsSpecView& sp, int term, uint8_t tf, const int64_t* labels, int64_t stride, int LN) {
  if (tf & KT_TERM_NS_INVALID) return false;
  const int q1 = __ldg(&sp.ns_req_off[term + 1]);
  for (int q = __ldg(&sp.ns_req_off[term]); q < q1; ++q) {
    const uint32_t key = __ldg(&sp.req_key[q]);
    const uint8_t op = __ldg(&sp.req_op[q]);
    bool has = false;
    uint32_t val = 0;
    for (int s = 0; s < LN; ++s) {
      const int64_t l = __ldg(&labels[(int64_t)s * stride]);
      if (l == KT_LABEL_EMPTY) continue;
      if ((uint32_t)((uint64_t)l >> 32) == key) { has = true; val = (uint32_t)((uint64_t)l & 0xffffffffu); break; }
    }
    bool ok;
    if (!has) {
      ok = op == KT_OP_NOTIN || op == KT_OP_DOESNOTEXIST;
    } else if (op == KT_OP_IN || op == KT_OP_NOTIN) {
      bool in = false;
      const int v1 = __ldg(&sp.req_val_off[q + 1]);
      for (int v = __ldg(&sp.req_val_off[q]); v < v1 && !in; ++v) in = __ldg(&sp.req_vals[v]) == val;
      ok = (op == KT_OP_IN) == in;
    } else {
      ok = op == KT_OP_EXISTS;
    }
    if (!ok) return false;
  }
  return true;
}

// One warp's nsmask entry of namespace ns and 32-throttle word w, one lane per throttle: its terms in order, as compile_tables
// builds them -- a ClusterThrottle term's namespaceSelector over the namespace's labels (slot s at labels[col + s * stride]; read
// for ns < n_ns only), a Throttle term's namespace equality, a KT_TERM_POD_INVALID term switching the later terms off where it
// applies -- one ballot per term plane, written by lane 0 to the namespace's entry of that word in nsmask ([NS][W][TPpad]).
__device__ __forceinline__ void ns_word_planes(const NsSpecView& sp, int w, int lane, int ns, const int64_t* labels, int col, int64_t stride,
                                               int LN, int32_t n_ns, uint32_t* nsmask) {
  const int t = w * 32 + lane;
  int term0 = 0, nterm = 0;
  bool cluster = false, own = false;
  if (t < sp.M) {
    const uint8_t f = __ldg(&sp.flags[t]);
    if ((f & KT_THR_RESPONSIBLE) && !(f & KT_THR_SELECTOR_ERROR)) {
      term0 = __ldg(&sp.term_off[t]);
      nterm = __ldg(&sp.term_off[t + 1]) - term0;
    }
    cluster = __ldg(&sp.kind[t]) != KT_KIND_THROTTLE;
    own = __ldg(&sp.ns_id[t]) == ns;
  }
  bool blocked = false;  // a KT_TERM_POD_INVALID term of this throttle applies to the namespace: the later terms are off
  uint32_t* row = nsmask + ((size_t)ns * sp.W + w) * sp.TPpad;
  for (int s = 0; s < sp.TPpad; ++s) {
    bool bit = false;
    if (s < nterm) {
      const int term = term0 + s;
      const uint8_t tf = __ldg(&sp.term_flags[term]);
      if ((tf & KT_TERM_POD_INVALID) || !(tf & kTermUnsat)) {
        const bool applies = cluster ? ns < n_ns && ns_term_holds(sp, term, tf, labels + col, stride, LN) : own;
        if (tf & KT_TERM_POD_INVALID) blocked |= applies;
        else bit = applies && !blocked;
      }
    }
    const uint32_t word = __ballot_sync(kFull, bit);
    if (lane == 0) row[s] = word;
  }
}

// nsmask rows of the kd listed namespaces ns_ids[i], labels [LN][kd]; n_ns: the namespace count (a ClusterThrottle term applies to
// namespaces below it only).  grid (ceil(W / 8), up to 65535 rows from y0), 256 threads: warp = word.
__global__ void __launch_bounds__(256) k_ns_rows(const NsSpecView sp, int32_t y0, int32_t kd, const int32_t* __restrict__ ns_ids,
                                                 const int64_t* __restrict__ labels, int LN, int32_t n_ns, uint32_t* __restrict__ nsmask) {
  const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= sp.W) return;  // whole warps
  const int i = y0 + blockIdx.y;
  const int ns = __ldg(&ns_ids[i]);
  ns_word_planes(sp, w, lane, ns, labels, i, kd, LN, n_ns, nsmask);
}

// nsmask entries of the nw listed words (words[]) for all NS namespaces, labels [LN][n_ns] (kt_update_selector_rows: the columns
// of those words changed).  One warp per (namespace, listed word): warp g takes namespace g % NS of word g / NS, so the warps of
// a CTA share one word's spec.  grid ceil(NS * nw / 8), 256 threads.
__global__ void __launch_bounds__(256) k_ns_cols(const NsSpecView sp, int32_t NS, int32_t nw, const int32_t* __restrict__ words,
                                                 const int64_t* __restrict__ labels, int LN, int32_t n_ns, uint32_t* __restrict__ nsmask) {
  const int64_t g = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (g >= (int64_t)NS * nw) return;  // whole warps
  const int lane = threadIdx.x & 31, ns = (int)(g % NS), w = __ldg(&words[g / NS]);
  ns_word_planes(sp, w, lane, ns, labels, ns, n_ns, LN, n_ns, nsmask);
}

// Word slices of the listed words: dst[words[j] * len + e] = src[j * len + e] (table / need slices of kt_update_selector_rows)
__global__ void __launch_bounds__(256) k_scatter_words(int64_t nw, const int32_t* __restrict__ words, int64_t len, const uint32_t* __restrict__ src,
                                                       uint32_t* __restrict__ dst) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nw * len; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = i / len, e = i - j * len;
    dst[(int64_t)__ldg(&words[j]) * len + e] = src[i];
  }
}

// One array of `rows` rows of `esize`-byte elements (1, 4 or 8) widened from m_old to m_new elements per row: element e < m_old of
// row r from src[r * m_old + e], the others from add[r * (m_new - m_old) + e - m_old], or zero when add is null.  dst must not
// overlap src.  With m_old = 0 and src null it is a plain copy of `add` into dst.  With a column map (map[m_new], a column
// move) element e of row r comes from src[r * m_old + map[e]] instead, or is zero where map[e] is -1; add is then unused.
struct WidenArray {
  const unsigned char* src;
  const unsigned char* add;
  unsigned char* dst;
  int64_t rows, m_old, m_new;
  int32_t esize;
  const int32_t* map;
};
constexpr int kMaxWiden = 24;
struct WidenBatch {
  WidenArray a[kMaxWiden];
  int32_t n;
};
template <class T>
__device__ __forceinline__ void widen_elems(const WidenArray& a, int64_t i0, int64_t stride) {
  const T* src = reinterpret_cast<const T*>(a.src);
  const T* add = reinterpret_cast<const T*>(a.add);
  T* dst = reinterpret_cast<T*>(a.dst);
  const int64_t k = a.m_new - a.m_old, n = a.rows * a.m_new;
  for (int64_t i = i0; i < n; i += stride) {
    const int64_t r = i / a.m_new, e = i - r * a.m_new;
    if (a.map) {
      const int32_t from = a.map[e];
      dst[i] = from >= 0 ? src[r * a.m_old + from] : T(0);
    } else {
      dst[i] = e < a.m_old ? src[r * a.m_old + e] : add ? add[r * k + (e - a.m_old)] : T(0);
    }
  }
}
// grid (x, b.n): blockIdx.y is the array
__global__ void __launch_bounds__(256) k_widen_cols(const WidenBatch b) {
  const WidenArray& a = b.a[blockIdx.y];
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
  if (a.esize == 8) widen_elems<uint64_t>(a, i0, stride);
  else if (a.esize == 4) widen_elems<uint32_t>(a, i0, stride);
  else widen_elems<uint8_t>(a, i0, stride);
}

// A bit-sliced array gathered by column: `outer` blocks of w_old 32-throttle words of `len` u32 each ([outer][w_old][len]) into
// [outer][w_new][len].  Output word (o, w, l) bit j is bit (s & 31) of input word (o, s >> 5, l) for s = map[32w + j], or the
// fill bit for s = -1 and for 32w + j >= m: bit 1 at even l when fill_even is set (the table's sat planes, as compile_tables
// starts a column), else 0.
struct GatherBitsArray {
  const uint32_t* src;
  uint32_t* dst;
  int64_t outer, len;
  int32_t w_old, w_new;
  bool fill_even;
};
struct GatherBitsBatch {
  GatherBitsArray a[3];
  const int32_t* map;
  int32_t m;
};
// grid (x, 3): blockIdx.y is the array.  One warp per run of 32 output words of one (o, w): lane j holds column 32w + j's source
// word and bit, each output word is one load per lane -- a broadcast when the run's sources share a word, as they do for a
// compaction -- and one ballot; lane l of the warp keeps word l of the run, so the run is stored in one coalesced write.
__global__ void __launch_bounds__(256) k_gather_bits(const GatherBitsBatch b) {
  const GatherBitsArray& a = b.a[blockIdx.y];
  const int lane = threadIdx.x & 31;
  const int64_t runs = (a.len + 31) >> 5, items = a.outer * a.w_new * runs;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t it = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); it < items; it += warps) {
    const int64_t run = it % runs, ow = it / runs, o = ow / a.w_new;
    const int32_t w = (int32_t)(ow - o * a.w_new);
    const int32_t col = w * 32 + lane;
    const int32_t s = col < b.m ? b.map[col] : -1;
    const uint32_t* in = s >= 0 ? a.src + ((size_t)o * a.w_old + (s >> 5)) * a.len : nullptr;
    const int64_t l0 = run << 5, l1 = min(a.len, l0 + 32);
    uint32_t mine = 0;
    for (int64_t l = l0; l < l1; ++l) {
      const bool bit = in ? (in[l] >> (s & 31)) & 1u : a.fill_even && !(l & 1);
      const uint32_t word = __ballot_sync(0xffffffffu, bit);
      if (lane == (int)(l - l0)) mine = word;
    }
    if (l0 + lane < l1) a.dst[((size_t)o * a.w_new + w) * a.len + l0 + lane] = mine;
  }
}

// kind and flags of the k listed throttle columns (kt_update_selector_rows)
__global__ void __launch_bounds__(128) k_scatter_kind_flags(int64_t k, const int32_t* __restrict__ idx, const uint8_t* __restrict__ src_kind,
                                                            const uint8_t* __restrict__ src_flags, uint8_t* kind, uint8_t* flags) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k) return;
  kind[idx[i]] = src_kind[i];
  flags[idx[i]] = src_flags[i];
}

__device__ __forceinline__ bool ns_word_live(const uint32_t* __restrict__ nsmask, int ns, int w, int W, int TPpad) {
  const uint32_t* e = nsmask + ((size_t)ns * W + w) * TPpad;
  uint32_t any = 0;
  for (int s = 0; s < TPpad; ++s) any |= __ldg(&e[s]);
  return any != 0;
}

// cnt[ns] = the words of namespace ns with a non-zero plane.  One warp per namespace, 8 per CTA.
__global__ void __launch_bounds__(256) k_ns_count(int32_t NS, int W, int TPpad, const uint32_t* __restrict__ nsmask, int32_t* __restrict__ cnt) {
  const int ns = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (ns >= NS) return;
  int c = 0;
  for (int w0 = 0; w0 < W; w0 += 32) {
    const int w = w0 + lane;
    c += __popc(__ballot_sync(kFull, w < W && ns_word_live(nsmask, ns, w, W, TPpad)));
  }
  if (lane == 0) cnt[ns] = c;
}

// off[0..NS] = exclusive scan of cnt[0..NS); out = {total, longest list}.  One CTA, each thread a run of consecutive namespaces.
__global__ void __launch_bounds__(kNsScanThreads) k_ns_scan(int32_t NS, const int32_t* __restrict__ cnt, int32_t* __restrict__ off, int32_t* __restrict__ out) {
  __shared__ int32_t part[kNsScanThreads];
  __shared__ int32_t longest;
  const int tid = threadIdx.x;
  const int per = (NS + kNsScanThreads - 1) / kNsScanThreads;
  const int lo = min(NS, tid * per), hi = min(NS, lo + per);
  int32_t sum = 0, mx = 0;
  for (int i = lo; i < hi; ++i) { sum += cnt[i]; mx = max(mx, cnt[i]); }
  if (tid == 0) longest = 0;
  part[tid] = sum;
  __syncthreads();
  atomicMax(&longest, mx);
  for (int d = 1; d < kNsScanThreads; d <<= 1) {  // inclusive scan of the per-thread sums
    const int32_t v = tid >= d ? part[tid - d] : 0;
    __syncthreads();
    part[tid] += v;
    __syncthreads();
  }
  int32_t at = part[tid] - sum;
  for (int i = lo; i < hi; ++i) { off[i] = at; at += cnt[i]; }
  if (tid == kNsScanThreads - 1) {
    off[NS] = part[tid];
    out[0] = part[tid];
    out[1] = longest;
  }
}

// nsw_idx[off[ns] ..] = the live words of namespace ns in ascending order.  One warp per namespace.
__global__ void __launch_bounds__(256) k_ns_fill(int32_t NS, int W, int TPpad, const uint32_t* __restrict__ nsmask, const int32_t* __restrict__ off,
                                                 int32_t* __restrict__ idx) {
  const int ns = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (ns >= NS) return;
  int at = off[ns];
  for (int w0 = 0; w0 < W; w0 += 32) {
    const int w = w0 + lane;
    const bool live = w < W && ns_word_live(nsmask, ns, w, W, TPpad);
    const uint32_t b = __ballot_sync(kFull, live);
    if (live) idx[at + __popc(b & ((1u << lane) - 1u))] = w;
    at += __popc(b);
  }
}

// The words inlined with each resident pod row, from the new word lists (k_translate_rows' winfo; the row offsets stay valid)
__global__ void __launch_bounds__(256) k_ns_winfo(int64_t n, const TableView tb, const int32_t* __restrict__ ns_col, uint32_t* __restrict__ winfo) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) winfo[p] = ns_winfo(tb, __ldg(&ns_col[p]));
}

}  // namespace kt
