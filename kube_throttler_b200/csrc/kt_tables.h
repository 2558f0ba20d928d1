// kt_tables.h -- selector compiler: turns the CSR selector table of include/kt_b200.h into the
// bit-sliced match tables the sm_90a kernels scan (DESIGN.md "Bit-sliced selector match").
//
// This is packer-side work that runs when Throttles/ClusterThrottles/Namespaces change, not per pass.
// It replaces what the reference redoes on EVERY MatchesToPod call:
//   metav1.LabelSelectorAsSelector(&t.PodSelector)      (v1alpha1/throttle_selector.go:49)
//   metav1.LabelSelectorAsSelector(&t.NamespaceSelector) (v1alpha1/clusterthrottle_selector.go:64)
// It contains no pod-evaluation code: matching pods happens only on the GPU.
#pragma once
#include <cstdint>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/kt_b200.h"

namespace kt {

// Host copy of everything table compilation depends on (the caller's pointers are not retained).
struct SelectorSpec {
  int32_t m = 0;
  std::vector<uint8_t> kind, flags;
  std::vector<int32_t> ns_id;
  std::vector<int32_t> term_off, pod_req_off, ns_req_off, req_val_off;
  std::vector<uint8_t> term_flags, req_op;
  std::vector<uint32_t> req_key, req_vals;
};

// A table row of a key that some podSelector requirement mentions
struct RowRef {
  int32_t row;
  bool other;    // the "some other value" row of the key
  uint32_t val;  // valid when !other
};
using RowsOfKey = std::unordered_map<uint32_t, std::vector<RowRef>>;

struct HostTables {
  int32_t M = 0;
  int32_t W = 0;       // ceil(M/32)
  int32_t Wp = 0;      // words per bitmap row (multiple of 4)
  int32_t TP = 1;      // max terms per throttle
  int32_t TPpad = 1;   // planes stored per entry (1, or TP rounded up to even)
  int32_t B = 1;       // counter bit-planes: bit_width(max #positive keys of a term)
  int32_t rows = 1;    // table rows incl. the neutral row (index rows-1)
  int32_t NS = 0;      // namespaces covered by nsmask
  uint32_t hash_mask = 0;
  std::vector<uint32_t> hash;    // [hash_mask+1][4]: {keyId, valId (0xffffffff = the key's "other value" row), row, 0}; empty = {~0,~0,0,0}
  // Two-level direct dictionary (the fast path; dictionary ids handed out by a packer are small and dense).
  // Rows are stored as "roff" = row * TPpad * 8, the byte offset of the row inside a word slice of `table`.
  //   keydir[keyId] = {other roff, vmin, vcnt, off}; off == 0xffffffff (vcnt = 0): the key's values live in `hash`
  //   keydir[n_keydir] = {neutral roff, 0, 0, 0}: sentinel for every key id >= n_keydir (unmentioned key)
  //   valrow[off + (valId - vmin)] = roff, or kOtherRoff (0xfffffffe) for "a value no requirement mentions";
  //   valrow[0] = kOtherRoff is the sentinel out-of-range values read.
  // n_keydir == 0 (some mentioned keyId >= kKeyDirMax): every label goes through `hash`.
  int32_t n_keydir = 0;
  std::vector<uint32_t> keydir;  // [n_keydir + 1][4]
  std::vector<uint32_t> valrow;
  std::vector<uint32_t> table;   // [W][rows][TPpad][2]: {sat, pos}
  std::vector<uint32_t> need;    // [W][TPpad][B]
  std::vector<uint8_t> term_unsat;  // [n_terms] 1: the podSelector needs more keys than a pod row holds (the term matches nobody)
  std::vector<uint32_t> nsmask;  // [NS][W][TPpad]
  std::vector<int32_t> nsw_off;  // [NS+1]
  std::vector<int32_t> nsw_idx;  // non-zero words per namespace
  int32_t max_ns_words = 0;      // longest per-namespace word list
  // the row dictionary the table was built with: every row of each mentioned key, and the row of each mentioned (key, value)
  RowsOfKey rows_of_key;
  std::map<uint64_t, int32_t> pair_row;  // (key << 32 | value) -> row
};

// Validates the CSR arrays and copies them.  Returns "" or an error description.
std::string copy_selector_spec(int32_t m, const kt_throttle_cols* cols, const kt_selector_table* sel, SelectorSpec* out);

// Builds the tables.  ns_labels: [LN][n_ns] (may be null when n_ns == 0).
std::string compile_tables(const kt_limits& lim, const SelectorSpec& spec, int32_t n_ns, const int64_t* ns_labels,
                           HostTables* out);

// One column's table bits, term need counts and unsatisfiable terms (see kt_tables.cc); compile_tables builds every column with it.
int32_t compile_column(const kt_limits& lim, const SelectorSpec& spec, int32_t t, const RowsOfKey& rows_of_key, int32_t rows,
                       int32_t TPpad, uint32_t* word_table, int32_t* need, uint8_t* term_unsat);

// The listed columns of h (compiled from old_spec) recompiled in place from `spec`, which equals old_spec but for the listed
// columns: their table bits, need planes and term_unsat entries, with compile_column.  `spec` may be longer than old_spec when
// every column it grew by is listed: M, W and Wp grow, and the words it adds are appended to `table` and `need` (the existing
// words keep their place).  false when one of them does not fit the resident tables -- a podSelector key or (key, value)
// without a row, more terms than TPpad, a need beyond the B counter planes, a Throttle namespace beyond NS --; h is then partly
// patched and must be compiled again.  The namespace masks and word lists are not touched (nsmask, nsw_off, nsw_idx,
// max_ns_words), nor resized when W grows.
bool patch_columns(const kt_limits& lim, const SelectorSpec& old_spec, const SelectorSpec& spec, const std::vector<int32_t>& listed,
                   HostTables* h);

constexpr uint32_t kKeyDirMax = 1u << 16;  // direct key table only for key ids below this

inline int32_t words_per_row(int32_t m) {
  int32_t w = (m + 31) / 32;
  w = (w + 3) / 4 * 4;
  return w < 4 ? 4 : w;
}

#ifdef __CUDACC__
#define KT_HOST_DEVICE __host__ __device__ __forceinline__
#else
#define KT_HOST_DEVICE inline
#endif
// 32-bit mixer of a (keyId, valId) label; the kernels and the table compiler must agree on it.
KT_HOST_DEVICE uint32_t label_hash(uint32_t key, uint32_t val) {
  uint32_t h = key * 0x9E3779B1u + val * 0x85EBCA77u;
  h ^= h >> 16;
  h *= 0x7feb352du;
  h ^= h >> 15;
  return h;
}

}  // namespace kt
