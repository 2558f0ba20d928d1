// kt_tables.cc -- selector compiler (see kt_tables.h).  Plain C++17, no CUDA.
//
// Formulation (DESIGN.md "Bit-sliced selector match").  Throttle t lives at bit (t & 31) of word
// (t >> 5); its s-th selectorTerm lives in plane s.  For a term J and a label key k that J constrains,
// everything J asks of k depends only on the pod's value for k (or its absence):
//   sat_J,k(v)   all of J's requirements on k hold for value v     -> one bit per (row(k,v), J)
//   pos_J,k      J has a requirement on k that needs the key present (In / Exists / matchLabels)
// Rows: one per (key, value) pair that any requirement mentions, one "other value" row per mentioned
// key, plus a neutral row (sat=~0, pos=0) for labels no selector mentions.  A pod matches J iff
//   AND over its labels of sat[row(label)]  AND  (#labels with pos) == need_J
// because pod label keys are distinct, so the count equals need_J exactly when every key J needs is
// present.  need_J = number of distinct keys J has a positive requirement on.
#include "kt_tables.h"

#include <algorithm>
#include <map>
#include <unordered_map>

namespace kt {

std::string copy_selector_spec(int32_t m, const kt_throttle_cols* cols, const kt_selector_table* sel, SelectorSpec* out) {
  if (m < 0) return "m < 0";
  if (!cols || !sel) return "null cols/sel";
  if (m > 0 && (!cols->kind || !cols->ns_id || !cols->flags || !sel->term_off)) return "null throttle columns";
  SelectorSpec s;
  s.m = m;
  s.kind.assign(cols->kind, cols->kind + m);
  s.flags.assign(cols->flags, cols->flags + m);
  s.ns_id.assign(cols->ns_id, cols->ns_id + m);
  if (m == 0) { s.term_off = {0}; s.pod_req_off = {0}; s.ns_req_off = {0}; s.req_val_off = {0}; *out = std::move(s); return ""; }
  s.term_off.assign(sel->term_off, sel->term_off + m + 1);
  const int32_t nt = sel->n_terms, nq = sel->n_reqs, nv = sel->n_vals;
  if (nt < 0 || nq < 0 || nv < 0) return "negative selector sizes";
  if (s.term_off[0] != 0 || s.term_off[m] != nt) return "term_off must span [0, n_terms]";
  for (int32_t t = 0; t < m; ++t)
    if (s.term_off[t] > s.term_off[t + 1]) return "term_off not monotone";
  if (nt > 0 && (!sel->pod_req_off || !sel->ns_req_off || !sel->term_flags)) return "null term arrays";
  if (nt > 0) {
    s.pod_req_off.assign(sel->pod_req_off, sel->pod_req_off + nt + 1);
    s.ns_req_off.assign(sel->ns_req_off, sel->ns_req_off + nt + 1);
    s.term_flags.assign(sel->term_flags, sel->term_flags + nt);
  } else {
    s.pod_req_off = {0};
    s.ns_req_off = {0};
  }
  for (int32_t i = 0; i < nt; ++i) {
    if (s.pod_req_off[i] < 0 || s.pod_req_off[i] > s.pod_req_off[i + 1] || s.pod_req_off[i + 1] > nq) return "pod_req_off out of range";
    if (s.ns_req_off[i] < 0 || s.ns_req_off[i] > s.ns_req_off[i + 1] || s.ns_req_off[i + 1] > nq) return "ns_req_off out of range";
  }
  if (nq > 0 && (!sel->req_key || !sel->req_op || !sel->req_val_off)) return "null requirement arrays";
  s.req_key.assign(sel->req_key, sel->req_key + nq);
  s.req_op.assign(sel->req_op, sel->req_op + nq);
  if (nq > 0) s.req_val_off.assign(sel->req_val_off, sel->req_val_off + nq + 1);
  else s.req_val_off = {0};
  for (int32_t q = 0; q < nq; ++q) {
    if (s.req_op[q] > KT_OP_DOESNOTEXIST) return "unknown requirement operator";
    if (s.req_val_off[q] < 0 || s.req_val_off[q] > s.req_val_off[q + 1] || s.req_val_off[q + 1] > nv) return "req_val_off out of range";
    if (s.req_key[q] == 0xffffffffu) return "key id 0xffffffff is reserved";
  }
  if (nv > 0 && !sel->req_vals) return "null req_vals";
  s.req_vals.assign(sel->req_vals, sel->req_vals + nv);
  for (uint32_t v : s.req_vals)
    if (v == 0xffffffffu) return "value id 0xffffffff is reserved";
  for (int32_t t = 0; t < m; ++t)
    if (s.kind[t] > KT_KIND_CLUSTERTHROTTLE) return "unknown throttle kind";
  *out = std::move(s);
  return "";
}

namespace {

// Does requirement q hold for a label whose key equals the requirement's key and whose value is `val`
// (or some value no requirement mentions when other==true)?
inline bool req_holds_present(const SelectorSpec& s, int32_t q, bool other, uint32_t val) {
  auto in_set = [&]() {
    if (other) return false;
    for (int32_t i = s.req_val_off[q]; i < s.req_val_off[q + 1]; ++i)
      if (s.req_vals[i] == val) return true;
    return false;
  };
  switch (s.req_op[q]) {
    case KT_OP_IN: return in_set();
    case KT_OP_NOTIN: return !in_set();
    case KT_OP_EXISTS: return true;
    default: return false;  // DoesNotExist with the key present
  }
}

// namespaceSelector evaluation for ONE namespace row (tiny: NS x cluster terms, only when
// namespaces or throttles change).  Namespaces are not pods: the pod hot path never runs here.
inline bool ns_term_matches(const SelectorSpec& s, int32_t term, const int64_t* ns_labels, int32_t n_ns, int32_t ns, int slots) {
  if (s.term_flags[term] & KT_TERM_NS_INVALID) return false;
  for (int32_t q = s.ns_req_off[term]; q < s.ns_req_off[term + 1]; ++q) {
    bool has = false;
    uint32_t val = 0;
    for (int i = 0; i < slots; ++i) {
      int64_t l = ns_labels[(int64_t)i * n_ns + ns];
      if (l == KT_LABEL_EMPTY) continue;
      if ((uint32_t)((uint64_t)l >> 32) == s.req_key[q]) { has = true; val = (uint32_t)((uint64_t)l & 0xffffffffu); break; }
    }
    bool ok = has ? req_holds_present(s, q, false, val) : (s.req_op[q] == KT_OP_NOTIN || s.req_op[q] == KT_OP_DOESNOTEXIST);
    if (!ok) return false;
  }
  return true;
}

// need counts of one column's terms -> its bit in the word's counter planes ([TPpad][B] of the word)
void put_need(int32_t t, int32_t n_terms, const int32_t* need, int32_t TPp, int32_t B, uint32_t* word_need) {
  for (int32_t sidx = 0; sidx < n_terms; ++sidx)
    for (int32_t b = 0; b < B; ++b)
      if ((need[sidx] >> b) & 1) word_need[(size_t)sidx * B + b] |= 1u << (t & 31);
}

}  // namespace

// Throttle t's bits in its word's slice of the table ([rows][TPpad][2], which the caller set to sat = 1 / pos = 0 for t), the
// need count of each of its terms (need[sidx]) and which of them can never match (term_unsat[sidx]); returns the largest need.
int32_t compile_column(const kt_limits& lim, const SelectorSpec& s, int32_t t, const RowsOfKey& rows_of_key, int32_t rows, int32_t TPp,
                       uint32_t* word_table, int32_t* need, uint8_t* term_unsat) {
  const uint32_t bit = 1u << (t & 31);
  int32_t max_need = 0;
  for (int32_t term = s.term_off[t], sidx = 0; term < s.term_off[t + 1]; ++term, ++sidx) {
    // group this term's requirements by key
    std::map<uint32_t, std::vector<int32_t>> by_key;
    for (int32_t q = s.pod_req_off[term]; q < s.pod_req_off[term + 1]; ++q) by_key[s.req_key[q]].push_back(q);
    int32_t nd = 0;
    for (auto& kv : by_key) {
      bool positive = false;
      for (int32_t q : kv.second) positive |= (s.req_op[q] == KT_OP_IN || s.req_op[q] == KT_OP_EXISTS);
      if (positive) ++nd;
      for (const RowRef& rr : rows_of_key.at(kv.first)) {
        bool sat = true;
        for (int32_t q : kv.second) sat &= req_holds_present(s, q, rr.other, rr.val);
        size_t e = ((size_t)rr.row * TPp + sidx) * 2;
        if (!sat) word_table[e] &= ~bit;
        if (positive) word_table[e + 1] |= bit;
      }
    }
    term_unsat[sidx] = 0;
    if (nd > lim.label_slots) { term_unsat[sidx] = 1; nd = 0; }  // needs more keys than a pod row can hold
    need[sidx] = nd;
    max_need = std::max(max_need, nd);
  }
  return max_need;
}

std::string compile_tables(const kt_limits& lim, const SelectorSpec& s, int32_t n_ns, const int64_t* ns_labels, HostTables* out) {
  HostTables h;
  const int32_t M = s.m;
  h.M = M;
  h.W = (M + 31) / 32;
  if (h.W == 0) h.W = 1;
  h.Wp = words_per_row(M);
  int32_t TP = 1;
  for (int32_t t = 0; t < M; ++t) TP = std::max(TP, s.term_off[t + 1] - s.term_off[t]);
  h.TP = TP;
  h.TPpad = TP == 1 ? 1 : (TP + 1) / 2 * 2;

  // ---- row dictionary over the podSelector requirements --------------------------------------
  std::map<uint32_t, int32_t> key_row;                 // key -> "other value" row
  std::map<uint64_t, int32_t>& pair_row = h.pair_row;  // (key<<32|val) -> row
  RowsOfKey& rows_of_key = h.rows_of_key;
  int32_t next_row = 0;
  const int32_t n_terms = s.term_off.empty() ? 0 : s.term_off[M];
  for (int32_t term = 0; term < n_terms; ++term)
    for (int32_t q = s.pod_req_off[term]; q < s.pod_req_off[term + 1]; ++q) {
      uint32_t k = s.req_key[q];
      if (!key_row.count(k)) {
        key_row[k] = next_row;
        rows_of_key[k].push_back(RowRef{next_row, true, 0});
        ++next_row;
      }
      for (int32_t i = s.req_val_off[q]; i < s.req_val_off[q + 1]; ++i) {
        uint64_t pk = ((uint64_t)k << 32) | s.req_vals[i];
        if (!pair_row.count(pk)) {
          pair_row[pk] = next_row;
          rows_of_key[k].push_back(RowRef{next_row, false, s.req_vals[i]});
          ++next_row;
        }
      }
    }
  h.rows = next_row + 1;  // + neutral row
  const int32_t rows = h.rows;
  const int32_t TPp = h.TPpad;

  // ---- sat / pos planes ----------------------------------------------------------------------
  h.table.assign((size_t)h.W * rows * TPp * 2, 0);
  for (size_t i = 0; i < h.table.size(); i += 2) h.table[i] = 0xffffffffu;  // sat = all ones, pos = 0
  std::vector<int32_t> need((size_t)M * TP, 0);
  h.term_unsat.assign((size_t)n_terms, 0);
  int32_t max_need = 0;
  for (int32_t t = 0; t < M; ++t)
    max_need = std::max(max_need, compile_column(lim, s, t, h.rows_of_key, rows, TPp, &h.table[(size_t)(t >> 5) * rows * TPp * 2],
                                                 &need[(size_t)t * TP], h.term_unsat.data() + s.term_off[t]));
  int32_t B = 1;
  while ((1 << B) <= max_need) ++B;
  B = B <= 2 ? 2 : 6;  // the kernels are instantiated for 2 and 6 counter bit-planes (need <= 3 / <= 63)
  h.B = B;
  h.need.assign((size_t)h.W * TPp * B, 0);
  for (int32_t t = 0; t < M; ++t) put_need(t, s.term_off[t + 1] - s.term_off[t], &need[(size_t)t * TP], TPp, B, &h.need[(size_t)(t >> 5) * TPp * B]);

  // ---- namespace masks: which (throttle, term) can apply to pods of namespace ns at all ---------
  int32_t NS = n_ns;
  for (int32_t t = 0; t < M; ++t)
    if (s.kind[t] == KT_KIND_THROTTLE && s.ns_id[t] >= 0) NS = std::max(NS, s.ns_id[t] + 1);
  h.NS = NS;
  h.nsmask.assign((size_t)NS * h.W * TPp, 0);
  // A term whose podSelector does not convert (KT_TERM_POD_INVALID) matches nobody, and MatchesToPod returns its error before it
  // looks at any LATER term -- but only for pods that get as far as that term: every pod of the namespace for a Throttle
  // (throttle_selector.go:30-42), the pods of the namespaces its namespaceSelector matches for a ClusterThrottle
  // (clusterthrottle_selector.go:45-56,71-87).  So the later terms are switched off exactly there: a pod's bit is then
  // "some valid term BEFORE the error matched", which is what the host needs to tell a match from the error.
  std::vector<uint8_t> blocked;
  for (int32_t t = 0; t < M; ++t) {
    bool live = (s.flags[t] & KT_THR_RESPONSIBLE) && !(s.flags[t] & KT_THR_SELECTOR_ERROR);
    if (!live) continue;
    const int32_t w = t >> 5;
    const uint32_t bit = 1u << (t & 31);
    bool any_blocked = false;
    for (int32_t term = s.term_off[t], sidx = 0; term < s.term_off[t + 1]; ++term, ++sidx) {
      if (s.term_flags[term] & KT_TERM_POD_INVALID) {
        if (!any_blocked) blocked.assign((size_t)NS, 0);
        any_blocked = true;
        if (s.kind[t] == KT_KIND_THROTTLE) {
          const int32_t ns = s.ns_id[t];
          if (ns >= 0 && ns < NS) blocked[(size_t)ns] = 1;
        } else {
          for (int32_t ns = 0; ns < n_ns; ++ns)
            if (ns_term_matches(s, term, ns_labels, n_ns, ns, lim.ns_label_slots)) blocked[(size_t)ns] = 1;
        }
        continue;
      }
      if (h.term_unsat[(size_t)term]) continue;
      if (s.kind[t] == KT_KIND_THROTTLE) {
        int32_t ns = s.ns_id[t];
        if (ns >= 0 && ns < NS && !(any_blocked && blocked[(size_t)ns])) h.nsmask[((size_t)ns * h.W + w) * TPp + sidx] |= bit;
      } else {
        for (int32_t ns = 0; ns < n_ns; ++ns)
          if (!(any_blocked && blocked[(size_t)ns]) && ns_term_matches(s, term, ns_labels, n_ns, ns, lim.ns_label_slots))
            h.nsmask[((size_t)ns * h.W + w) * TPp + sidx] |= bit;
      }
    }
  }
  h.nsw_off.assign(NS + 1, 0);
  for (int32_t ns = 0; ns < NS; ++ns) {
    for (int32_t w = 0; w < h.W; ++w) {
      uint32_t any = 0;
      for (int32_t sidx = 0; sidx < TPp; ++sidx) any |= h.nsmask[((size_t)ns * h.W + w) * TPp + sidx];
      if (any) h.nsw_idx.push_back(w);
    }
    h.nsw_off[ns + 1] = (int32_t)h.nsw_idx.size();
    h.max_ns_words = std::max(h.max_ns_words, h.nsw_off[ns + 1] - h.nsw_off[ns]);
  }

  // ---- label -> row hash (open addressing, linear probing, <= 50% load) --------------------------
  size_t entries = key_row.size() + pair_row.size();
  size_t cap = 16;
  while (cap < entries * 2 + 2) cap <<= 1;
  h.hash_mask = (uint32_t)(cap - 1);
  h.hash.assign(cap * 4, 0);
  for (size_t i = 0; i < cap; ++i) h.hash[4 * i] = h.hash[4 * i + 1] = 0xffffffffu;
  auto insert = [&](uint32_t key, uint32_t val, int32_t row) {
    size_t slot = label_hash(key, val) & h.hash_mask;
    while ((h.hash[4 * slot] & h.hash[4 * slot + 1]) != 0xffffffffu) slot = (slot + 1) & h.hash_mask;
    h.hash[4 * slot] = key;
    h.hash[4 * slot + 1] = val;
    h.hash[4 * slot + 2] = (uint32_t)row;
  };
  for (auto& kv : key_row) insert(kv.first, 0xffffffffu, kv.second);
  for (auto& kv : pair_row) insert((uint32_t)(kv.first >> 32), (uint32_t)kv.first, kv.second);

  // ---- two-level direct dictionary ---------------------------------------------------------------
  // key ids small enough -> one keydir entry per id up to the largest mentioned one; per key the mentioned
  // value ids either form a compact range (direct valrow slice) or stay in the hash (off = ~0).
  const uint32_t row_bytes = (uint32_t)TPp * 8u, kOther = 0xfffffffeu;
  const uint32_t neutral_roff = (uint32_t)(rows - 1) * row_bytes;
  h.n_keydir = 0;
  h.valrow.assign(1, kOther);  // [0]: sentinel
  if (!key_row.empty() && key_row.rbegin()->first < kKeyDirMax) h.n_keydir = (int32_t)key_row.rbegin()->first + 1;
  const uint32_t nk = (uint32_t)h.n_keydir;
  h.keydir.assign(((size_t)nk + 1) * 4, 0);
  for (uint32_t k = 0; k <= nk; ++k) h.keydir[4 * (size_t)k] = neutral_roff;  // unmentioned key / sentinel: neutral row, no values
  if (nk > 0) {
    for (auto& kv : key_row) {
      const uint32_t k = kv.first;
      uint32_t vmin = 0xffffffffu, vmax = 0, cnt = 0;
      for (const RowRef& rr : rows_of_key[k])
        if (!rr.other) { vmin = std::min(vmin, rr.val); vmax = std::max(vmax, rr.val); ++cnt; }
      uint32_t* e = &h.keydir[4 * (size_t)k];
      e[0] = (uint32_t)kv.second * row_bytes;
      if (cnt == 0) continue;  // only Exists / DoesNotExist on this key
      const uint64_t span = (uint64_t)vmax - vmin + 1;
      if (span > (uint64_t)cnt * 4 + 64 || h.valrow.size() + span >= (1ull << 31)) { e[3] = 0xffffffffu; continue; }  // sparse value ids: hashed
      e[1] = vmin;
      e[2] = (uint32_t)span;
      e[3] = (uint32_t)h.valrow.size();
      h.valrow.resize(h.valrow.size() + span, kOther);
      for (const RowRef& rr : rows_of_key[k])
        if (!rr.other) h.valrow[e[3] + (rr.val - vmin)] = (uint32_t)rr.row * row_bytes;
    }
  }

  *out = std::move(h);
  return "";
}

bool patch_columns(const kt_limits& lim, const SelectorSpec& old_s, const SelectorSpec& s, const std::vector<int32_t>& listed, HostTables* h) {
  const int32_t M = s.m, TPp = h->TPpad, B = h->B, rows = h->rows;
  if (M < h->M) return false;
  std::vector<char> is_listed((size_t)M, 0);
  for (int32_t t : listed) {  // does every listed column fit the resident tables?
    is_listed[(size_t)t] = 1;
    if (s.term_off[t + 1] - s.term_off[t] > TPp) return false;
    if (s.kind[t] == KT_KIND_THROTTLE && s.ns_id[t] >= h->NS) return false;
    for (int32_t term = s.term_off[t]; term < s.term_off[t + 1]; ++term)
      for (int32_t q = s.pod_req_off[term]; q < s.pod_req_off[term + 1]; ++q) {
        if (!h->rows_of_key.count(s.req_key[q])) return false;
        for (int32_t i = s.req_val_off[q]; i < s.req_val_off[q + 1]; ++i)
          if (!h->pair_row.count(((uint64_t)s.req_key[q] << 32) | s.req_vals[i])) return false;
      }
  }
  for (int32_t t = h->M; t < M; ++t)
    if (!is_listed[(size_t)t]) return false;  // a column the spec grew by must be listed
  if (M > h->M) {  // new words appended as compile_tables starts them (sat = 1, pos = 0, no need); existing words keep their place
    const int32_t W = std::max(1, (M + 31) / 32);
    h->table.resize((size_t)W * rows * TPp * 2, 0);
    for (size_t e = (size_t)h->W * rows * TPp * 2; e < h->table.size(); e += 2) h->table[e] = 0xffffffffu;
    h->need.resize((size_t)W * TPp * B, 0);
    h->M = M;
    h->W = W;
    h->Wp = words_per_row(M);
  }
  // term_unsat follows the new term numbering: the unlisted columns keep theirs
  std::vector<uint8_t> unsat((size_t)s.term_off[M], 0);
  for (int32_t t = 0; t < M; ++t)
    if (!is_listed[(size_t)t])
      std::copy(h->term_unsat.begin() + old_s.term_off[t], h->term_unsat.begin() + old_s.term_off[t + 1], unsat.begin() + s.term_off[t]);
  std::vector<int32_t> need((size_t)TPp);
  for (int32_t t : listed) {
    const uint32_t bit = 1u << (t & 31);
    uint32_t* word_table = &h->table[(size_t)(t >> 5) * rows * TPp * 2];
    uint32_t* word_need = &h->need[(size_t)(t >> 5) * TPp * B];
    for (size_t e = 0; e < (size_t)rows * TPp * 2; e += 2) {  // as compile_tables starts: sat = 1, pos = 0
      word_table[e] |= bit;
      word_table[e + 1] &= ~bit;
    }
    for (size_t e = 0; e < (size_t)TPp * B; ++e) word_need[e] &= ~bit;
    const int32_t nt = s.term_off[t + 1] - s.term_off[t];
    if (compile_column(lim, s, t, h->rows_of_key, rows, TPp, word_table, need.data(), unsat.data() + s.term_off[t]) >= (1 << B)) return false;
    put_need(t, nt, need.data(), TPp, B, word_need);
  }
  h->term_unsat.swap(unsat);
  h->TP = 1;
  for (int32_t t = 0; t < M; ++t) h->TP = std::max(h->TP, s.term_off[t + 1] - s.term_off[t]);
  return true;
}

}  // namespace kt
