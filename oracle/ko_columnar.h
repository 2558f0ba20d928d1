// ko_columnar.h -- ORACLE (test infrastructure only).
//
// Columnar CPU restatement: consumes exactly the int64 columns the GPU engine consumes
// (include/kt_b200.h) and recomputes every output with plain nested loops -- no tables, no
// bit tricks -- so that it shares no code or idea with the CUDA path.  It is itself pinned
// against the object-level oracle (ko_model.h) by tests/test_oracle_columnar.py, which builds
// an object World from the same columns (ko_world_from_columns) and compares every output.
//
// Semantics restated (reference file:line):
//   selector term/requirement   v1alpha1/throttle_selector.go:30-54, clusterthrottle_selector.go:30-87
//   row filters                 controllers/throttle_controller.go:213-219, pod_util.go:22-28
//   used = sum over matches     throttle_controller.go:116-119, resource_amount.go:91-110
//   CalculateThreshold          throttle_types.go:65-106, temporary_threshold_override.go:59-72
//   IsThrottled / IsThrottledFor resource_amount.go:127-159, :46-65
//   CheckThrottledFor           throttle_types.go:128-153, clusterthrottle_types.go:30-55
//   admit                       scheduler_plugin/plugin.go:177-180
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

#include "../include/kt_b200.h"

namespace ko {

struct PodCols {
  int64_t n = 0;
  const int64_t* labels = nullptr;   // [L][n]
  const int64_t* req = nullptr;      // [R][n]
  const uint32_t* present = nullptr; // [n]
  const uint32_t* flags = nullptr;   // [n]
  const int32_t* ns_id = nullptr;    // [n]
};

struct ColumnarInput {
  kt_limits lim;
  PodCols running, pending;
  int32_t n_ns = 0;
  const int64_t* ns_labels = nullptr;  // [LN][n_ns]
  int32_t m = 0;
  kt_throttle_cols thr;
  kt_selector_table sel;
  const kt_status_cols* status = nullptr;  // GIVEN_STATUS
  const int64_t* reserved = nullptr;       // [R][m]
  const uint32_t* reserved_present = nullptr;
  const int64_t* reserved_cnt = nullptr;
  int64_t now = 0;
  uint32_t flags = 0;
  int32_t words_per_row = 0;
};

struct ColumnarOutput {
  kt_reconcile_out rec;        // any pointer may be null
  uint32_t* run_bitmap = nullptr;   // [N][W]
  uint32_t* pend_bitmap = nullptr;  // [P][W]
  uint32_t* codes = nullptr;        // [P][2W]
  uint8_t* admit = nullptr;         // [P]
};

namespace col {

// labels.Requirement.Matches on an id-encoded label row (slots hold (key<<32)|val, -1 = empty).
inline bool req_matches(const kt_selector_table& s, int32_t q, const int64_t* labels, int64_t stride, int64_t row, int slots) {
  uint32_t key = s.req_key[q];
  bool has = false;
  uint32_t val = 0;
  for (int i = 0; i < slots; ++i) {
    int64_t l = labels[(int64_t)i * stride + row];
    if (l == KT_LABEL_EMPTY) continue;
    if ((uint32_t)((uint64_t)l >> 32) == key) { has = true; val = (uint32_t)((uint64_t)l & 0xffffffffu); break; }
  }
  auto in_set = [&]() {
    for (int32_t v = s.req_val_off[q]; v < s.req_val_off[q + 1]; ++v)
      if (s.req_vals[v] == val) return true;
    return false;
  };
  switch (s.req_op[q]) {
    case KT_OP_IN: return has && in_set();
    case KT_OP_NOTIN: return !has || !in_set();
    case KT_OP_EXISTS: return has;
    case KT_OP_DOESNOTEXIST: return !has;
  }
  return false;
}

inline bool term_pod_match(const kt_selector_table& s, int32_t term, const PodCols& pods, int64_t p, int L) {
  for (int32_t q = s.pod_req_off[term]; q < s.pod_req_off[term + 1]; ++q)
    if (!req_matches(s, q, pods.labels, pods.n, p, L)) return false;
  return true;
}
inline bool term_ns_match(const ColumnarInput& in, int32_t term, int32_t ns) {
  const kt_selector_table& s = in.sel;
  if (s.term_flags[term] & KT_TERM_NS_INVALID) return false;
  for (int32_t q = s.ns_req_off[term]; q < s.ns_req_off[term + 1]; ++q)
    if (!req_matches(s, q, in.ns_labels, in.n_ns, ns, in.lim.ns_label_slots)) return false;
  return true;
}

// Selector.MatchesToPod for throttle t (either kind); ns = the pod's namespace id.
inline bool throttle_matches(const ColumnarInput& in, int32_t t, const PodCols& pods, int64_t p) {
  int32_t ns = pods.ns_id[p];
  if (in.thr.kind[t] == KT_KIND_THROTTLE) {
    if (ns != in.thr.ns_id[t]) return false;  // namespaced lister (throttle_controller.go:222,249)
  } else {
    if (ns < 0 || ns >= in.n_ns) return false;  // namespace not found => no match on device (host raises)
  }
  for (int32_t term = in.sel.term_off[t]; term < in.sel.term_off[t + 1]; ++term) {
    if (in.thr.kind[t] == KT_KIND_CLUSTERTHROTTLE && !term_ns_match(in, term, ns)) continue;
    // podSelector conversion error: MatchesToPod returns (false, err) here and never looks at the later terms
    // (throttle_selector.go:30-42, clusterthrottle_selector.go:45-56); the error itself is the host's business
    if (in.sel.term_flags[term] & KT_TERM_POD_INVALID) return false;
    if (term_pod_match(in.sel, term, pods, p, in.lim.label_slots)) return true;
  }
  return false;
}

struct Amount {  // a ResourceAmount in column form
  int64_t v[KT_MAX_RESOURCES];
  uint32_t present;  // bit r, KT_COUNT_BIT
  int64_t cnt;
};

// threshold.IsThrottled(used, onEqual) -> mask (bit r / KT_COUNT_BIT)
inline uint32_t is_throttled(const Amount& thr, const Amount& used, bool on_equal, int R) {
  uint32_t m = 0;
  if ((thr.present & KT_COUNT_BIT) && (used.present & KT_COUNT_BIT))
    if (on_equal ? used.cnt >= thr.cnt : used.cnt > thr.cnt) m |= KT_COUNT_BIT;
  for (int r = 0; r < R; ++r) {
    if (!((thr.present >> r) & 1)) continue;
    if (!((used.present >> r) & 1)) continue;
    if (on_equal ? used.v[r] >= thr.v[r] : used.v[r] > thr.v[r]) m |= 1u << r;
  }
  return m;
}
// IsResourceAmountThrottled.IsThrottledFor(pod)
inline bool is_throttled_for(uint32_t mask, uint32_t pod_nonzero) { return (mask & KT_COUNT_BIT) || (mask & pod_nonzero & ~KT_COUNT_BIT); }

inline Amount add(const Amount& a, const Amount& b, int R) {
  Amount o;
  o.present = a.present | b.present;
  o.cnt = ((a.present & KT_COUNT_BIT) ? a.cnt : 0) + ((b.present & KT_COUNT_BIT) ? b.cnt : 0);
  for (int r = 0; r < R; ++r) o.v[r] = (((a.present >> r) & 1) ? a.v[r] : 0) + (((b.present >> r) & 1) ? b.v[r] : 0);
  return o;
}

inline bool live_throttle(const ColumnarInput& in, int32_t t) {
  return (in.thr.flags[t] & KT_THR_RESPONSIBLE) && !(in.thr.flags[t] & KT_THR_SELECTOR_ERROR);
}

// PreFilter's view of throttle t under KT_EVAL_GIVEN_STATUS: the observed status's threshold (the spec's while the status has
// none), used amounts and throttled mask.
inline void given_status_view(const ColumnarInput& in, int32_t t, Amount* threshold, Amount* st_used, uint32_t* st_throttled) {
  const int R = in.lim.n_resources;
  const int32_t M = in.m;
  const kt_status_cols& s = *in.status;
  if (s.calculated[t]) {
    threshold->present = s.calc_present[t];
    threshold->cnt = s.calc_cnt[t];
    for (int r = 0; r < R; ++r) threshold->v[r] = s.calc_thr[(int64_t)r * M + t];
  } else {
    threshold->present = in.thr.thr_present[t];
    threshold->cnt = in.thr.thr_cnt[t];
    for (int r = 0; r < R; ++r) threshold->v[r] = in.thr.thr[(int64_t)r * M + t];
  }
  st_used->present = s.used_present[t];
  st_used->cnt = s.used_cnt[t];
  for (int r = 0; r < R; ++r) st_used->v[r] = s.used[(int64_t)r * M + t];
  *st_throttled = s.throttled[t];
}

// CheckThrottledFor(pod, reserved, onEqual) of pending pod p on throttle t: the 2-bit code.  already = used + reserved.
inline uint32_t check_code(const ColumnarInput& in, int32_t t, const Amount& threshold, const Amount& already, uint32_t st_throttled, int64_t p) {
  const int R = in.lim.n_resources;
  const bool on_equal = in.flags & KT_EVAL_ON_EQUAL;
  const bool e3 = in.thr.kind[t] == KT_KIND_THROTTLE ? true : on_equal;  // Q1
  Amount pod{};
  pod.present = in.pending.present[p] | KT_COUNT_BIT;
  pod.cnt = 1;
  uint32_t nz = 0;
  for (int r = 0; r < R; ++r) {
    pod.v[r] = in.pending.req[(int64_t)r * in.pending.n + p];
    if (((pod.present >> r) & 1) && pod.v[r] != 0) nz |= 1u << r;
  }
  if (is_throttled_for(is_throttled(threshold, pod, false, R), nz)) return KT_CHECK_POD_REQUESTS_EXCEEDS_THRESHOLD;
  if (is_throttled_for(st_throttled, nz)) return KT_CHECK_ACTIVE;
  if (is_throttled_for(is_throttled(threshold, already, e3, R), nz)) return KT_CHECK_ACTIVE;
  const Amount tot = add(already, pod, R);
  return is_throttled_for(is_throttled(threshold, tot, on_equal, R), nz) ? KT_CHECK_INSUFFICIENT : KT_CHECK_NOT_THROTTLED;
}

inline Amount reserved_of(const int64_t* reserved, const uint32_t* present, const int64_t* cnt, int32_t M, int32_t t, int R) {
  Amount res{};
  res.present = present ? present[t] : 0;
  res.cnt = cnt ? cnt[t] : 0;
  for (int r = 0; r < R; ++r) res.v[r] = reserved ? reserved[(int64_t)r * M + t] : 0;
  return res;
}

}  // namespace col

// The whole pass.  Returns 0 or -1 (bad input).
inline int columnar_evaluate(const ColumnarInput& in, const ColumnarOutput& out) {
  using namespace col;
  const int R = in.lim.n_resources;
  const int64_t N = in.running.n, P = in.pending.n;
  const int32_t M = in.m, W = in.words_per_row;
  if (W * 32 < M) return -1;
  const bool given = in.flags & KT_EVAL_GIVEN_STATUS;

  if (out.run_bitmap) std::memset(out.run_bitmap, 0, sizeof(uint32_t) * (size_t)N * W);
  if (out.pend_bitmap) std::memset(out.pend_bitmap, 0, sizeof(uint32_t) * (size_t)P * W);
  if (out.codes) std::memset(out.codes, 0, sizeof(uint32_t) * (size_t)P * 2 * W);
  if (out.admit) std::memset(out.admit, 1, (size_t)P);

  std::vector<Amount> used(M), calc(M);
  std::vector<uint32_t> throttled(M, 0);
  std::vector<uint8_t> ovr_active(M, 0);

  // ---- reconcile half -------------------------------------------------------------------
  for (int32_t t = 0; t < M; ++t) {
    Amount u{};
    u.present = 0; u.cnt = 0;
    for (int r = 0; r < R; ++r) u.v[r] = 0;
    bool live = (in.thr.flags[t] & KT_THR_RESPONSIBLE) && !(in.thr.flags[t] & KT_THR_SELECTOR_ERROR);
    if (live && !(in.flags & KT_EVAL_SKIP_RECONCILE)) {
      for (int64_t p = 0; p < N; ++p) {
        uint32_t f = in.running.flags[p];
        if (!((f & KT_POD_SCHEDULER_MATCH) && (f & KT_POD_SCHEDULED))) continue;  // shouldCountIn
        if (!throttle_matches(in, t, in.running, p)) continue;
        if (out.run_bitmap) out.run_bitmap[(size_t)p * W + (t >> 5)] |= 1u << (t & 31);
        if (!(f & KT_POD_NOT_FINISHED)) continue;
        u.present |= KT_COUNT_BIT;
        u.cnt += 1;
        uint32_t pr = in.running.present[p];
        for (int r = 0; r < R; ++r)
          if ((pr >> r) & 1) { u.present |= 1u << r; u.v[r] += in.running.req[(int64_t)r * N + p]; }
      }
    }
    used[t] = u;

    // CalculateThreshold(now): merged active overrides REPLACE the spec threshold (Q7)
    Amount c{};
    c.present = in.thr.thr_present[t];
    c.cnt = in.thr.thr_cnt[t];
    for (int r = 0; r < R; ++r) c.v[r] = in.thr.thr[(int64_t)r * M + t];
    bool active_found = false;
    Amount o{};
    o.present = 0; o.cnt = 0;
    for (int r = 0; r < R; ++r) o.v[r] = 0;
    for (int32_t i = in.thr.ovr_off[t]; i < in.thr.ovr_off[t + 1]; ++i) {
      if (in.thr.ovr_flags[i] & KT_OVR_PARSE_ERROR) continue;
      bool act = in.thr.ovr_begin[i] <= in.now && in.now <= in.thr.ovr_end[i];
      if (!act) continue;
      active_found = true;
      uint32_t op = in.thr.ovr_present[i];
      if (!(o.present & KT_COUNT_BIT) && (op & KT_COUNT_BIT)) { o.present |= KT_COUNT_BIT; o.cnt = in.thr.ovr_cnt[i]; }
      for (int r = 0; r < R; ++r)
        if (((op >> r) & 1) && !((o.present >> r) & 1)) { o.present |= 1u << r; o.v[r] = in.thr.ovr_thr[(int64_t)r * in.thr.n_ovr + i]; }
    }
    if (active_found) c = o;
    calc[t] = c;
    ovr_active[t] = active_found;
    throttled[t] = live ? is_throttled(c, u, true, R) : 0;  // reconcile uses onEqual=true (throttle_controller.go:133)

    if (out.rec.used) for (int r = 0; r < R; ++r) out.rec.used[(int64_t)r * M + t] = u.v[r];
    if (out.rec.used_present) out.rec.used_present[t] = u.present;
    if (out.rec.used_cnt) out.rec.used_cnt[t] = u.cnt;
    if (out.rec.throttled) out.rec.throttled[t] = throttled[t];
    if (out.rec.calc_thr) for (int r = 0; r < R; ++r) out.rec.calc_thr[(int64_t)r * M + t] = c.v[r];
    if (out.rec.calc_present) out.rec.calc_present[t] = c.present;
    if (out.rec.calc_cnt) out.rec.calc_cnt[t] = c.cnt;
    if (out.rec.override_active) out.rec.override_active[t] = active_found;
  }
  if (in.flags & KT_EVAL_SKIP_CHECK) return 0;

  // ---- check half -----------------------------------------------------------------------
  for (int32_t t = 0; t < M; ++t) {
    if (!live_throttle(in, t)) continue;
    // which status does PreFilter see?
    Amount threshold, st_used;
    uint32_t st_throttled;
    if (given) {
      given_status_view(in, t, &threshold, &st_used, &st_throttled);
    } else {
      threshold = calc[t];
      st_used = used[t];
      st_throttled = throttled[t];
    }
    const Amount already = add(st_used, reserved_of(in.reserved, in.reserved_present, in.reserved_cnt, M, t, R), R);

    for (int64_t p = 0; p < P; ++p) {
      if (!throttle_matches(in, t, in.pending, p)) continue;
      if (out.pend_bitmap) out.pend_bitmap[(size_t)p * W + (t >> 5)] |= 1u << (t & 31);
      const uint32_t code = check_code(in, t, threshold, already, st_throttled, p);
      if (out.codes) out.codes[(size_t)p * 2 * W + (t >> 4)] |= code << (2 * (t & 15));
      if (code != KT_CHECK_NOT_THROTTLED && out.admit) out.admit[p] = 0;
    }
  }
  return 0;
}

// Queue-ordered greedy admission, one pod per cycle (scheduler_plugin/plugin.go:148-238): the pending rows
// [first, first + count) in row order, each checked (PreFilter) against the observed status + the reservations so far; on
// Success its ResourceAmountOfPod -- every present request, zero or not, and Counts{Pod: 1} -- joins the reservation of
// every throttle it affects (Reserve, reserved_resource_amounts.go:66-136).  Rows outside the queue keep the codes of one
// KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE pass.  in.status is required; in.flags contributes KT_EVAL_ON_EQUAL only.
// res / res_present / res_cnt ([R][m], [m], [m]) receive the final reservations.  O(P x m) for the one pass, then
// O(count x m).  Returns the admitted count, or -1 (bad input).
inline int64_t columnar_admit_queue(const ColumnarInput& in_, int64_t first, int64_t count, const ColumnarOutput& out_, int64_t* res,
                                    uint32_t* res_present, int64_t* res_cnt) {
  using namespace col;
  const int R = in_.lim.n_resources;
  const int64_t P = in_.pending.n;
  const int32_t M = in_.m, W = in_.words_per_row;
  if (!in_.status || first < 0 || count < 0 || first + count > P || W * 32 < M) return -1;
  ColumnarInput in = in_;
  in.flags = KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE | (in_.flags & KT_EVAL_ON_EQUAL);
  for (int32_t t = 0; t < M; ++t) {
    const Amount a = reserved_of(in_.reserved, in_.reserved_present, in_.reserved_cnt, M, t, R);
    for (int r = 0; r < R; ++r) res[(int64_t)r * M + t] = a.v[r];
    res_present[t] = a.present;
    res_cnt[t] = a.cnt;
  }
  std::vector<uint32_t> bitmap((size_t)P * W + 1, 0);
  ColumnarOutput out = out_;
  out.pend_bitmap = bitmap.data();
  if (columnar_evaluate(in, out) != 0) return -1;
  if (out_.pend_bitmap) std::memcpy(out_.pend_bitmap, bitmap.data(), sizeof(uint32_t) * (size_t)P * W);

  std::vector<Amount> threshold(M), st_used(M);
  std::vector<uint32_t> st_throttled(M, 0);
  for (int32_t t = 0; t < M; ++t)
    if (live_throttle(in, t)) given_status_view(in, t, &threshold[t], &st_used[t], &st_throttled[t]);
  const uint32_t rmask = R >= 32 ? 0xffffffffu : ((1u << R) - 1u);
  int64_t admitted = 0;
  for (int64_t p = first; p < first + count; ++p) {
    const uint32_t* row = &bitmap[(size_t)p * W];
    bool ok = true;
    if (out.codes) std::memset(&out.codes[(size_t)p * 2 * W], 0, sizeof(uint32_t) * 2 * W);
    for (int32_t t = 0; t < M; ++t) {
      if (!((row[t >> 5] >> (t & 31)) & 1)) continue;  // the pass sets bits of live throttles only
      const Amount already = add(st_used[t], reserved_of(res, res_present, res_cnt, M, t, R), R);
      const uint32_t code = check_code(in, t, threshold[t], already, st_throttled[t], p);
      if (out.codes) out.codes[(size_t)p * 2 * W + (t >> 4)] |= code << (2 * (t & 15));
      if (code != KT_CHECK_NOT_THROTTLED) ok = false;
    }
    if (out.admit) out.admit[p] = ok;
    if (!ok) continue;
    ++admitted;
    const uint32_t pres = in.pending.present[p] & rmask;
    for (int32_t t = 0; t < M; ++t) {
      if (!((row[t >> 5] >> (t & 31)) & 1)) continue;
      for (int r = 0; r < R; ++r)
        if ((pres >> r) & 1) res[(int64_t)r * M + t] += in.pending.req[(int64_t)r * P + p];
      res_present[t] |= pres | KT_COUNT_BIT;
      res_cnt[t] += 1;
    }
  }
  return admitted;
}

}  // namespace ko
