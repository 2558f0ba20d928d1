// The oracle-backed engine test double with the throttle-side column deltas (engine_oracle_throttle_rows.cc) plus the threshold
// column deltas kt_update_threshold_rows: spec.threshold and the override CSR of the listed columns replaced in the recorded spec
// columns (the CSR rebuilt when a count changes), with the engine's argument and state checks.  It counts its calls
// (kt_test_threshold_calls), so that tests/test_threshold_rows_host.py can check what a threshold or override edit costs.  Linked
// with kt_host.cc so that the host layer's delta path can be checked against a twin plugin on whole-table uploads and the
// object-level oracle without a GPU.  Test infrastructure only: what it checks is kt_host.cc; the kernels are checked by
// tests/test_threshold_rows.py on the GPU.
#include "engine_oracle_throttle_rows.cc"

namespace {
int64_t g_threshold_calls = 0;
}

extern "C" {

int kt_update_threshold_rows(kt_ctx* c, int64_t k, const int32_t* idx, const kt_throttle_cols* t) {
  if (!c || k < 0) return KT_ERR_INVALID;
  if (k > 0 && (!idx || !t || !t->thr || !t->thr_present || !t->thr_cnt || !t->ovr_off))
    return fail(c, KT_ERR_INVALID, "kt_update_threshold_rows: null column");
  if (t && (t->kind || t->ns_id || t->flags)) return fail(c, KT_ERR_INVALID, "kt_update_threshold_rows: kind, ns_id and flags must be null");
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_update_threshold_rows before kt_upload_throttles");
  if (k == 0) return KT_OK;
  if (int rc = check_columns(c, k, idx)) return rc;
  const int32_t* off = t->ovr_off;
  if (off[0] != 0 || off[k] != t->n_ovr) return fail(c, KT_ERR_INVALID, "kt_update_threshold_rows: ovr_off must span [0, n_ovr]");
  for (int64_t i = 0; i < k; ++i)
    if (off[i] > off[i + 1]) return fail(c, KT_ERR_INVALID, "kt_update_threshold_rows: ovr_off not monotone");
  if (t->n_ovr > 0 && (!t->ovr_begin || !t->ovr_end || !t->ovr_flags || !t->ovr_thr || !t->ovr_present || !t->ovr_cnt))
    return fail(c, KT_ERR_INVALID, "kt_update_threshold_rows: null override columns");
  ++g_threshold_calls;
  const size_t M = (size_t)c->m, R = (size_t)c->lim.n_resources, K = (size_t)k, N = (size_t)t->n_ovr, O = (size_t)c->n_ovr;
  std::vector<int64_t> listed(M, -1);
  for (size_t i = 0; i < K; ++i) {
    const size_t col = (size_t)idx[i];
    listed[col] = (int64_t)i;
    for (size_t r = 0; r < R; ++r) c->thr[r * M + col] = t->thr[r * K + i];
    c->thr_present[col] = t->thr_present[i];
    c->thr_cnt[col] = t->thr_cnt[i];
  }
  // the override CSR, column by column: the listed columns from the call, the others as they were
  std::vector<int32_t> ovr_off{0};
  std::vector<int64_t> begin, end, cnt, vals;  // vals: R per entry
  std::vector<uint8_t> flags;
  std::vector<uint32_t> present;
  for (size_t col = 0; col < M; ++col) {
    const bool mine = listed[col] >= 0;
    const size_t e0 = mine ? (size_t)off[listed[col]] : (size_t)c->ovr_off[col], e1 = mine ? (size_t)off[listed[col] + 1] : (size_t)c->ovr_off[col + 1];
    for (size_t e = e0; e < e1; ++e) {
      begin.push_back(mine ? t->ovr_begin[e] : c->ovr_begin[e]);
      end.push_back(mine ? t->ovr_end[e] : c->ovr_end[e]);
      flags.push_back(mine ? t->ovr_flags[e] : c->ovr_flags[e]);
      present.push_back(mine ? t->ovr_present[e] : c->ovr_present[e]);
      cnt.push_back(mine ? t->ovr_cnt[e] : c->ovr_cnt[e]);
      for (size_t r = 0; r < R; ++r) vals.push_back(mine ? t->ovr_thr[r * N + e] : c->ovr_thr[r * O + e]);
    }
    ovr_off.push_back((int32_t)begin.size());
  }
  const size_t n = begin.size();
  c->ovr_thr.assign(R * n, 0);
  for (size_t e = 0; e < n; ++e)
    for (size_t r = 0; r < R; ++r) c->ovr_thr[r * n + e] = vals[e * R + r];
  c->ovr_off.swap(ovr_off); c->ovr_begin.swap(begin); c->ovr_end.swap(end); c->ovr_flags.swap(flags); c->ovr_present.swap(present);
  c->ovr_cnt.swap(cnt);
  c->n_ovr = (int32_t)n;
  c->evaluated = false;
  return KT_OK;
}

// the kt_update_threshold_rows calls that changed columns since the library was loaded
int64_t kt_test_threshold_calls() { return g_threshold_calls; }
}
