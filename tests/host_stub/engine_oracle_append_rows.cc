// The oracle-backed engine test double with the selector column deltas (engine_oracle_selector_rows.cc) plus the column appends
// kt_append_throttle_rows: k columns appended to the recorded spec (kind, ns_id, flags, thresholds, the override CSR and the
// selector CSR laid out again column by column), the status and the reservations held before the call widened by zero columns,
// with the engine's argument and state checks.  It counts its calls (kt_test_append_calls), so that
// tests/test_append_rows_host.py can check which creations took the delta.  Linked with kt_host.cc so that the host layer's
// creation path can be checked against a twin plugin on whole-table uploads and the object-level oracle without a GPU.  Test
// infrastructure only: what it checks is kt_host.cc; the kernels are checked by tests/test_append_rows.py on the GPU.
#include "engine_oracle_selector_rows.cc"

namespace {
int64_t g_append_calls = 0;

// rows x m -> rows x (m + k) with the k new columns zero
template <class T>
void widen(std::vector<T>& v, size_t rows, size_t m, size_t k) {
  std::vector<T> out(rows * (m + k), 0);
  for (size_t r = 0; r < rows; ++r) std::copy(v.begin() + r * m, v.begin() + (r + 1) * m, out.begin() + r * (m + k));
  v.swap(out);
}
}  // namespace

extern "C" {

int kt_append_throttle_rows(kt_ctx* c, int64_t k, const kt_throttle_cols* t, const kt_selector_table* s, int32_t* recompiled) {
  if (!c || k < 0) return KT_ERR_INVALID;
  if (recompiled) *recompiled = 0;
  if (k > 0 && (!t || !t->kind || !t->ns_id || !t->flags || !t->thr || !t->thr_present || !t->thr_cnt || !t->ovr_off || !s || !s->term_off))
    return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: null column");
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_append_throttle_rows before kt_upload_throttles");
  if (k == 0) return KT_OK;
  const int32_t* off = t->ovr_off;
  if (off[0] != 0 || off[k] != t->n_ovr) return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: ovr_off must span [0, n_ovr]");
  for (int64_t i = 0; i < k; ++i)
    if (off[i] > off[i + 1]) return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: ovr_off not monotone");
  if (s->term_off[0] != 0 || s->term_off[k] != s->n_terms) return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: term_off must span [0, n_terms]");
  for (int64_t i = 0; i < k; ++i)
    if (s->term_off[i] > s->term_off[i + 1]) return fail(c, KT_ERR_INVALID, "kt_append_throttle_rows: term_off not monotone");
  ++g_append_calls;
  const size_t M = (size_t)c->m, R = (size_t)c->lim.n_resources, K = (size_t)k, N = (size_t)t->n_ovr, O = (size_t)c->n_ovr;
  // spec and thresholds: the new columns after the held ones
  c->kind.insert(c->kind.end(), t->kind, t->kind + K);
  c->thr_ns.insert(c->thr_ns.end(), t->ns_id, t->ns_id + K);
  c->tflags.insert(c->tflags.end(), t->flags, t->flags + K);
  widen(c->thr, R, M, K);
  for (size_t r = 0; r < R; ++r)
    for (size_t i = 0; i < K; ++i) c->thr[r * (M + K) + M + i] = t->thr[r * K + i];
  c->thr_present.insert(c->thr_present.end(), t->thr_present, t->thr_present + K);
  c->thr_cnt.insert(c->thr_cnt.end(), t->thr_cnt, t->thr_cnt + K);
  // overrides: the new entries after the held ones
  for (size_t i = 0; i < K; ++i) c->ovr_off.push_back((int32_t)(O + (size_t)off[i + 1]));
  c->ovr_begin.insert(c->ovr_begin.end(), t->ovr_begin, t->ovr_begin + N);
  c->ovr_end.insert(c->ovr_end.end(), t->ovr_end, t->ovr_end + N);
  c->ovr_flags.insert(c->ovr_flags.end(), t->ovr_flags, t->ovr_flags + N);
  c->ovr_present.insert(c->ovr_present.end(), t->ovr_present, t->ovr_present + N);
  c->ovr_cnt.insert(c->ovr_cnt.end(), t->ovr_cnt, t->ovr_cnt + N);
  widen(c->ovr_thr, R, O, N);
  for (size_t r = 0; r < R; ++r)
    for (size_t e = 0; e < N; ++e) c->ovr_thr[r * (O + N) + O + e] = t->ovr_thr[r * N + e];
  c->n_ovr = (int32_t)(O + N);
  // the selector CSR: the held terms, then the new ones; all podSelector requirements first
  struct Src {
    const int32_t *pod_req_off, *ns_req_off, *req_val_off;
    const uint8_t* req_op;
    const uint32_t *req_key, *req_vals;
  };
  const Src held{c->pod_req_off.data(), c->ns_req_off.data(), c->req_val_off.data(), c->req_op.data(), c->req_key.data(), c->req_vals.data()};
  const Src mine{s->pod_req_off, s->ns_req_off, s->req_val_off, s->req_op, s->req_key, s->req_vals};
  std::vector<std::pair<const Src*, int32_t>> terms;
  for (int32_t j = 0; j < c->n_terms; ++j) terms.emplace_back(&held, j);
  for (int32_t j = 0; j < s->n_terms; ++j) terms.emplace_back(&mine, j);
  std::vector<int32_t> pod_req_off{0}, ns_req_off, req_val_off{0};
  std::vector<uint8_t> req_op;
  std::vector<uint32_t> req_key, req_vals;
  auto push = [&](const Src& src, int32_t q0, int32_t q1) {
    for (int32_t q = q0; q < q1; ++q) {
      req_key.push_back(src.req_key[q]);
      req_op.push_back(src.req_op[q]);
      for (int32_t v = src.req_val_off[q]; v < src.req_val_off[q + 1]; ++v) req_vals.push_back(src.req_vals[v]);
      req_val_off.push_back((int32_t)req_vals.size());
    }
  };
  for (auto& x : terms) {
    push(*x.first, x.first->pod_req_off[x.second], x.first->pod_req_off[x.second + 1]);
    pod_req_off.push_back((int32_t)req_key.size());
  }
  ns_req_off.push_back((int32_t)req_key.size());
  for (auto& x : terms) {
    push(*x.first, x.first->ns_req_off[x.second], x.first->ns_req_off[x.second + 1]);
    ns_req_off.push_back((int32_t)req_key.size());
  }
  for (size_t i = 0; i < K; ++i) c->term_off.push_back(c->n_terms + s->term_off[i + 1]);
  c->term_flags.insert(c->term_flags.end(), s->term_flags, s->term_flags + s->n_terms);
  c->n_terms += s->n_terms; c->n_reqs = (int32_t)req_key.size(); c->n_vals = (int32_t)req_vals.size();
  c->pod_req_off.swap(pod_req_off); c->ns_req_off.swap(ns_req_off); c->req_val_off.swap(req_val_off); c->req_op.swap(req_op);
  c->req_key.swap(req_key); c->req_vals.swap(req_vals);
  // the status and the reservations held, widened by zero columns
  if (c->have_status) {
    widen(c->st_calculated, 1, M, K); widen(c->st_calc_thr, R, M, K); widen(c->st_calc_present, 1, M, K); widen(c->st_calc_cnt, 1, M, K);
    widen(c->st_used, R, M, K); widen(c->st_used_present, 1, M, K); widen(c->st_used_cnt, 1, M, K); widen(c->st_throttled, 1, M, K);
  }
  if (c->have_reserved) { widen(c->reserved, R, M, K); widen(c->reserved_present, 1, M, K); widen(c->reserved_cnt, 1, M, K); }
  c->m = (int32_t)(M + K);
  c->evaluated = false;
  return KT_OK;
}

// the kt_append_throttle_rows calls that appended columns since the library was loaded
int64_t kt_test_append_calls() { return g_append_calls; }
}
