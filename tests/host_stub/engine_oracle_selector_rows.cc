// The oracle-backed engine test double with the threshold column deltas (engine_oracle_threshold_rows.cc) plus the selector
// column deltas kt_update_selector_rows: kind, ns_id, flags and the selector terms of the listed columns replaced in the recorded
// spec (the CSR laid out again column by column), with the engine's argument and state checks.  It counts its calls
// (kt_test_selector_calls), so that tests/test_selector_rows_host.py can check which deletions and selector edits took the delta.
// Linked with kt_host.cc so that the host layer's delta path can be checked against a twin plugin on whole-table uploads and the
// object-level oracle without a GPU.  Test infrastructure only: what it checks is kt_host.cc; the kernels are checked by
// tests/test_selector_rows.py on the GPU.
#include "engine_oracle_threshold_rows.cc"

namespace {
int64_t g_selector_calls = 0;
}

extern "C" {

int kt_update_selector_rows(kt_ctx* c, int64_t k, const int32_t* idx, const kt_throttle_cols* t, const kt_selector_table* s,
                            int32_t* recompiled) {
  if (!c || k < 0) return KT_ERR_INVALID;
  if (recompiled) *recompiled = 0;
  if (k > 0 && (!idx || !t || !t->kind || !t->ns_id || !t->flags || !s || !s->term_off))
    return fail(c, KT_ERR_INVALID, "kt_update_selector_rows: null column");
  if (t && (t->thr || t->thr_present || t->thr_cnt || t->ovr_off || t->ovr_begin || t->ovr_end || t->ovr_flags || t->ovr_thr ||
            t->ovr_present || t->ovr_cnt))
    return fail(c, KT_ERR_INVALID, "kt_update_selector_rows: threshold and override columns must be null");
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_update_selector_rows before kt_upload_throttles");
  if (k == 0) return KT_OK;
  if (int rc = check_columns(c, k, idx)) return rc;
  if (s->term_off[0] != 0 || s->term_off[k] != s->n_terms) return fail(c, KT_ERR_INVALID, "kt_update_selector_rows: term_off must span [0, n_terms]");
  for (int64_t i = 0; i < k; ++i)
    if (s->term_off[i] > s->term_off[i + 1]) return fail(c, KT_ERR_INVALID, "kt_update_selector_rows: term_off not monotone");
  ++g_selector_calls;
  const size_t M = (size_t)c->m;
  std::vector<int64_t> from(M, -1);
  for (int64_t i = 0; i < k; ++i) {
    from[(size_t)idx[i]] = i;
    c->kind[(size_t)idx[i]] = t->kind[i];
    c->thr_ns[(size_t)idx[i]] = t->ns_id[i];
    c->tflags[(size_t)idx[i]] = t->flags[i];
  }
  // the CSR, column by column: the listed columns from the call, the others as they were; all podSelector requirements first
  struct Src {
    const int32_t *term_off, *pod_req_off, *ns_req_off, *req_val_off;
    const uint8_t *term_flags, *req_op;
    const uint32_t *req_key, *req_vals;
  };
  const Src mine{s->term_off, s->pod_req_off, s->ns_req_off, s->req_val_off, s->term_flags, s->req_op, s->req_key, s->req_vals};
  const Src held{c->term_off.data(), c->pod_req_off.data(), c->ns_req_off.data(), c->req_val_off.data(), c->term_flags.data(),
                 c->req_op.data(), c->req_key.data(), c->req_vals.data()};
  std::vector<std::pair<const Src*, int32_t>> terms;
  std::vector<int32_t> term_off{0}, pod_req_off{0}, ns_req_off, req_val_off{0};
  std::vector<uint8_t> term_flags, req_op;
  std::vector<uint32_t> req_key, req_vals;
  for (size_t col = 0; col < M; ++col) {
    const Src& src = from[col] >= 0 ? mine : held;
    const size_t at = from[col] >= 0 ? (size_t)from[col] : col;
    for (int32_t term = src.term_off[at]; term < src.term_off[at + 1]; ++term) {
      terms.emplace_back(&src, term);
      term_flags.push_back(src.term_flags[term]);
    }
    term_off.push_back((int32_t)terms.size());
  }
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
  c->n_terms = (int32_t)term_flags.size(); c->n_reqs = (int32_t)req_key.size(); c->n_vals = (int32_t)req_vals.size();
  c->term_off.swap(term_off); c->pod_req_off.swap(pod_req_off); c->ns_req_off.swap(ns_req_off); c->req_val_off.swap(req_val_off);
  c->term_flags.swap(term_flags); c->req_op.swap(req_op); c->req_key.swap(req_key); c->req_vals.swap(req_vals);
  c->evaluated = false;
  return KT_OK;
}

// the kt_update_selector_rows calls that changed columns since the library was loaded
int64_t kt_test_selector_calls() { return g_selector_calls; }
}
