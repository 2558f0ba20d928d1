// The oracle-backed engine test double with the column appends (engine_oracle_append_rows.cc) plus the column moves
// kt_move_throttle_columns: column j of the recorded spec, thresholds, overrides, status and reservations taken from previous
// column src[j], or an empty column for -1 (ClusterThrottle, ns_id -1, flags 0, no terms, zero status, nothing reserved), with the
// engine's argument and state checks.  It counts its calls (kt_test_move_calls), so that tests/test_move_columns_host.py can
// check which creations and deletions took the move.  Test infrastructure only: what it checks is kt_host.cc; the kernels are
// checked by tests/test_move_columns.py on the GPU.
#include "engine_oracle_append_rows.cc"

namespace {
int64_t g_move_calls = 0;

// rows x m_old -> rows x m with column j from src[j] (zero for -1)
template <class T>
void gather(std::vector<T>& v, size_t rows, size_t m_old, const int32_t* src, size_t m) {
  std::vector<T> out(rows * m, 0);
  for (size_t r = 0; r < rows; ++r)
    for (size_t j = 0; j < m; ++j)
      if (src[j] >= 0) out[r * m + j] = v[r * m_old + (size_t)src[j]];
  v.swap(out);
}
}  // namespace

extern "C" {

int kt_move_throttle_columns(kt_ctx* c, int32_t m, const int32_t* src) {
  if (!c || m < 0 || (m > 0 && !src)) return c ? fail(c, KT_ERR_INVALID, "kt_move_throttle_columns: bad m or null src") : KT_ERR_INVALID;
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_move_throttle_columns before kt_upload_throttles");
  const size_t M = (size_t)c->m, R = (size_t)c->lim.n_resources, K = (size_t)m;
  std::vector<char> named(M, 0);
  for (size_t j = 0; j < K; ++j) {
    if (src[j] < -1 || src[j] >= (int32_t)M) return fail(c, KT_ERR_INVALID, "kt_move_throttle_columns: entry out of range");
    if (src[j] >= 0 && named[(size_t)src[j]]++) return fail(c, KT_ERR_INVALID, "kt_move_throttle_columns: column listed twice");
  }
  ++g_move_calls;
  std::vector<uint8_t> kind(K, KT_KIND_CLUSTERTHROTTLE), tflags(K, 0);
  std::vector<int32_t> thr_ns(K, -1);
  for (size_t j = 0; j < K; ++j)
    if (src[j] >= 0) { kind[j] = c->kind[(size_t)src[j]]; tflags[j] = c->tflags[(size_t)src[j]]; thr_ns[j] = c->thr_ns[(size_t)src[j]]; }
  c->kind.swap(kind); c->tflags.swap(tflags); c->thr_ns.swap(thr_ns);
  gather(c->thr, R, M, src, K); gather(c->thr_present, 1, M, src, K); gather(c->thr_cnt, 1, M, src, K);
  // overrides: each column's entries in the new column order
  std::vector<int32_t> ovr_off{0};
  std::vector<int64_t> ob, oe, oc;
  std::vector<uint8_t> of;
  std::vector<uint32_t> op;
  std::vector<size_t> entries;
  for (size_t j = 0; j < K; ++j) {
    if (src[j] >= 0)
      for (int32_t e = c->ovr_off[(size_t)src[j]]; e < c->ovr_off[(size_t)src[j] + 1]; ++e) {
        entries.push_back((size_t)e);
        ob.push_back(c->ovr_begin[(size_t)e]); oe.push_back(c->ovr_end[(size_t)e]); of.push_back(c->ovr_flags[(size_t)e]);
        op.push_back(c->ovr_present[(size_t)e]); oc.push_back(c->ovr_cnt[(size_t)e]);
      }
    ovr_off.push_back((int32_t)entries.size());
  }
  const size_t O = (size_t)c->n_ovr, N = entries.size();
  std::vector<int64_t> othr(R * N, 0);
  for (size_t r = 0; r < R; ++r)
    for (size_t i = 0; i < N; ++i) othr[r * N + i] = c->ovr_thr[r * O + entries[i]];
  c->ovr_off.swap(ovr_off); c->ovr_begin.swap(ob); c->ovr_end.swap(oe); c->ovr_flags.swap(of); c->ovr_present.swap(op);
  c->ovr_cnt.swap(oc); c->ovr_thr.swap(othr);
  c->n_ovr = (int32_t)N;
  // the selector CSR laid out again column by column: all podSelector requirements first
  std::vector<int32_t> terms, term_off{0}, pod_req_off{0}, ns_req_off, req_val_off{0};
  std::vector<uint8_t> term_flags, req_op;
  std::vector<uint32_t> req_key, req_vals;
  for (size_t j = 0; j < K; ++j) {
    if (src[j] >= 0)
      for (int32_t t = c->term_off[(size_t)src[j]]; t < c->term_off[(size_t)src[j] + 1]; ++t) {
        terms.push_back(t);
        term_flags.push_back(c->term_flags[(size_t)t]);
      }
    term_off.push_back((int32_t)terms.size());
  }
  auto push = [&](int32_t q0, int32_t q1) {
    for (int32_t q = q0; q < q1; ++q) {
      req_key.push_back(c->req_key[(size_t)q]);
      req_op.push_back(c->req_op[(size_t)q]);
      for (int32_t v = c->req_val_off[(size_t)q]; v < c->req_val_off[(size_t)q + 1]; ++v) req_vals.push_back(c->req_vals[(size_t)v]);
      req_val_off.push_back((int32_t)req_vals.size());
    }
  };
  for (int32_t t : terms) {
    push(c->pod_req_off[(size_t)t], c->pod_req_off[(size_t)t + 1]);
    pod_req_off.push_back((int32_t)req_key.size());
  }
  ns_req_off.push_back((int32_t)req_key.size());
  for (int32_t t : terms) {
    push(c->ns_req_off[(size_t)t], c->ns_req_off[(size_t)t + 1]);
    ns_req_off.push_back((int32_t)req_key.size());
  }
  c->term_off.swap(term_off); c->term_flags.swap(term_flags); c->pod_req_off.swap(pod_req_off); c->ns_req_off.swap(ns_req_off);
  c->req_val_off.swap(req_val_off); c->req_op.swap(req_op); c->req_key.swap(req_key); c->req_vals.swap(req_vals);
  c->n_terms = (int32_t)c->term_flags.size(); c->n_reqs = (int32_t)c->req_key.size(); c->n_vals = (int32_t)c->req_vals.size();
  // the status and the reservations held, gathered the same way
  if (c->have_status) {
    gather(c->st_calculated, 1, M, src, K); gather(c->st_calc_thr, R, M, src, K); gather(c->st_calc_present, 1, M, src, K);
    gather(c->st_calc_cnt, 1, M, src, K); gather(c->st_used, R, M, src, K); gather(c->st_used_present, 1, M, src, K);
    gather(c->st_used_cnt, 1, M, src, K); gather(c->st_throttled, 1, M, src, K);
  }
  if (c->have_reserved) { gather(c->reserved, R, M, src, K); gather(c->reserved_present, 1, M, src, K); gather(c->reserved_cnt, 1, M, src, K); }
  c->m = m;
  c->evaluated = false;
  return KT_OK;
}

// the kt_move_throttle_columns calls since the library was loaded
int64_t kt_test_move_calls() { return g_move_calls; }
}
