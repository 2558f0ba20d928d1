// The oracle-backed engine test double with the throttle-side column deltas (engine_oracle_throttle_rows.cc) plus the namespace
// row deltas kt_update_namespace_rows: the listed rows replaced in the recorded namespace rows (the count grown, the rows it grows
// by label-less), with the engine's argument checks.  It counts the calls that move namespace and throttle state to the device
// (kt_test_namespace_calls), so that tests/test_namespace_rows_host.py can check what a Namespace event costs.  Linked with
// kt_host.cc so that the host layer's row path can be checked against a twin plugin on whole-table uploads and the object-level
// oracle without a GPU.  Test infrastructure only: what it checks is kt_host.cc; the kernels are checked by
// tests/test_namespace_rows.py on the GPU.
#define kt_upload_namespaces kt_upload_namespaces_uncounted
#include "engine_oracle_throttle_rows.cc"
#undef kt_upload_namespaces

namespace {
int64_t g_ns_calls[2] = {};  // kt_upload_namespaces, kt_update_namespace_rows
}

extern "C" {

int kt_upload_namespaces(kt_ctx* c, int32_t n_ns, const int64_t* labels) {
  ++g_ns_calls[0];
  return kt_upload_namespaces_uncounted(c, n_ns, labels);
}

int kt_update_namespace_rows(kt_ctx* c, int32_t n_ns, int64_t k, const int32_t* idx, const int64_t* labels) {
  if (!c || k < 0) return KT_ERR_INVALID;
  const size_t LN = (size_t)c->lim.ns_label_slots;
  if (k > 0 && (!idx || (LN > 0 && !labels))) return fail(c, KT_ERR_INVALID, "kt_update_namespace_rows: null column");
  if (n_ns < c->n_ns) return fail(c, KT_ERR_INVALID, "kt_update_namespace_rows: n_ns shrinks");
  std::vector<int32_t> s(idx, idx + k);
  std::sort(s.begin(), s.end());
  if (k > 0 && (s.front() < 0 || s.back() >= n_ns)) return fail(c, KT_ERR_INVALID, "kt_update_namespace_rows: namespace out of range");
  if (std::adjacent_find(s.begin(), s.end()) != s.end()) return fail(c, KT_ERR_INVALID, "kt_update_namespace_rows: namespace listed twice");
  if (k == 0 && n_ns == c->n_ns) return KT_OK;
  ++g_ns_calls[1];
  const size_t old_n = (size_t)c->n_ns, N = (size_t)n_ns, K = (size_t)k;
  std::vector<int64_t> rows(LN * N, KT_LABEL_EMPTY);
  for (size_t l = 0; l < LN; ++l)
    for (size_t i = 0; i < old_n; ++i) rows[l * N + i] = c->ns_labels[l * old_n + i];
  for (size_t i = 0; i < K; ++i)
    for (size_t l = 0; l < LN; ++l) rows[l * N + (size_t)idx[i]] = labels[l * K + i];
  c->ns_labels.swap(rows);
  c->n_ns = n_ns;
  c->evaluated = false;
  return KT_OK;
}

// the calls since the library was loaded: kt_upload_namespaces, kt_update_namespace_rows
void kt_test_namespace_calls(int64_t* out) {
  for (int i = 0; i < 2; ++i) out[i] = g_ns_calls[i];
}
}
