// The oracle-backed engine test double (engine_oracle.cc, with kt_check_pending_rows of engine_oracle_check_rows.cc) plus
// kt_check_pods: PreFilter of pods given by value, computed by the columnar oracle on a private copy of the recorded tables,
// status and reservations whose pending table holds just those pods (a GIVEN_STATUS | SKIP_RECONCILE pass; nothing of the
// context changes).  It counts its kt_check_pods and kt_evaluate calls and the uploads of pending rows
// (kt_test_check_pods_calls), so that tests/test_check_pods_host.py can check what a manifest PreFilter or Reserve costs on the
// device.  Linked with kt_host.cc so that the host layer's kt_check_pods path can be checked against the same host layer on
// engine_oracle_check_rows.cc (which lacks the call, so it keeps the scratch-row pass) and the object-level oracle without a
// GPU.  Test infrastructure only: what it checks is kt_host.cc; the kernel is checked by tests/test_check_pods.py on the GPU.
#define kt_evaluate kt_evaluate_uncounted
#define kt_upload_pods kt_upload_pods_uncounted
#define kt_update_pod_rows kt_update_pod_rows_uncounted
#include "engine_oracle_check_rows.cc"
#undef kt_evaluate
#undef kt_upload_pods
#undef kt_update_pod_rows

namespace {
int64_t g_calls[3] = {};  // kt_check_pods, kt_evaluate, pending-row uploads (kt_upload_pods / kt_update_pod_rows of KT_PODS_PENDING)
}

extern "C" {

int kt_evaluate(kt_ctx* c, int64_t now, uint32_t flags) {
  ++g_calls[1];
  return kt_evaluate_uncounted(c, now, flags);
}
int kt_upload_pods(kt_ctx* c, int kind, int64_t n, const int64_t* labels, const int64_t* req, const uint32_t* present, const uint32_t* flags, const int32_t* ns) {
  if (kind == KT_PODS_PENDING) ++g_calls[2];
  return kt_upload_pods_uncounted(c, kind, n, labels, req, present, flags, ns);
}
int kt_update_pod_rows(kt_ctx* c, int kind, int64_t k, const int64_t* rows, const int64_t* labels, const int64_t* req, const uint32_t* present,
                       const uint32_t* flags, const int32_t* ns) {
  if (kind == KT_PODS_PENDING) ++g_calls[2];
  return kt_update_pod_rows_uncounted(c, kind, k, rows, labels, req, present, flags, ns);
}

int kt_check_pods(kt_ctx* c, uint32_t flags, int64_t k, const int64_t* labels, const int64_t* req, const uint32_t* present, const int32_t* ns_id,
                  uint32_t* words, uint32_t* codes, uint8_t* admit) {
  if (!c || k < 0) return KT_ERR_INVALID;
  if (k > 0 && (!labels || !req || !present || !ns_id)) return fail(c, KT_ERR_INVALID, "kt_check_pods: null input column");
  if (flags & ~KT_EVAL_ON_EQUAL) return fail(c, KT_ERR_INVALID, "kt_check_pods: flags must be 0 or KT_EVAL_ON_EQUAL");
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_check_pods before kt_upload_throttles");
  if (!c->have_status) return fail(c, KT_ERR_STATE, "kt_check_pods without kt_upload_status");
  ++g_calls[0];
  if (k == 0) return KT_OK;
  const size_t L = (size_t)c->lim.label_slots, R = (size_t)c->lim.n_resources, K = (size_t)k;
  kt_ctx t = *c;
  Pods& p = t.pods[KT_PODS_PENDING];
  p.n = k;
  p.labels.assign(labels, labels + L * K);
  p.req.assign(req, req + R * K);
  p.present.assign(present, present + K);
  p.flags.assign(K, 0);  // the pass reads no flags of a pending row
  p.ns.assign(ns_id, ns_id + K);
  t.pods[KT_PODS_RUNNING] = Pods();
  const int rc = evaluate(&t, 0, KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE | flags, nullptr);
  if (rc != KT_OK) return fail(c, rc, t.err.c_str());
  const size_t Wp = (size_t)t.words();
  if (words) std::memcpy(words, t.pend_bitmap.data(), K * Wp * 4);
  if (codes) std::memcpy(codes, t.codes.data(), K * 2 * Wp * 4);
  if (admit) std::memcpy(admit, t.admit.data(), K);
  return KT_OK;
}

// {kt_check_pods calls, kt_evaluate calls, pending-row uploads} since the library was loaded
void kt_test_check_pods_calls(int64_t* out) {
  for (int i = 0; i < 3; ++i) out[i] = g_calls[i];
}
}
