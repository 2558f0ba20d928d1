// The oracle-backed engine test double (engine_oracle.cc, with kt_reconcile_throttles of engine_oracle_reconcile.cc and
// kt_get_match_columns as in engine_oracle_columns.cc) plus kt_match_pods: the affected throttles of pods given by value,
// computed by the columnar oracle on a private copy of the recorded tables whose pending table holds just those pods (a
// GIVEN_STATUS | SKIP_RECONCILE pass; nothing of the context changes).  It counts its kt_match_pods and kt_evaluate calls
// (kt_test_device_calls), so that tests/test_apply_events.py can check what a batch of informer events costs on the device.
// Linked with kt_host.cc so that kth_apply_events can be checked against kth_apply / kth_delete and the object-level oracle
// without a GPU.  Test infrastructure only: what it checks is kt_host.cc; the kernel is checked by tests/test_match_pods.py.
#define kt_evaluate kt_evaluate_uncounted
#include "engine_oracle_reconcile.cc"
#undef kt_evaluate

namespace {
int64_t g_match_calls = 0, g_evaluate_calls = 0;
}

extern "C" {

int kt_evaluate(kt_ctx* c, int64_t now, uint32_t flags) {
  ++g_evaluate_calls;
  return kt_evaluate_uncounted(c, now, flags);
}

int kt_match_pods(kt_ctx* c, int64_t k, const int64_t* labels, const int32_t* ns_id, uint32_t* words) {
  if (!c || k < 0) return KT_ERR_INVALID;
  const size_t L = (size_t)c->lim.label_slots, K = (size_t)k;
  if (k > 0 && (!labels || !ns_id || !words)) return fail(c, KT_ERR_INVALID, "kt_match_pods: null pointer");
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_match_pods before kt_upload_throttles");
  ++g_match_calls;
  if (k == 0) return KT_OK;
  kt_ctx t = *c;
  Pods& p = t.pods[KT_PODS_PENDING];
  p.n = k;
  p.labels.assign(labels, labels + L * K);
  p.req.assign((size_t)c->lim.n_resources * K, 0);
  p.present.assign(K, 0);
  p.flags.assign(K, KT_POD_SCHEDULER_MATCH | KT_POD_NOT_FINISHED);
  p.ns.assign(ns_id, ns_id + K);
  t.pods[KT_PODS_RUNNING] = Pods();
  if (!t.have_status) {  // the match reads no status: any observed status serves the given-status pass
    const size_t M = (size_t)t.m, R = (size_t)t.lim.n_resources;
    t.st_calculated.assign(M, 0); t.st_calc_thr.assign(R * M, 0); t.st_calc_present.assign(M, 0); t.st_calc_cnt.assign(M, 0);
    t.st_used.assign(R * M, 0); t.st_used_present.assign(M, 0); t.st_used_cnt.assign(M, 0); t.st_throttled.assign(M, 0);
    t.have_status = true;
  }
  const int rc = evaluate(&t, 0, KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE, nullptr);
  if (rc != KT_OK) return fail(c, rc, t.err.c_str());
  std::memcpy(words, t.pend_bitmap.data(), K * (size_t)t.words() * 4);
  return KT_OK;
}

// the relation from the throttles' side, read from the recorded bitmap columns row by row (engine_oracle_columns.cc)
int kt_get_match_columns(kt_ctx* c, int kind, int64_t k, const int32_t* idx, int64_t* off, int64_t* rows, uint8_t* codes, int64_t cap) {
  if (!c || k < 0 || cap < 0 || !off || (k > 0 && !idx) || (cap > 0 && !rows) || (kind != KT_PODS_RUNNING && kind != KT_PODS_PENDING))
    return KT_ERR_INVALID;
  if (kind == KT_PODS_RUNNING && codes) return fail(c, KT_ERR_INVALID, "codes belong to the pending rows");
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_match_columns before kt_evaluate");
  for (int64_t j = 0; j < k; ++j)
    if (idx[j] < 0 || idx[j] >= c->m) return fail(c, KT_ERR_INVALID, "throttle out of range");
  const std::vector<uint32_t>& b = kind == KT_PODS_RUNNING ? c->run_bitmap : c->pend_bitmap;
  const size_t Wp = (size_t)c->words();
  std::vector<int64_t> got;
  std::vector<uint8_t> got_codes;
  off[0] = 0;
  for (int64_t j = 0; j < k; ++j) {
    const size_t t = (size_t)idx[j];
    for (int64_t r = 0; r < c->pods[kind].n; ++r)
      if ((b[(size_t)r * Wp + (t >> 5)] >> (t & 31)) & 1u) {
        got.push_back(r);
        if (kind == KT_PODS_PENDING) got_codes.push_back((uint8_t)((c->codes[(size_t)r * 2 * Wp + (t >> 4)] >> (2 * (t & 15))) & 3u));
      }
    off[j + 1] = (int64_t)got.size();
  }
  if ((int64_t)got.size() <= cap)
    for (size_t i = 0; i < got.size(); ++i) {
      rows[i] = got[i];
      if (codes) codes[i] = got_codes[i];
    }
  return KT_OK;
}

// {kt_match_pods calls, kt_evaluate calls} since the library was loaded
void kt_test_device_calls(int64_t* out) {
  out[0] = g_match_calls;
  out[1] = g_evaluate_calls;
}
}
