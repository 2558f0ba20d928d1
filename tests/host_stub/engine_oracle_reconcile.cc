// The oracle-backed engine test double (engine_oracle.cc) plus kt_reconcile_throttles: reconcile(key) of listed throttles,
// computed by the columnar oracle on the recorded current columns (a FRESH_STATUS reconcile-only pass whose results are put
// back afterwards, so that every getter answers as before the call).  Linked with kt_host.cc by tests/test_reconcile_keys.py so
// that kth_reconcile can be checked against the object-level oracle without a GPU.  Test infrastructure only: what it checks
// is kt_host.cc; the kernels are checked by tests/test_reconcile_throttles.py on the GPU.
#include "engine_oracle.cc"

extern "C" int kt_reconcile_throttles(kt_ctx* c, int64_t now, int64_t k, const int32_t* idx, const kt_reconcile_out* o, int64_t* off, int64_t* rows,
                                      int64_t cap) {
  if (!c || !o || !off || k < 0 || cap < 0 || (k > 0 && !idx) || (cap > 0 && !rows)) return KT_ERR_INVALID;
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_reconcile_throttles before kt_upload_throttles");
  for (int64_t j = 0; j < k; ++j)
    if (idx[j] < 0 || idx[j] >= c->m) return fail(c, KT_ERR_INVALID, "throttle out of range");
  off[0] = 0;
  if (k == 0) return KT_OK;
  // the results of the last pass, restored below
  const std::vector<int64_t> used = c->o_used, used_cnt = c->o_used_cnt, calc_thr = c->o_calc_thr, calc_cnt = c->o_calc_cnt;
  const std::vector<uint32_t> used_present = c->o_used_present, throttled = c->o_throttled, calc_present = c->o_calc_present,
                              run_bitmap = c->run_bitmap, pend_bitmap = c->pend_bitmap, codes = c->codes;
  const std::vector<uint8_t> ovr_active = c->o_ovr_active, admit = c->admit;
  const bool evaluated = c->evaluated;
  int rc = evaluate(c, now, KT_EVAL_FRESH_STATUS | KT_EVAL_SKIP_CHECK, nullptr);
  if (rc == KT_OK) rc = kt_get_reconcile_rows(c, k, idx, o);
  if (rc == KT_OK) {
    const size_t Wp = (size_t)c->words();
    std::vector<int64_t> got;
    for (int64_t j = 0; j < k; ++j) {
      const size_t t = (size_t)idx[j];
      for (int64_t r = 0; r < c->pods[KT_PODS_RUNNING].n; ++r)
        if ((c->run_bitmap[(size_t)r * Wp + (t >> 5)] >> (t & 31)) & 1u) got.push_back(r);
      off[j + 1] = (int64_t)got.size();
    }
    if ((int64_t)got.size() <= cap)
      for (size_t i = 0; i < got.size(); ++i) rows[i] = got[i];
  }
  c->o_used = used; c->o_used_cnt = used_cnt; c->o_calc_thr = calc_thr; c->o_calc_cnt = calc_cnt;
  c->o_used_present = used_present; c->o_throttled = throttled; c->o_calc_present = calc_present; c->o_ovr_active = ovr_active;
  c->run_bitmap = run_bitmap; c->pend_bitmap = pend_bitmap; c->codes = codes; c->admit = admit;
  c->evaluated = evaluated;
  return rc;
}
