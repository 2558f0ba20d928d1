// The oracle-backed engine test double (engine_oracle.cc) plus kt_check_pending_rows: PreFilter of listed pending rows, computed
// by the columnar oracle on the recorded current columns (a GIVEN_STATUS | SKIP_RECONCILE pass whose results are put back
// afterwards, so that every getter answers as before the call).  Linked with kt_host.cc by tests/test_prefilter_keys.py so that
// kth_pre_filter_keys can be checked against kth_pre_filter_key and the object-level oracle without a GPU.  Test infrastructure
// only: what it checks is kt_host.cc; the kernels are checked by tests/test_check_rows.py on the GPU.
#include "engine_oracle.cc"

extern "C" int kt_check_pending_rows(kt_ctx* c, uint32_t flags, int64_t k, const int64_t* rows, uint32_t* words, uint32_t* codes, uint8_t* admit) {
  if (!c || k < 0 || (k > 0 && !rows)) return KT_ERR_INVALID;
  if (flags & ~KT_EVAL_ON_EQUAL) return fail(c, KT_ERR_INVALID, "kt_check_pending_rows: flags must be 0 or KT_EVAL_ON_EQUAL");
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_check_pending_rows before kt_upload_throttles");
  if (!c->have_status) return fail(c, KT_ERR_STATE, "kt_check_pending_rows without kt_upload_status");
  for (int64_t i = 0; i < k; ++i)
    if (rows[i] < 0 || rows[i] >= c->pods[KT_PODS_PENDING].n) return fail(c, KT_ERR_INVALID, "row out of range");
  if (k == 0) return KT_OK;
  // the results of the last pass, restored below
  const std::vector<int64_t> used = c->o_used, used_cnt = c->o_used_cnt, calc_thr = c->o_calc_thr, calc_cnt = c->o_calc_cnt;
  const std::vector<uint32_t> used_present = c->o_used_present, throttled = c->o_throttled, calc_present = c->o_calc_present,
                              run_bitmap = c->run_bitmap, pend_bitmap = c->pend_bitmap, codes_before = c->codes;
  const std::vector<uint8_t> ovr_active = c->o_ovr_active, admit_before = c->admit;
  const bool evaluated = c->evaluated;
  int rc = evaluate(c, 0, KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE | flags, nullptr);
  if (rc == KT_OK) {
    const size_t Wp = (size_t)c->words();
    for (int64_t i = 0; i < k; ++i) {
      const size_t r = (size_t)rows[i];
      if (words) std::memcpy(words + (size_t)i * Wp, c->pend_bitmap.data() + r * Wp, Wp * 4);
      if (codes) std::memcpy(codes + (size_t)i * 2 * Wp, c->codes.data() + r * 2 * Wp, 2 * Wp * 4);
      if (admit) admit[i] = c->admit[r];
    }
  }
  c->o_used = used; c->o_used_cnt = used_cnt; c->o_calc_thr = calc_thr; c->o_calc_cnt = calc_cnt;
  c->o_used_present = used_present; c->o_throttled = throttled; c->o_calc_present = calc_present; c->o_ovr_active = ovr_active;
  c->run_bitmap = run_bitmap; c->pend_bitmap = pend_bitmap; c->codes = codes_before; c->admit = admit_before;
  c->evaluated = evaluated;
  return rc;
}
