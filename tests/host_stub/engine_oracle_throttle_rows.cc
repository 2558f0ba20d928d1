// The oracle-backed engine test double (engine_oracle.cc, with kt_reconcile_throttles of engine_oracle_reconcile.cc) plus the
// throttle-side column deltas kt_update_status_rows / kt_update_reserved_rows: scatters into the recorded status and reservation
// columns, with the engine's argument and state checks.  It counts the calls that move throttle state to the device
// (kt_test_throttle_calls), so that tests/test_status_echo.py can check which of them a status echo, a Reserve or a spec edit
// makes.  Linked with kt_host.cc so that the host layer's delta paths can be checked against a twin plugin and the object-level
// oracle without a GPU.  Test infrastructure only: what it checks is kt_host.cc; the kernels are checked by
// tests/test_throttle_rows.py on the GPU.
#define kt_upload_throttles kt_upload_throttles_uncounted
#define kt_upload_status kt_upload_status_uncounted
#define kt_set_reserved kt_set_reserved_uncounted
#define kt_evaluate kt_evaluate_uncounted
#include "engine_oracle_reconcile.cc"
#undef kt_upload_throttles
#undef kt_upload_status
#undef kt_set_reserved
#undef kt_evaluate

#include <algorithm>

namespace {
// kt_upload_throttles, kt_upload_status, kt_set_reserved, kt_update_status_rows, kt_update_reserved_rows, kt_evaluate
int64_t g_calls[6] = {};

int check_columns(kt_ctx* c, int64_t k, const int32_t* idx) {
  for (int64_t i = 0; i < k; ++i)
    if (idx[i] < 0 || idx[i] >= c->m) return fail(c, KT_ERR_INVALID, "throttle out of range");
  std::vector<int32_t> s(idx, idx + k);
  std::sort(s.begin(), s.end());
  if (std::adjacent_find(s.begin(), s.end()) != s.end()) return fail(c, KT_ERR_INVALID, "throttle listed twice");
  return KT_OK;
}
}  // namespace

extern "C" {

int kt_upload_throttles(kt_ctx* c, int32_t m, const kt_throttle_cols* t, const kt_selector_table* s) {
  ++g_calls[0];
  return kt_upload_throttles_uncounted(c, m, t, s);
}
int kt_upload_status(kt_ctx* c, const kt_status_cols* st) {
  ++g_calls[1];
  return kt_upload_status_uncounted(c, st);
}
int kt_set_reserved(kt_ctx* c, const int64_t* reserved, const uint32_t* present, const int64_t* cnt) {
  ++g_calls[2];
  return kt_set_reserved_uncounted(c, reserved, present, cnt);
}
int kt_evaluate(kt_ctx* c, int64_t now, uint32_t flags) {
  ++g_calls[5];
  return kt_evaluate_uncounted(c, now, flags);
}

int kt_update_status_rows(kt_ctx* c, int64_t k, const int32_t* idx, const kt_status_cols* st) {
  if (!c || k < 0) return KT_ERR_INVALID;
  if (k > 0 && (!idx || !st || !st->calculated || !st->calc_thr || !st->calc_present || !st->calc_cnt || !st->used || !st->used_present ||
                !st->used_cnt || !st->throttled))
    return fail(c, KT_ERR_INVALID, "kt_update_status_rows: null column");
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_update_status_rows before kt_upload_throttles");
  if (!c->have_status) return fail(c, KT_ERR_STATE, "kt_update_status_rows before kt_upload_status");
  if (k == 0) return KT_OK;
  if (int rc = check_columns(c, k, idx)) return rc;
  ++g_calls[3];
  const size_t M = (size_t)c->m, R = (size_t)c->lim.n_resources, K = (size_t)k;
  for (size_t i = 0; i < K; ++i) {
    const size_t t = (size_t)idx[i];
    for (size_t r = 0; r < R; ++r) {
      c->st_calc_thr[r * M + t] = st->calc_thr[r * K + i];
      c->st_used[r * M + t] = st->used[r * K + i];
    }
    c->st_calculated[t] = st->calculated[i]; c->st_calc_present[t] = st->calc_present[i]; c->st_calc_cnt[t] = st->calc_cnt[i];
    c->st_used_present[t] = st->used_present[i]; c->st_used_cnt[t] = st->used_cnt[i]; c->st_throttled[t] = st->throttled[i];
  }
  c->evaluated = false;
  return KT_OK;
}

int kt_update_reserved_rows(kt_ctx* c, int64_t k, const int32_t* idx, const int64_t* reserved, const uint32_t* present, const int64_t* cnt) {
  if (!c || k < 0) return KT_ERR_INVALID;
  if (k > 0 && (!idx || !reserved || !present || !cnt)) return fail(c, KT_ERR_INVALID, "kt_update_reserved_rows: null column");
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_update_reserved_rows before kt_upload_throttles");
  if (k == 0) return KT_OK;
  if (int rc = check_columns(c, k, idx)) return rc;
  ++g_calls[4];
  const size_t M = (size_t)c->m, R = (size_t)c->lim.n_resources, K = (size_t)k;
  if (!c->have_reserved) {  // nothing reserved on the other columns
    c->reserved.assign(R * M, 0); c->reserved_present.assign(M, 0); c->reserved_cnt.assign(M, 0);
  }
  for (size_t i = 0; i < K; ++i) {
    const size_t t = (size_t)idx[i];
    for (size_t r = 0; r < R; ++r) c->reserved[r * M + t] = reserved[r * K + i];
    c->reserved_present[t] = present[i];
    c->reserved_cnt[t] = cnt[i];
  }
  c->have_reserved = true;
  c->evaluated = false;
  return KT_OK;
}

// the calls since the library was loaded, in the order of g_calls
void kt_test_throttle_calls(int64_t* out) {
  for (int i = 0; i < 6; ++i) out[i] = g_calls[i];
}
}
