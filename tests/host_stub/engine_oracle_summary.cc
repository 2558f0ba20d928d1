// The oracle-backed engine test double (engine_oracle.cc, with kt_reconcile_throttles, kt_get_match_columns and kt_match_pods as
// engine_oracle_match_pods.cc has them) plus kt_get_check_summary: the pending rows of the last pass summarised per throttle, counted row by row from the recorded dense
// codes, admit bytes and pending request columns.  Linked with kt_host.cc by tests/test_queue_report.py so that kth_queue_report
// can be checked against kth_pre_filter_queue, kth_affected_pods and kth_pre_filter_key without a GPU.  Test infrastructure only:
// what it checks is kt_host.cc; the kernel is checked by tests/test_check_summary.py on the GPU.
#include "engine_oracle_match_pods.cc"

extern "C" int kt_get_check_summary(kt_ctx* c, int64_t first, int64_t count, const uint8_t* row_class, const kt_check_summary* o) {
  if (!c || !o) return KT_ERR_INVALID;
  const int64_t P = c->pods[KT_PODS_PENDING].n;
  if (first < 0 || count < 0 || first > P - count) return fail(c, KT_ERR_INVALID, "rows outside the pending table");
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_check_summary before kt_evaluate");
  const size_t M = (size_t)c->m, R = (size_t)c->lim.n_resources, Wc = 2 * (size_t)c->words(), N = (size_t)P;
  std::vector<int64_t> status_cnt(3 * M), sole_cnt(M), held(R * M);
  std::vector<uint32_t> held_present(M);
  for (int64_t i = 0; i < count; ++i) {
    const size_t row = (size_t)(first + i);
    const uint8_t cls = row_class ? row_class[i] : 1;
    if (cls == 0 || c->admit[row]) continue;
    std::vector<std::pair<size_t, uint32_t>> nz;  // (throttle, code)
    for (size_t t = 0; t < M; ++t) {
      const uint32_t code = (c->codes[row * Wc + (t >> 4)] >> (2 * (t & 15))) & 3u;
      if (code) nz.emplace_back(t, code);
    }
    const uint32_t present = c->pods[KT_PODS_PENDING].present[row] & ~KT_COUNT_BIT;
    for (auto& e : nz) {
      const size_t t = e.first;
      ++status_cnt[(size_t)(e.second - 1) * M + t];
      if (cls == 1 && nz.size() == 1) ++sole_cnt[t];
      held_present[t] |= present | KT_COUNT_BIT;
      for (size_t r = 0; r < R; ++r)
        if ((present >> r) & 1) held[r * M + t] += c->pods[KT_PODS_PENDING].req[r * N + row];
    }
  }
  if (o->status_cnt && M) std::memcpy(o->status_cnt, status_cnt.data(), 3 * M * 8);
  if (o->sole_cnt && M) std::memcpy(o->sole_cnt, sole_cnt.data(), M * 8);
  if (o->held && M) std::memcpy(o->held, held.data(), R * M * 8);
  if (o->held_present && M) std::memcpy(o->held_present, held_present.data(), M * 4);
  return KT_OK;
}
