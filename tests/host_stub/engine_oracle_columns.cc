// The oracle-backed engine test double (engine_oracle.cc) plus kt_get_match_columns: the relation from the throttles' side,
// read from the recorded bitmap columns row by row.  Linked with kt_host.cc by tests/test_affected_pods.py so that
// kth_affected_pods can be checked against the object-level oracle without a GPU.  Test infrastructure only: what it checks
// is kt_host.cc; the device transpose is checked by tests/test_match_columns.py on the GPU.
#include "engine_oracle.cc"

extern "C" int kt_get_match_columns(kt_ctx* c, int kind, int64_t k, const int32_t* idx, int64_t* off, int64_t* rows, uint8_t* codes,
                                    int64_t cap) {
  if (!c || k < 0 || cap < 0 || !off || (k > 0 && !idx) || (cap > 0 && !rows) || (kind != KT_PODS_RUNNING && kind != KT_PODS_PENDING))
    return KT_ERR_INVALID;
  if (kind == KT_PODS_RUNNING && codes) return fail(c, KT_ERR_INVALID, "codes belong to the pending rows");
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_match_columns before kt_evaluate");
  for (int64_t j = 0; j < k; ++j)
    if (idx[j] < 0 || idx[j] >= c->m) return fail(c, KT_ERR_INVALID, "throttle out of range");
  const std::vector<uint32_t>& b = kind == KT_PODS_RUNNING ? c->run_bitmap : c->pend_bitmap;
  const size_t Wp = (size_t)c->words();
  const int64_t n = c->pods[kind].n;
  std::vector<int64_t> got;
  std::vector<uint8_t> got_codes;
  off[0] = 0;
  for (int64_t j = 0; j < k; ++j) {
    const size_t t = (size_t)idx[j];
    for (int64_t r = 0; r < n; ++r)
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
