// Second test double for the device engine (include/kt_b200.h): it RECORDS the columns the host layer uploads and, when asked
// for a pass, hands them to the columnar ORACLE (oracle/ko_columnar.h through ko_columnar_evaluate).  With it the host layer
// of the product (kt_host.cc: packer, dictionaries, scales, status bookkeeping, reservation cache, PreFilter reasons, queue
// admission) can be exercised by the scenario suites WITHOUT a GPU -- useful when a host-side change has to be checked and
// no device is at hand.  It is test infrastructure in the strictest sense:
//   * it lives under tests/ and is linked only into tests/_build/libkt_hostoracle.so by tests/conftest.py;
//   * nothing under kube_throttler_b200/ knows it exists; the product library has no CPU path and fails without a device;
//   * what it checks is kt_host.cc, never the CUDA kernels: GPU parity is established by the `-m gpu` tests alone.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/kt_b200.h"

// must match oracle/ko_capi.cc
struct ko_columnar_args {
  kt_limits lim;
  int64_t n_running;
  const int64_t* run_labels; const int64_t* run_req; const uint32_t* run_present; const uint32_t* run_flags; const int32_t* run_ns;
  int64_t n_pending;
  const int64_t* pend_labels; const int64_t* pend_req; const uint32_t* pend_present; const uint32_t* pend_flags; const int32_t* pend_ns;
  int32_t n_ns; const int64_t* ns_labels;
  int32_t m;
  const kt_throttle_cols* thr;
  const kt_selector_table* sel;
  const kt_status_cols* status;
  const int64_t* reserved; const uint32_t* reserved_present; const int64_t* reserved_cnt;
  int64_t now; uint32_t flags; int32_t words_per_row;
  kt_reconcile_out rec;
  uint32_t* run_bitmap; uint32_t* pend_bitmap; uint32_t* codes; uint8_t* admit;
};
extern "C" int ko_columnar_evaluate(const ko_columnar_args* a);
extern "C" int ko_columnar_admit_queue(const ko_columnar_args* a, int64_t first, int64_t count, int64_t* res, uint32_t* res_present,
                                       int64_t* res_cnt, int64_t* admitted);

namespace {
template <class T>
std::vector<T> vec(const T* p, size_t n) { return p && n ? std::vector<T>(p, p + n) : std::vector<T>(); }
template <class T>
const T* ptr(const std::vector<T>& v) { static const T zero[1] = {}; return v.empty() ? zero : v.data(); }

struct Pods {
  int64_t n = 0;
  std::vector<int64_t> labels, req;
  std::vector<uint32_t> present, flags;
  std::vector<int32_t> ns;
};
}  // namespace

struct kt_ctx {
  kt_limits lim{};
  std::string err;
  Pods pods[2];
  int32_t n_ns = 0;
  std::vector<int64_t> ns_labels;
  bool have_throttles = false, have_status = false, have_reserved = false, evaluated = false;
  int32_t m = 0;
  // deep copies of kt_throttle_cols / kt_selector_table / kt_status_cols
  std::vector<uint8_t> kind, tflags, ovr_flags, term_flags, req_op, st_calculated;
  std::vector<int32_t> thr_ns, ovr_off, term_off, pod_req_off, ns_req_off, req_val_off;
  std::vector<int64_t> thr, thr_cnt, ovr_begin, ovr_end, ovr_thr, ovr_cnt, st_calc_thr, st_calc_cnt, st_used, st_used_cnt, reserved, reserved_cnt;
  std::vector<uint32_t> thr_present, ovr_present, req_key, req_vals, st_calc_present, st_used_present, st_throttled, reserved_present;
  int32_t n_ovr = 0, n_terms = 0, n_reqs = 0, n_vals = 0;
  // results of the last pass
  std::vector<int64_t> o_used, o_used_cnt, o_calc_thr, o_calc_cnt;
  std::vector<uint32_t> o_used_present, o_throttled, o_calc_present, run_bitmap, pend_bitmap, codes;
  std::vector<uint8_t> o_ovr_active, admit;
  int64_t sparse_cap = 0;
  int32_t words() const { const int32_t w = (m + 31) / 32; const int32_t p = (w + 3) / 4 * 4; return p < 4 ? 4 : p; }
};

static int fail(kt_ctx* c, int code, const char* msg) { c->err = msg; return code; }

struct AdmitCall { int64_t first, count, admitted; };  // a queue to admit after the pass

extern "C" {
static int evaluate(kt_ctx* c, int64_t now, uint32_t flags, AdmitCall* q);

int kt_create(kt_ctx** out, int, const kt_limits* lim) {
  if (!out || !lim || lim->abi_version != KT_ABI_VERSION) return KT_ERR_INVALID;
  if (lim->n_resources < 1 || lim->n_resources > KT_MAX_RESOURCES || lim->label_slots < 1 || lim->label_slots > KT_MAX_LABEL_SLOTS) return KT_ERR_LIMIT;
  *out = new kt_ctx();
  (*out)->lim = *lim;
  return KT_OK;
}
void kt_destroy(kt_ctx* c) { delete c; }
const char* kt_last_error(const kt_ctx* c) { return c ? c->err.c_str() : "null context"; }

int kt_upload_pods(kt_ctx* c, int kind, int64_t n, const int64_t* labels, const int64_t* req, const uint32_t* present, const uint32_t* flags, const int32_t* ns) {
  if (!c || (kind != KT_PODS_RUNNING && kind != KT_PODS_PENDING) || n < 0) return KT_ERR_INVALID;
  Pods& s = c->pods[kind];
  const size_t L = (size_t)c->lim.label_slots, R = (size_t)c->lim.n_resources, N = (size_t)n;
  s.n = n;
  s.labels = vec(labels, L * N); s.req = vec(req, R * N); s.present = vec(present, N); s.flags = vec(flags, N); s.ns = vec(ns, N);
  c->evaluated = false;
  return KT_OK;
}
int kt_update_pod_rows(kt_ctx* c, int kind, int64_t k, const int64_t* rows, const int64_t* labels, const int64_t* req, const uint32_t* present,
                       const uint32_t* flags, const int32_t* ns) {
  if (!c || (kind != KT_PODS_RUNNING && kind != KT_PODS_PENDING) || k < 0) return KT_ERR_INVALID;
  Pods& s = c->pods[kind];
  const int L = c->lim.label_slots, R = c->lim.n_resources;
  for (int64_t i = 0; i < k; ++i) {
    const int64_t row = rows[i];
    if (row < 0 || row >= s.n) return fail(c, KT_ERR_INVALID, "delta row out of range");
    for (int l = 0; l < L; ++l) s.labels[(size_t)l * s.n + row] = labels[(size_t)l * k + i];
    for (int r = 0; r < R; ++r) s.req[(size_t)r * s.n + row] = req[(size_t)r * k + i];
    s.present[row] = present[i]; s.flags[row] = flags[i]; s.ns[row] = ns[i];
  }
  c->evaluated = false;
  return KT_OK;
}
int kt_upload_namespaces(kt_ctx* c, int32_t n_ns, const int64_t* labels) {
  if (!c || n_ns < 0) return KT_ERR_INVALID;
  c->n_ns = n_ns;
  c->ns_labels = vec(labels, (size_t)c->lim.ns_label_slots * n_ns);
  c->evaluated = false;
  return KT_OK;
}
int kt_upload_throttles(kt_ctx* c, int32_t m, const kt_throttle_cols* t, const kt_selector_table* s) {
  if (!c || m < 0 || !t || !s) return KT_ERR_INVALID;
  const size_t M = (size_t)m, R = (size_t)c->lim.n_resources, O = (size_t)t->n_ovr;
  c->m = m;
  c->kind = vec(t->kind, M); c->thr_ns = vec(t->ns_id, M); c->tflags = vec(t->flags, M); c->thr = vec(t->thr, R * M);
  c->thr_present = vec(t->thr_present, M); c->thr_cnt = vec(t->thr_cnt, M); c->ovr_off = vec(t->ovr_off, M + 1); c->n_ovr = t->n_ovr;
  c->ovr_begin = vec(t->ovr_begin, O); c->ovr_end = vec(t->ovr_end, O); c->ovr_flags = vec(t->ovr_flags, O); c->ovr_thr = vec(t->ovr_thr, R * O);
  c->ovr_present = vec(t->ovr_present, O); c->ovr_cnt = vec(t->ovr_cnt, O);
  c->n_terms = s->n_terms; c->n_reqs = s->n_reqs; c->n_vals = s->n_vals;
  c->term_off = vec(s->term_off, M + 1); c->term_flags = vec(s->term_flags, (size_t)s->n_terms);
  c->pod_req_off = vec(s->pod_req_off, (size_t)s->n_terms + 1); c->ns_req_off = vec(s->ns_req_off, (size_t)s->n_terms + 1);
  c->req_key = vec(s->req_key, (size_t)s->n_reqs); c->req_op = vec(s->req_op, (size_t)s->n_reqs);
  c->req_val_off = vec(s->req_val_off, (size_t)s->n_reqs + 1); c->req_vals = vec(s->req_vals, (size_t)s->n_vals);
  c->have_throttles = true;
  c->have_status = c->have_reserved = false;  // as the engine: both belong to the previous set of throttle columns
  c->evaluated = false;
  return KT_OK;
}
int kt_upload_status(kt_ctx* c, const kt_status_cols* st) {
  if (!c || !st) return KT_ERR_INVALID;
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_upload_status before kt_upload_throttles");
  const size_t M = (size_t)c->m, R = (size_t)c->lim.n_resources;
  c->st_calculated = vec(st->calculated, M); c->st_calc_thr = vec(st->calc_thr, R * M); c->st_calc_present = vec(st->calc_present, M);
  c->st_calc_cnt = vec(st->calc_cnt, M); c->st_used = vec(st->used, R * M); c->st_used_present = vec(st->used_present, M);
  c->st_used_cnt = vec(st->used_cnt, M); c->st_throttled = vec(st->throttled, M);
  c->have_status = true;
  c->evaluated = false;
  return KT_OK;
}
int kt_set_reserved(kt_ctx* c, const int64_t* reserved, const uint32_t* present, const int64_t* cnt) {
  if (!c) return KT_ERR_INVALID;
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_set_reserved before kt_upload_throttles");
  c->evaluated = false;
  if (!reserved && !present && !cnt) { c->have_reserved = false; return KT_OK; }
  if (!reserved || !present || !cnt) return fail(c, KT_ERR_INVALID, "reserved columns must be all set or all null");
  const size_t M = (size_t)c->m, R = (size_t)c->lim.n_resources;
  c->reserved = vec(reserved, R * M); c->reserved_present = vec(present, M); c->reserved_cnt = vec(cnt, M);
  c->have_reserved = true;
  return KT_OK;
}
int32_t kt_match_words(const kt_ctx* c) { return c && c->have_throttles ? c->words() : 0; }

int kt_evaluate(kt_ctx* c, int64_t now, uint32_t flags) { return evaluate(c, now, flags, nullptr); }

// Queue-ordered greedy admission: the columnar oracle's pod-by-pod loop (columnar_admit_queue; the device runs a prefix-sum
// fixpoint, csrc/kt_admit.cuh) -- PreFilter against the observed status + the reservations so far, and on Success the pod's
// ResourceAmountOfPod joins the reservation of every throttle it affects (plugin.go:148-238).  The reservations uploaded with
// kt_set_reserved are left as they were, as on the device.
int kt_admit_queue(kt_ctx* c, int64_t first, int64_t count, uint32_t flags, int32_t* rounds, int64_t* admitted) {
  if (!c || first < 0 || count < 0) return KT_ERR_INVALID;
  if (!c->have_status) return fail(c, KT_ERR_STATE, "kt_admit_queue without kt_upload_status");
  if (first + count > c->pods[KT_PODS_PENDING].n) return fail(c, KT_ERR_INVALID, "queue rows outside the pending table");
  AdmitCall q{first, count, 0};
  const int rc = evaluate(c, 0, KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE | (flags & KT_EVAL_ON_EQUAL), &q);
  if (rc != KT_OK) return rc;
  if (rounds) *rounds = 2;
  if (admitted) *admitted = q.admitted;
  return KT_OK;
}

static int evaluate(kt_ctx* c, int64_t now, uint32_t flags, AdmitCall* q) {
  if (!c) return KT_ERR_INVALID;
  if (!c->have_throttles) return fail(c, KT_ERR_STATE, "kt_evaluate before kt_upload_throttles");
  if ((flags & KT_EVAL_GIVEN_STATUS) && !c->have_status) return fail(c, KT_ERR_STATE, "KT_EVAL_GIVEN_STATUS without kt_upload_status");
  const size_t M = (size_t)c->m, R = (size_t)c->lim.n_resources, Wp = (size_t)c->words();
  const Pods &run = c->pods[KT_PODS_RUNNING], &pend = c->pods[KT_PODS_PENDING];
  kt_throttle_cols t{};
  t.kind = ptr(c->kind); t.ns_id = ptr(c->thr_ns); t.flags = ptr(c->tflags); t.thr = ptr(c->thr); t.thr_present = ptr(c->thr_present);
  t.thr_cnt = ptr(c->thr_cnt); t.ovr_off = ptr(c->ovr_off); t.n_ovr = c->n_ovr; t.ovr_begin = ptr(c->ovr_begin); t.ovr_end = ptr(c->ovr_end);
  t.ovr_flags = ptr(c->ovr_flags); t.ovr_thr = ptr(c->ovr_thr); t.ovr_present = ptr(c->ovr_present); t.ovr_cnt = ptr(c->ovr_cnt);
  kt_selector_table s{};
  s.n_terms = c->n_terms; s.n_reqs = c->n_reqs; s.n_vals = c->n_vals; s.term_off = ptr(c->term_off); s.term_flags = ptr(c->term_flags);
  s.pod_req_off = ptr(c->pod_req_off); s.ns_req_off = ptr(c->ns_req_off); s.req_key = ptr(c->req_key); s.req_op = ptr(c->req_op);
  s.req_val_off = ptr(c->req_val_off); s.req_vals = ptr(c->req_vals);
  kt_status_cols st{};
  st.calculated = ptr(c->st_calculated); st.calc_thr = ptr(c->st_calc_thr); st.calc_present = ptr(c->st_calc_present); st.calc_cnt = ptr(c->st_calc_cnt);
  st.used = ptr(c->st_used); st.used_present = ptr(c->st_used_present); st.used_cnt = ptr(c->st_used_cnt); st.throttled = ptr(c->st_throttled);
  c->o_used.assign(R * M, 0); c->o_used_cnt.assign(M, 0); c->o_calc_thr.assign(R * M, 0); c->o_calc_cnt.assign(M, 0);
  c->o_used_present.assign(M, 0); c->o_throttled.assign(M, 0); c->o_calc_present.assign(M, 0); c->o_ovr_active.assign(M, 0);
  c->run_bitmap.assign((size_t)run.n * Wp + 1, 0); c->pend_bitmap.assign((size_t)pend.n * Wp + 1, 0);
  c->codes.assign((size_t)pend.n * 2 * Wp + 1, 0); c->admit.assign((size_t)pend.n + 1, 0);
  ko_columnar_args a{};
  a.lim = c->lim;
  a.n_running = run.n; a.run_labels = ptr(run.labels); a.run_req = ptr(run.req); a.run_present = ptr(run.present); a.run_flags = ptr(run.flags); a.run_ns = ptr(run.ns);
  a.n_pending = pend.n; a.pend_labels = ptr(pend.labels); a.pend_req = ptr(pend.req); a.pend_present = ptr(pend.present); a.pend_flags = ptr(pend.flags); a.pend_ns = ptr(pend.ns);
  a.n_ns = c->n_ns; a.ns_labels = ptr(c->ns_labels);
  a.m = c->m; a.thr = &t; a.sel = &s; a.status = c->have_status ? &st : nullptr;
  a.reserved = c->have_reserved ? ptr(c->reserved) : nullptr;
  a.reserved_present = c->have_reserved ? ptr(c->reserved_present) : nullptr;
  a.reserved_cnt = c->have_reserved ? ptr(c->reserved_cnt) : nullptr;
  a.now = now; a.flags = flags; a.words_per_row = (int32_t)Wp;
  a.rec = kt_reconcile_out{c->o_used.data(), c->o_used_present.data(), c->o_used_cnt.data(), c->o_throttled.data(), c->o_calc_thr.data(),
                           c->o_calc_present.data(), c->o_calc_cnt.data(), c->o_ovr_active.data()};
  a.run_bitmap = c->run_bitmap.data(); a.pend_bitmap = c->pend_bitmap.data(); a.codes = c->codes.data(); a.admit = c->admit.data();
  if (ko_columnar_evaluate(&a) != 0) return fail(c, KT_ERR_INVALID, "ko_columnar_evaluate failed");
  if (q) {  // the queue rows again, pod by pod (the pass above gave the reconcile columns and the rows outside the queue)
    std::vector<int64_t> res(R * M + 1), res_cnt(M + 1);
    std::vector<uint32_t> res_present(M + 1);
    if (ko_columnar_admit_queue(&a, q->first, q->count, res.data(), res_present.data(), res_cnt.data(), &q->admitted) != 0)
      return fail(c, KT_ERR_INVALID, "ko_columnar_admit_queue failed");
  }
  c->evaluated = true;
  return KT_OK;
}
int kt_get_reconcile(kt_ctx* c, const kt_reconcile_out* o) {
  if (!c || !o) return KT_ERR_INVALID;
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_reconcile before kt_evaluate");
  auto put = [](auto* dst, const auto& v) { if (dst && !v.empty()) std::memcpy(dst, v.data(), v.size() * sizeof(v[0])); };
  put(o->used, c->o_used); put(o->used_present, c->o_used_present); put(o->used_cnt, c->o_used_cnt); put(o->throttled, c->o_throttled);
  put(o->calc_thr, c->o_calc_thr); put(o->calc_present, c->o_calc_present); put(o->calc_cnt, c->o_calc_cnt); put(o->override_active, c->o_ovr_active);
  return KT_OK;
}
int kt_get_match_bitmap(kt_ctx* c, int kind, uint32_t* words) {
  if (!c || !words || (kind != KT_PODS_RUNNING && kind != KT_PODS_PENDING)) return KT_ERR_INVALID;
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_match_bitmap before kt_evaluate");
  const std::vector<uint32_t>& b = kind == KT_PODS_RUNNING ? c->run_bitmap : c->pend_bitmap;
  std::memcpy(words, b.data(), (size_t)c->pods[kind].n * c->words() * 4);
  return KT_OK;
}
int kt_get_match_rows(kt_ctx* c, int kind, int64_t k, const int64_t* rows, uint32_t* words) {
  if (!c || k < 0 || (k > 0 && (!rows || !words)) || (kind != KT_PODS_RUNNING && kind != KT_PODS_PENDING)) return KT_ERR_INVALID;
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_match_rows before kt_evaluate");
  const std::vector<uint32_t>& b = kind == KT_PODS_RUNNING ? c->run_bitmap : c->pend_bitmap;
  const size_t Wp = (size_t)c->words();
  for (int64_t i = 0; i < k; ++i) {
    if (rows[i] < 0 || rows[i] >= c->pods[kind].n) return fail(c, KT_ERR_INVALID, "row out of range");
    std::memcpy(words + (size_t)i * Wp, b.data() + (size_t)rows[i] * Wp, Wp * 4);
  }
  return KT_OK;
}
int kt_get_check(kt_ctx* c, uint32_t* codes, uint8_t* admit) {
  if (!c) return KT_ERR_INVALID;
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_check before kt_evaluate");
  const size_t P = (size_t)c->pods[KT_PODS_PENDING].n, Wp = (size_t)c->words();
  if (codes && P) std::memcpy(codes, c->codes.data(), P * 2 * Wp * 4);
  if (admit && P) std::memcpy(admit, c->admit.data(), P);
  return KT_OK;
}
int kt_get_check_rows(kt_ctx* c, int64_t k, const int64_t* rows, uint32_t* codes, uint8_t* admit) {
  if (!c || k < 0 || (k > 0 && !rows)) return KT_ERR_INVALID;
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_check_rows before kt_evaluate");
  const size_t Wc = 2 * (size_t)c->words();
  for (int64_t i = 0; i < k; ++i) {
    if (rows[i] < 0 || rows[i] >= c->pods[KT_PODS_PENDING].n) return fail(c, KT_ERR_INVALID, "row out of range");
    if (codes) std::memcpy(codes + (size_t)i * Wc, c->codes.data() + (size_t)rows[i] * Wc, Wc * 4);
    if (admit) admit[i] = c->admit[(size_t)rows[i]];
  }
  return KT_OK;
}
// Status diff of the last reconciling pass against the uploaded status, the obvious way (the device does it inside the pass).
int kt_get_changed(kt_ctx* c, int32_t* idx, int64_t cap, int64_t* count, uint8_t* flags) {
  if (!c || !count) return KT_ERR_INVALID;
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_changed before kt_evaluate");
  if (!c->have_status) return fail(c, KT_ERR_STATE, "kt_get_changed without kt_upload_status");
  const size_t M = (size_t)c->m, R = (size_t)c->lim.n_resources;
  int64_t n = 0;
  for (size_t t = 0; t < M; ++t) {
    const bool live = (c->tflags[t] & KT_THR_RESPONSIBLE) && !(c->tflags[t] & KT_THR_SELECTOR_ERROR);
    bool diff = false;
    if (live) {
      diff = !c->st_calculated[t] || c->o_used_present[t] != c->st_used_present[t] || c->o_throttled[t] != c->st_throttled[t] ||
             c->o_calc_present[t] != c->st_calc_present[t];
      if ((c->o_used_present[t] & KT_COUNT_BIT) && c->o_used_cnt[t] != c->st_used_cnt[t]) diff = true;
      if ((c->o_calc_present[t] & KT_COUNT_BIT) && c->o_calc_cnt[t] != c->st_calc_cnt[t]) diff = true;
      for (size_t r = 0; r < R; ++r) {
        if (((c->o_used_present[t] >> r) & 1) && c->o_used[r * M + t] != c->st_used[r * M + t]) diff = true;
        if (((c->o_calc_present[t] >> r) & 1) && c->o_calc_thr[r * M + t] != c->st_calc_thr[r * M + t]) diff = true;
      }
    }
    if (flags) flags[t] = diff;
    if (diff) { if (n < cap && idx) idx[n] = (int32_t)t; ++n; }
  }
  *count = n;
  return KT_OK;
}
int kt_get_reconcile_rows(kt_ctx* c, int64_t k, const int32_t* idx, const kt_reconcile_out* o) {
  if (!c || !o || k < 0 || (k > 0 && !idx)) return KT_ERR_INVALID;
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_reconcile_rows before kt_evaluate");
  const size_t M = (size_t)c->m, R = (size_t)c->lim.n_resources, K = (size_t)k;
  for (size_t i = 0; i < K; ++i) {
    const size_t t = (size_t)idx[i];
    if (t >= M) return fail(c, KT_ERR_INVALID, "throttle out of range");
    for (size_t r = 0; r < R; ++r) {
      if (o->used) o->used[r * K + i] = c->o_used[r * M + t];
      if (o->calc_thr) o->calc_thr[r * K + i] = c->o_calc_thr[r * M + t];
    }
    if (o->used_cnt) o->used_cnt[i] = c->o_used_cnt[t];
    if (o->calc_cnt) o->calc_cnt[i] = c->o_calc_cnt[t];
    if (o->used_present) o->used_present[i] = c->o_used_present[t];
    if (o->throttled) o->throttled[i] = c->o_throttled[t];
    if (o->calc_present) o->calc_present[i] = c->o_calc_present[t];
    if (o->override_active) o->override_active[i] = c->o_ovr_active[t];
  }
  return KT_OK;
}
// the sparse list of the double: the non-zero code words of the dense rows, in row order
int kt_set_sparse_check(kt_ctx* c, int64_t cap) {
  if (!c || cap < 0) return KT_ERR_INVALID;
  c->sparse_cap = cap;
  c->evaluated = false;
  return KT_OK;
}
int kt_get_check_sparse(kt_ctx* c, uint8_t* admit, uint32_t* entries, int64_t cap, int64_t* count) {
  if (!c || !count) return KT_ERR_INVALID;
  if (!c->evaluated) return fail(c, KT_ERR_STATE, "kt_get_check_sparse before kt_evaluate");
  if (!c->sparse_cap) return fail(c, KT_ERR_STATE, "kt_get_check_sparse without kt_set_sparse_check");
  const size_t P = (size_t)c->pods[KT_PODS_PENDING].n, Wc = 2 * (size_t)c->words();
  if (admit && P) std::memcpy(admit, c->admit.data(), P);
  int64_t n = 0;
  const int64_t room = cap < c->sparse_cap ? cap : c->sparse_cap;
  for (size_t row = 0; row < P; ++row)
    for (size_t j = 0; j < Wc; ++j) {
      const uint32_t word = c->codes[row * Wc + j];
      if (!word) continue;
      if (n < room) { entries[3 * n] = (uint32_t)row; entries[3 * n + 1] = (uint32_t)j; entries[3 * n + 2] = word; }
      ++n;
    }
  *count = n;
  return KT_OK;
}
}
