// ko_capi.cc -- ORACLE C API (test infrastructure only).  Loaded with ctypes by tests/, by
// __graft_entry__.smoke() and by bench.py's cpu_baseline / --impl reference leg.  Nothing under
// kube_throttler_b200/ may include, link or dlopen this.
//
//   ko_eval(json)            -> json   unit-level calls (KATs transcribed from the reference tests)
//   ko_world_*               -> object-level world: apply manifests, reconcile, PreFilter, Reserve
//   ko_columnar_evaluate     -> columnar oracle on the engine's own int64 columns
//   ko_world_from_columns    -> object World built from those columns (cross-validation + the
//                               "reference-shaped" CPU baseline)
#include <atomic>
#include <chrono>
#include <cstring>
#include <mutex>
#include <thread>
#ifdef __linux__
#include <pthread.h>
#include <sched.h>
#endif

#include "ko_columnar.h"
#include "ko_json.h"
#include "ko_model.h"

using kojson::Value;
using namespace ko;

namespace {

thread_local std::string g_ret;
const char* ret(const std::string& s) { g_ret = s; return g_ret.c_str(); }
const char* ret(const Value& v) { return ret(kojson::dump(v)); }
Value err_obj(const std::string& m) { Value o = Value::object(); o.set("error", Value::str(m)); return o; }

// ---------- JSON -> objects -----------------------------------------------------------
ResourceList rl_from(const Value& v) {
  ResourceList rl;
  for (auto& kv : v.members()) rl[kv.first] = ParseQuantity(kv.second.scalar_text());
  return rl;
}
ResourceAmount ra_from(const Value& v) {
  ResourceAmount a;
  if (!v.is_obj()) return a;
  const Value& rc = v.get("resourceCounts");
  if (rc.is_obj()) { a.hasCounts = true; a.pod = rc.get("pod").int_or(0); }
  const Value& rr = v.get("resourceRequests");
  if (rr.is_obj()) { a.requestsNil = false; a.requests = rl_from(rr); }
  return a;
}
IsResourceAmountThrottled throttled_from(const Value& v) {
  IsResourceAmountThrottled t;
  if (!v.is_obj()) return t;
  t.pod = v.get("resourceCounts").get("pod").bool_or(false);
  const Value& rr = v.get("resourceRequests");
  if (rr.is_obj()) { t.requestsNil = false; for (auto& kv : rr.members()) t.requests[kv.first] = kv.second.bool_or(false); }
  return t;
}
LabelMap labels_from(const Value& v) {
  LabelMap m;
  for (auto& kv : v.members()) m[kv.first] = kv.second.str_or("");
  return m;
}
LabelSelector selector_from(const Value& v) {
  LabelSelector s;
  if (!v.is_obj()) return s;
  s.matchLabels = labels_from(v.get("matchLabels"));
  for (auto& e : v.get("matchExpressions").items()) {
    LabelSelectorRequirement r;
    r.key = e.get("key").str_or("");
    r.op = e.get("operator").str_or("");
    for (auto& x : e.get("values").items()) r.values.push_back(x.str_or(""));
    s.matchExpressions.push_back(std::move(r));
  }
  return s;
}
std::vector<SelectorTerm> terms_from(const Value& selector) {
  std::vector<SelectorTerm> terms;
  // the reference's JSON tag is "selectorTerms" (Go field SelecterTerms, throttle_selector.go:26)
  for (auto& t : selector.get("selectorTerms").items()) {
    SelectorTerm st;
    st.podSelector = selector_from(t.get("podSelector"));
    st.namespaceSelector = selector_from(t.get("namespaceSelector"));
    terms.push_back(std::move(st));
  }
  return terms;
}
Pod pod_from(const Value& v) {
  Pod p;
  const Value& md = v.get("metadata");
  p.ns = md.get("namespace").str_or("");
  p.name = md.get("name").str_or("");
  p.labels = labels_from(md.get("labels"));
  const Value& spec = v.get("spec");
  p.schedulerName = spec.get("schedulerName").str_or("");
  p.nodeName = spec.get("nodeName").str_or("");
  p.phase = v.get("status").get("phase").str_or("");
  for (auto& c : spec.get("initContainers").items()) p.initContainers.push_back(Container{rl_from(c.get("resources").get("requests"))});
  for (auto& c : spec.get("containers").items()) p.containers.push_back(Container{rl_from(c.get("resources").get("requests"))});
  if (spec.get("overhead").is_obj()) { p.hasOverhead = true; p.overhead = rl_from(spec.get("overhead")); }
  return p;
}
Namespace ns_from(const Value& v) {
  Namespace n;
  n.name = v.get("metadata").get("name").str_or("");
  n.labels = labels_from(v.get("metadata").get("labels"));
  return n;
}
Time time_from(const Value& v) {
  Time t;
  if (v.is_str() && !v.s.empty()) {
    std::string e = ParseRFC3339(v.s, &t);
    if (!e.empty()) throw std::runtime_error(e);
  }
  return t;
}
Throttle throttle_from(const Value& v) {
  Throttle t;
  t.kind = v.get("kind").str_or("Throttle") == "ClusterThrottle" ? KindClusterThrottle : KindThrottle;
  const Value& md = v.get("metadata");
  t.ns = t.kind == KindThrottle ? md.get("namespace").str_or("") : "";
  t.name = md.get("name").str_or("");
  const Value& spec = v.get("spec");
  t.throttlerName = spec.get("throttlerName").str_or("");
  t.threshold = ra_from(spec.get("threshold"));
  for (auto& o : spec.get("temporaryThresholdOverrides").items()) {
    TemporaryThresholdOverride ov;
    ov.begin = o.get("begin").str_or("");
    ov.end = o.get("end").str_or("");
    ov.threshold = ra_from(o.get("threshold"));
    t.overrides.push_back(std::move(ov));
  }
  t.terms = terms_from(spec.get("selector"));
  const Value& st = v.get("status");
  if (st.is_obj()) {
    const Value& ct = st.get("calculatedThreshold");
    t.status.calculatedThreshold.threshold = ra_from(ct.get("threshold"));
    Time at = time_from(ct.get("calculatedAt"));
    t.status.calculatedThreshold.calculatedAt = at;
    t.status.calculatedThreshold.calculatedAtSet = !at.IsZero();
    for (auto& m : ct.get("messages").items()) t.status.calculatedThreshold.messages.push_back(m.str_or(""));
    t.status.throttled = throttled_from(st.get("throttled"));
    t.status.used = ra_from(st.get("used"));
  }
  return t;
}

// ---------- objects -> JSON -----------------------------------------------------------
Value rl_to(const ResourceList& rl) {
  Value o = Value::object();
  for (auto& kv : rl) o.set(kv.first, Value::str(QuantityDecimalString(kv.second)));
  return o;
}
Value ra_to(const ResourceAmount& a) {
  Value o = Value::object();
  if (a.hasCounts) { Value c = Value::object(); c.set("pod", Value::number(a.pod)); o.set("resourceCounts", c); }
  if (!a.requestsNil) o.set("resourceRequests", rl_to(a.requests));
  return o;
}
Value throttled_to(const IsResourceAmountThrottled& t) {
  Value o = Value::object();
  Value c = Value::object();
  c.set("pod", Value::boolean(t.pod));
  o.set("resourceCounts", c);
  if (!t.requestsNil) {
    Value r = Value::object();
    for (auto& kv : t.requests) r.set(kv.first, Value::boolean(kv.second));
    o.set("resourceRequests", r);
  }
  return o;
}
Value calc_to(const CalculatedThreshold& c) {
  Value o = Value::object();
  o.set("threshold", ra_to(c.threshold));
  o.set("calculatedAtSet", Value::boolean(c.calculatedAtSet));
  o.set("calculatedAtUnix", Value::number(c.calculatedAt.sec));
  if (!c.messages.empty()) {
    Value m = Value::array();
    for (auto& s : c.messages) m.push(Value::str(s));
    o.set("messages", m);
  }
  return o;
}
Value status_to(const ThrottleStatus& s) {
  Value o = Value::object();
  o.set("calculatedThreshold", calc_to(s.calculatedThreshold));
  o.set("throttled", throttled_to(s.throttled));
  o.set("used", ra_to(s.used));
  return o;
}
Value names_to(const std::vector<const Throttle*>& v) {
  Value a = Value::array();
  for (auto* t : v) a.push(Value::str(t->NN()));
  return a;
}
Value check_to(const CheckResult& r) {
  Value o = Value::object();
  o.set("active", names_to(r.active));
  o.set("insufficient", names_to(r.insufficient));
  o.set("podRequestsExceedsThreshold", names_to(r.exceeds));
  o.set("affected", names_to(r.affected));
  if (!r.error.empty()) o.set("error", Value::str(r.error));
  return o;
}
Value prefilter_to(const PreFilterResult& r) {
  Value o = Value::object();
  o.set("code", Value::str(r.code));
  Value rs = Value::array();
  for (auto& s : r.reasons) rs.push(Value::str(s));
  o.set("reasons", rs);
  if (r.hasEvent) {
    Value e = Value::object();
    e.set("type", Value::str("Warning"));
    e.set("reason", Value::str("ResourceRequestsExceedsThrottleThreshold"));
    e.set("message", Value::str(r.eventMessage));
    o.set("event", e);
  }
  o.set("throttle", check_to(r.thr));
  o.set("clusterthrottle", check_to(r.clthr));
  return o;
}

// ---------- unit-level dispatch -------------------------------------------------------
Value eval_call(const Value& req) {
  std::string fn = req.get("fn").str_or("");
  if (fn == "ParseQuantity") {
    Quantity q = ParseQuantity(req.get("value").scalar_text());
    Value o = Value::object();
    o.set("decimal", Value::str(QuantityDecimalString(q)));
    o.set("format", Value::number((int)q.format));
    return o;
  }
  if (fn == "Quantity.Cmp") {
    return Value::number(ParseQuantity(req.get("a").scalar_text()).Cmp(ParseQuantity(req.get("b").scalar_text())));
  }
  if (fn == "ResourceList.Add" || fn == "ResourceList.Sub" || fn == "ResourceList.SetMax" || fn == "ResourceList.SetMin") {
    ResourceList lhs = rl_from(req.get("lhs")), rhs = rl_from(req.get("rhs"));
    if (fn == "ResourceList.Add") RL_Add(lhs, rhs);
    else if (fn == "ResourceList.Sub") RL_Sub(lhs, rhs);
    else if (fn == "ResourceList.SetMax") RL_SetMax(lhs, rhs);
    else RL_SetMin(lhs, rhs);
    return rl_to(lhs);
  }
  if (fn == "ResourceList.GreaterOrEqual") return Value::boolean(RL_GreaterOrEqual(rl_from(req.get("lhs")), rl_from(req.get("rhs"))));
  if (fn == "ResourceList.EqualTo") return Value::boolean(RL_EqualTo(rl_from(req.get("lhs")), rl_from(req.get("rhs"))));
  if (fn == "PodRequestResourceList") return rl_to(PodRequestResourceList(pod_from(req.get("pod"))));
  if (fn == "ResourceAmountOfPod") return ra_to(ResourceAmountOfPod(pod_from(req.get("pod"))));
  if (fn == "ResourceAmount.Add") return ra_to(RA_Add(ra_from(req.get("a")), ra_from(req.get("b"))));
  if (fn == "ResourceAmount.Sub") return ra_to(RA_Sub(ra_from(req.get("a")), ra_from(req.get("b"))));
  if (fn == "ResourceAmount.IsThrottled")
    return throttled_to(RA_IsThrottled(ra_from(req.get("threshold")), ra_from(req.get("used")), req.get("onEqual").bool_or(false)));
  if (fn == "IsThrottledFor") return Value::boolean(IsThrottledFor(throttled_from(req.get("throttled")), pod_from(req.get("pod"))));
  if (fn == "ThrottleSelector.MatchesToPod" || fn == "ClusterThrottleSelector.MatchesToPod" ||
      fn == "ClusterThrottleSelector.MatchesToNamespace") {
    std::vector<SelectorTerm> terms = terms_from(req.get("selector"));
    SelectorError e;
    bool m;
    if (fn == "ThrottleSelector.MatchesToPod") m = ThrottleSelector_MatchesToPod(terms, pod_from(req.get("pod")), &e);
    else if (fn == "ClusterThrottleSelector.MatchesToPod") m = ClusterSelector_MatchesToPod(terms, pod_from(req.get("pod")), ns_from(req.get("namespace")), &e);
    else m = ClusterSelector_MatchesToNamespace(terms, ns_from(req.get("namespace")));
    Value o = Value::object();
    o.set("match", Value::boolean(m));
    if (e.failed) o.set("error", Value::str(e.msg));
    return o;
  }
  if (fn == "TemporaryThresholdOverride.IsActive") {
    TemporaryThresholdOverride ov;
    ov.begin = req.get("override").get("begin").str_or("");
    ov.end = req.get("override").get("end").str_or("");
    Time now = time_from(req.get("now"));
    if (req.get("nowOffsetSec").kind == Value::Number) now.sec += req.get("nowOffsetSec").int_or(0);
    bool active = false;
    std::string e = Override_IsActive(ov, now, &active);
    Value o = Value::object();
    o.set("active", Value::boolean(active));
    if (!e.empty()) o.set("error", Value::str(e));
    return o;
  }
  if (fn == "CalculateThreshold") {
    Throttle t = throttle_from(req.get("throttle"));
    return calc_to(CalculateThreshold(t, time_from(req.get("now"))));
  }
  if (fn == "NextOverrideHappensIn") {
    Throttle t = throttle_from(req.get("throttle"));
    __int128 d = 0;
    bool have = NextOverrideHappensIn(t, time_from(req.get("now")), &d);
    Value o = Value::object();
    o.set("have", Value::boolean(have));
    o.set("nanos", Value::number((long long)d));
    return o;
  }
  if (fn == "CheckThrottledFor") {
    Throttle t = throttle_from(req.get("throttle"));
    CheckThrottleStatus s = CheckThrottledFor(t, pod_from(req.get("pod")), ra_from(req.get("reserved")), req.get("onEqual").bool_or(false));
    return Value::str(CheckStatusName(s));
  }
  if (fn == "ParseRFC3339") {
    Time t;
    std::string e = ParseRFC3339(req.get("value").str_or(""), &t);
    Value o = Value::object();
    if (!e.empty()) o.set("error", Value::str(e));
    o.set("unix", Value::number(t.sec));
    o.set("nsec", Value::number(t.nsec));
    return o;
  }
  return err_obj("unknown fn: " + fn);
}

struct KoWorld {
  World w;
  std::vector<Throttle*> colThrottles;  // from-columns: column index -> object
  std::vector<Pod> colPending;
};

}  // namespace

extern "C" {

const char* ko_eval(const char* json) {
  try {
    return ret(eval_call(kojson::parse(json)));
  } catch (const std::exception& e) {
    return ret(err_obj(e.what()));
  }
}

void* ko_world_new(const char* throttler_name, const char* target_scheduler_name) {
  auto* k = new KoWorld();
  k->w.throttlerName = throttler_name;
  k->w.targetSchedulerName = target_scheduler_name;
  return k;
}
void ko_world_free(void* h) { delete (KoWorld*)h; }

// pod informer Delete event
const char* ko_world_delete_pod(void* h, const char* ns, const char* name) {
  try {
    ((KoWorld*)h)->w.deletePod(ns ? ns : "", name ? name : "");
    return ret(Value::object());
  } catch (const std::exception& e) {
    return ret(err_obj(e.what()));
  }
}

const char* ko_world_delete_namespace(void* h, const char* name) {
  try {
    ((KoWorld*)h)->w.deleteNamespace(name ? name : "");
    return ret(Value::object());
  } catch (const std::exception& e) {
    return ret(err_obj(e.what()));
  }
}

// throttle / clusterthrottle informer Delete event (kind 0 = Throttle, 1 = ClusterThrottle)
const char* ko_world_delete_throttle(void* h, int kind, const char* ns, const char* name) {
  try {
    ((KoWorld*)h)->w.deleteThrottle(kind != 0, ns ? ns : "", name ? name : "");
    return ret(Value::object());
  } catch (const std::exception& e) {
    return ret(err_obj(e.what()));
  }
}

// apply one manifest (kind: Pod | Namespace | Throttle | ClusterThrottle); upsert by name
const char* ko_world_apply(void* h, const char* json) {
  try {
    KoWorld* k = (KoWorld*)h;
    Value v = kojson::parse(json);
    std::string kind = v.get("kind").str_or("");
    if (kind == "Pod") k->w.applyPod(pod_from(v));
    else if (kind == "Namespace") k->w.upsertNamespace(ns_from(v));
    else if (kind == "Throttle" || kind == "ClusterThrottle") k->w.upsertThrottle(throttle_from(v), !v.get("status").is_obj());
    else return ret(err_obj("unknown kind: " + kind));
    return ret(Value::object());
  } catch (const std::exception& e) {
    return ret(err_obj(e.what()));
  }
}

const char* ko_world_reconcile_all(void* h, const char* now_rfc3339) {
  try {
    KoWorld* k = (KoWorld*)h;
    Time now;
    std::string e = ParseRFC3339(now_rfc3339, &now);
    if (!e.empty()) return ret(err_obj(e));
    e = k->w.reconcileAll(now);
    if (!e.empty()) return ret(err_obj(e));
    return ret(Value::object());
  } catch (const std::exception& e) {
    return ret(err_obj(e.what()));
  }
}

// status of a (Cluster)Throttle as JSON; ns == "" for ClusterThrottle
const char* ko_world_get_status(void* h, const char* ns, const char* name) {
  KoWorld* k = (KoWorld*)h;
  const Throttle* t = nullptr;
  if (ns[0] == 0) {
    auto it = k->w.clthrIndex.find(name);
    if (it != k->w.clthrIndex.end()) t = k->w.clusterThrottles[it->second].get();
  } else {
    auto it = k->w.thrIndex.find(std::string(ns) + "/" + name);
    if (it != k->w.thrIndex.end()) t = k->w.throttles[it->second].get();
  }
  if (!t) return ret(err_obj("not found"));
  return ret(status_to(t->status));
}

const char* ko_world_prefilter(void* h, const char* pod_json) {
  try {
    KoWorld* k = (KoWorld*)h;
    return ret(prefilter_to(k->w.PreFilter(pod_from(kojson::parse(pod_json)))));
  } catch (const std::exception& e) {
    return ret(err_obj(e.what()));
  }
}
const char* ko_world_reserve(void* h, const char* pod_json) {
  try {
    KoWorld* k = (KoWorld*)h;
    std::string e = k->w.Reserve(pod_from(kojson::parse(pod_json)));
    Value o = Value::object();
    o.set("code", Value::str(e.empty() ? "Success" : "Error"));
    if (!e.empty()) o.set("message", Value::str(e));
    return ret(o);
  } catch (const std::exception& e) {
    return ret(err_obj(e.what()));
  }
}
const char* ko_world_unreserve(void* h, const char* pod_json) {
  try {
    KoWorld* k = (KoWorld*)h;
    k->w.Unreserve(pod_from(kojson::parse(pod_json)));
    return ret(Value::object());
  } catch (const std::exception& e) {
    return ret(err_obj(e.what()));
  }
}
// reservedResourceAmount(nn) of one controller's cache
const char* ko_world_reserved(void* h, int kind, const char* thr_nn) {
  KoWorld* k = (KoWorld*)h;
  std::vector<std::string> pods;
  ResourceAmount a = (kind == 0 ? k->w.thrCache : k->w.clthrCache).reservedResourceAmount(thr_nn, &pods);
  Value o = Value::object();
  o.set("amount", ra_to(a));
  Value p = Value::array();
  for (auto& s : pods) p.push(Value::str(s));
  o.set("pods", p);
  return ret(o);
}

// ---------- columnar oracle ------------------------------------------------------------
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
  // outputs (nullable)
  kt_reconcile_out rec;
  uint32_t* run_bitmap; uint32_t* pend_bitmap; uint32_t* codes; uint8_t* admit;
};

static ColumnarInput to_input(const ko_columnar_args* a) {
  ColumnarInput in;
  in.lim = a->lim;
  in.running = PodCols{a->n_running, a->run_labels, a->run_req, a->run_present, a->run_flags, a->run_ns};
  in.pending = PodCols{a->n_pending, a->pend_labels, a->pend_req, a->pend_present, a->pend_flags, a->pend_ns};
  in.n_ns = a->n_ns;
  in.ns_labels = a->ns_labels;
  in.m = a->m;
  in.thr = *a->thr;
  in.sel = *a->sel;
  in.status = a->status;
  in.reserved = a->reserved;
  in.reserved_present = a->reserved_present;
  in.reserved_cnt = a->reserved_cnt;
  in.now = a->now;
  in.flags = a->flags;
  in.words_per_row = a->words_per_row;
  return in;
}

int ko_columnar_evaluate(const ko_columnar_args* a) {
  ColumnarInput in = to_input(a);
  ColumnarOutput out;
  out.rec = a->rec;
  out.run_bitmap = a->run_bitmap;
  out.pend_bitmap = a->pend_bitmap;
  out.codes = a->codes;
  out.admit = a->admit;
  return columnar_evaluate(in, out);
}

// columnar_admit_queue: a->codes / admit / pend_bitmap receive the pending rows (each nullable), res* the final reservations.
int ko_columnar_admit_queue(const ko_columnar_args* a, int64_t first, int64_t count, int64_t* res, uint32_t* res_present, int64_t* res_cnt,
                            int64_t* admitted) {
  ColumnarInput in = to_input(a);
  ColumnarOutput out;
  out.rec = kt_reconcile_out{};
  out.pend_bitmap = a->pend_bitmap;
  out.codes = a->codes;
  out.admit = a->admit;
  const int64_t n = columnar_admit_queue(in, first, count, out, res, res_present, res_cnt);
  if (n < 0) return -1;
  *admitted = n;
  return 0;
}

// ---------- object World from columns -------------------------------------------------
// Names: label key "k<id>", value "v<id>", namespace "ns<id>", resource "r<i>", throttles "t<idx>".
// Column integers become whole-unit Quantities (any common scale gives identical decisions).
static LabelMap labels_of(const int64_t* labels, int64_t stride, int64_t row, int slots) {
  LabelMap m;
  for (int i = 0; i < slots; ++i) {
    int64_t l = labels[(int64_t)i * stride + row];
    if (l == KT_LABEL_EMPTY) continue;
    m["k" + std::to_string((uint32_t)((uint64_t)l >> 32))] = "v" + std::to_string((uint32_t)((uint64_t)l & 0xffffffffu));
  }
  return m;
}
static Quantity q_of(int64_t v) { Quantity q; q.nano = (i128)v * 1000000000; return q; }
static ResourceAmount amount_of(const int64_t* vals, int64_t stride, int64_t idx, uint32_t present, int64_t cnt, int R) {
  ResourceAmount a;
  if (present & KT_COUNT_BIT) { a.hasCounts = true; a.pod = cnt; }
  for (int r = 0; r < R; ++r)
    if ((present >> r) & 1) { a.requestsNil = false; a.requests["r" + std::to_string(r)] = q_of(vals[(int64_t)r * stride + idx]); }
  return a;
}
static Pod pod_of(const PodCols& c, int64_t p, int L, int R, const char* prefix, const std::string& sched) {
  Pod pod;
  pod.ns = "ns" + std::to_string(c.ns_id[p]);
  pod.name = std::string(prefix) + std::to_string(p);
  pod.labels = labels_of(c.labels, c.n, p, L);
  uint32_t f = c.flags[p];
  pod.schedulerName = (f & KT_POD_SCHEDULER_MATCH) ? sched : "other-scheduler";
  pod.nodeName = (f & KT_POD_SCHEDULED) ? "node" : "";
  pod.phase = (f & KT_POD_NOT_FINISHED) ? "Running" : "Succeeded";
  Container ctr;
  for (int r = 0; r < R; ++r)
    if ((c.present[p] >> r) & 1) ctr.requests["r" + std::to_string(r)] = q_of(c.req[(int64_t)r * c.n + p]);
  pod.containers.push_back(std::move(ctr));
  return pod;
}
static LabelSelector selector_of(const kt_selector_table& s, int32_t q0, int32_t q1) {
  LabelSelector ls;
  for (int32_t q = q0; q < q1; ++q) {
    LabelSelectorRequirement r;
    r.key = "k" + std::to_string(s.req_key[q]);
    switch (s.req_op[q]) {
      case KT_OP_IN: r.op = "In"; break;
      case KT_OP_NOTIN: r.op = "NotIn"; break;
      case KT_OP_EXISTS: r.op = "Exists"; break;
      default: r.op = "DoesNotExist";
    }
    for (int32_t v = s.req_val_off[q]; v < s.req_val_off[q + 1]; ++v) r.values.push_back("v" + std::to_string(s.req_vals[v]));
    ls.matchExpressions.push_back(std::move(r));
  }
  return ls;
}

void* ko_world_from_columns(const ko_columnar_args* a) {
  ColumnarInput in = to_input(a);
  const int R = in.lim.n_resources, L = in.lim.label_slots;
  auto* k = new KoWorld();
  k->w.throttlerName = "kube-throttler";
  k->w.targetSchedulerName = "my-scheduler";
  for (int32_t n = 0; n < in.n_ns; ++n) {
    Namespace ns;
    ns.name = "ns" + std::to_string(n);
    ns.labels = labels_of(in.ns_labels, in.n_ns, n, in.lim.ns_label_slots);
    k->w.upsertNamespace(std::move(ns));
  }
  for (int64_t p = 0; p < in.running.n; ++p) k->w.upsertPod(pod_of(in.running, p, L, R, "run", k->w.targetSchedulerName));
  for (int64_t p = 0; p < in.pending.n; ++p) k->colPending.push_back(pod_of(in.pending, p, L, R, "pend", k->w.targetSchedulerName));
  const bool given = in.flags & KT_EVAL_GIVEN_STATUS;
  for (int32_t t = 0; t < in.m; ++t) {
    Throttle thr;
    thr.kind = in.thr.kind[t] == KT_KIND_THROTTLE ? KindThrottle : KindClusterThrottle;
    thr.ns = thr.kind == KindThrottle ? "ns" + std::to_string(in.thr.ns_id[t]) : "";
    thr.name = "t" + std::to_string(t);
    thr.throttlerName = (in.thr.flags[t] & KT_THR_RESPONSIBLE) ? k->w.throttlerName : "somebody-else";
    thr.threshold = amount_of(in.thr.thr, in.m, t, in.thr.thr_present[t], in.thr.thr_cnt[t], R);
    for (int32_t i = in.thr.ovr_off[t]; i < in.thr.ovr_off[t + 1]; ++i) {
      TemporaryThresholdOverride ov;
      // encode the instants back to RFC3339 is unnecessary: begin/end are compared as instants; we
      // emit unix-second strings the oracle parser does not accept, so instead store as RFC3339 UTC.
      auto fmt = [](int64_t ns, bool open) -> std::string {
        if (open) return "";
        int64_t sec = ns / 1000000000, rem = ns % 1000000000;
        if (rem < 0) { rem += 1000000000; sec -= 1; }
        int64_t days = sec / 86400, sod = sec % 86400;
        if (sod < 0) { sod += 86400; days -= 1; }
        // civil_from_days
        int64_t z = days + 719468;
        int64_t era = (z >= 0 ? z : z - 146096) / 146097;
        unsigned doe = (unsigned)(z - era * 146097);
        unsigned yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
        int64_t y = (int64_t)yoe + era * 400;
        unsigned doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
        unsigned mp = (5 * doy + 2) / 153;
        unsigned d = doy - (153 * mp + 2) / 5 + 1;
        unsigned mth = mp < 10 ? mp + 3 : mp - 9;
        if (mth <= 2) y += 1;
        char buf[64];
        std::snprintf(buf, sizeof buf, "%04lld-%02u-%02uT%02d:%02d:%02d.%09lldZ", (long long)y, mth, d, (int)(sod / 3600), (int)(sod % 3600 / 60),
                      (int)(sod % 60), (long long)rem);
        return buf;
      };
      ov.begin = (in.thr.ovr_flags[i] & KT_OVR_PARSE_ERROR) ? "not-a-time" : fmt(in.thr.ovr_begin[i], in.thr.ovr_begin[i] == KT_TIME_OPEN_BEGIN);
      ov.end = fmt(in.thr.ovr_end[i], in.thr.ovr_end[i] == KT_TIME_OPEN_END);
      ov.threshold = amount_of(in.thr.ovr_thr, in.thr.n_ovr, i, in.thr.ovr_present[i], in.thr.ovr_cnt[i], R);
      thr.overrides.push_back(std::move(ov));
    }
    for (int32_t term = in.sel.term_off[t]; term < in.sel.term_off[t + 1]; ++term) {
      SelectorTerm st;
      st.podSelector = selector_of(in.sel, in.sel.pod_req_off[term], in.sel.pod_req_off[term + 1]);
      st.namespaceSelector = selector_of(in.sel, in.sel.ns_req_off[term], in.sel.ns_req_off[term + 1]);
      if (in.sel.term_flags[term] & KT_TERM_NS_INVALID) st.namespaceSelector.matchExpressions.push_back({"k0", "BogusOperator", {}});
      thr.terms.push_back(std::move(st));
    }
    if (in.thr.flags[t] & KT_THR_SELECTOR_ERROR) {
      if (thr.terms.empty()) thr.terms.emplace_back();
      thr.terms[0].podSelector.matchExpressions.push_back({"k0", "BogusOperator", {}});
    }
    if (given && in.status) {
      const kt_status_cols& s = *in.status;
      thr.status.calculatedThreshold.calculatedAtSet = s.calculated[t];
      if (s.calculated[t]) thr.status.calculatedThreshold.calculatedAt.sec = 1;
      thr.status.calculatedThreshold.threshold = amount_of(s.calc_thr, in.m, t, s.calc_present[t], s.calc_cnt[t], R);
      thr.status.used = amount_of(s.used, in.m, t, s.used_present[t], s.used_cnt[t], R);
      thr.status.throttled.pod = s.throttled[t] & KT_COUNT_BIT;
      for (int r = 0; r < R; ++r)
        if ((s.throttled[t] >> r) & 1) { thr.status.throttled.requestsNil = false; thr.status.throttled.requests["r" + std::to_string(r)] = true; }
    }
    // reservation cache: one synthetic reserved pod per throttle carrying the column totals
    uint32_t rp = in.reserved_present ? in.reserved_present[t] : 0;
    k->w.upsertThrottle(std::move(thr));
    Throttle* stored = in.thr.kind[t] == KT_KIND_THROTTLE ? k->w.throttles.back().get() : k->w.clusterThrottles.back().get();
    k->colThrottles.push_back(stored);
    if (rp) {
      ResourceAmount ra = amount_of(in.reserved, in.m, t, rp, in.reserved_cnt ? in.reserved_cnt[t] : 0, R);
      auto& cache = stored->kind == KindThrottle ? k->w.thrCache : k->w.clthrCache;
      cache.cache[stored->NN()]["reserved/synthetic"] = ra;
    }
  }
  return k;
}

// Worker i of a timed run sits on its own CPU (the i-th of the process's affinity mask, wrapping): without it the same
// code measured 1e8 .. 3e8 checks/s from run to run on a 128-thread host (threads migrating, two on one core).
static void pin_worker(int i) {
#ifdef __linux__
  cpu_set_t all;
  CPU_ZERO(&all);
  if (sched_getaffinity(0, sizeof all, &all) != 0) return;
  const int n = CPU_COUNT(&all);
  if (n <= 0) return;
  int want = i % n, cpu = -1;
  for (int c = 0; c < CPU_SETSIZE; ++c)
    if (CPU_ISSET(c, &all) && want-- == 0) { cpu = c; break; }
  if (cpu < 0) return;
  cpu_set_t one;
  CPU_ZERO(&one);
  CPU_SET(cpu, &one);
  pthread_setaffinity_np(pthread_self(), sizeof one, &one);
#else
  (void)i;
#endif
}

// Run the reference-shaped path on a from-columns world and emit the engine's output layout.
//   threads   : worker threads (reconcile over throttles, PreFilter over pending pods)
//   max_pending / max_reconcile : bounded sample (<=0 => all)
// Returns elapsed seconds of the timed region (reconcile + checks), or <0 on error.
double ko_world_run_columns(void* h, const ko_columnar_args* a, int threads, int64_t max_pending, int32_t max_reconcile,
                            double* reconcile_seconds, double* check_seconds) {
  KoWorld* k = (KoWorld*)h;
  ColumnarInput in = to_input(a);
  const int R = in.lim.n_resources;
  const int32_t M = in.m, W = in.words_per_row;
  int64_t P = (int64_t)k->colPending.size();
  if (max_pending > 0 && max_pending < P) P = max_pending;
  int32_t MR = M;
  if (max_reconcile > 0 && max_reconcile < MR) MR = max_reconcile;
  if (threads < 1) threads = 1;
  Time now;
  {
    int64_t sec = in.now / 1000000000, rem = in.now % 1000000000;
    if (rem < 0) { rem += 1000000000; sec -= 1; }
    now.sec = sec; now.nsec = (int)rem;
  }
  std::atomic<bool> failed{false};
  auto t0 = std::chrono::steady_clock::now();
  if (!(in.flags & KT_EVAL_SKIP_RECONCILE) && !(in.flags & KT_EVAL_GIVEN_STATUS)) {
    // The reservation cache is only touched by unreserve; serialise that like keyMutex does.
    std::atomic<int32_t> next{0};
    std::mutex mu;
    auto worker = [&]() {
      while (true) {
        int32_t t = next.fetch_add(1);
        if (t >= MR) break;
        Throttle& thr = *k->colThrottles[t];
        if (!k->w.isResponsibleFor(thr)) continue;
        std::vector<const Pod*> nonterm, term;
        std::string e = k->w.affectedPods(thr, &nonterm, &term);
        if (!e.empty()) continue;  // selector error: reconcile returns err, status untouched
        ResourceAmount used;
        for (const Pod* p : nonterm) used = RA_Add(used, ResourceAmountOfPod(*p));
        ThrottleStatus ns = thr.status;
        ns.used = used;
        CalculatedThreshold calc = CalculateThreshold(thr, now);
        if (!RA_SemanticEqual(thr.status.calculatedThreshold.threshold, calc.threshold) || thr.status.calculatedThreshold.messages != calc.messages)
          ns.calculatedThreshold = calc;
        ns.throttled = RA_IsThrottled(ns.calculatedThreshold.threshold, ns.used, true);
        thr.status = ns;
        (void)mu;  // synthetic reservations are not pods of the snapshot: nothing to un-reserve
      }
    };
    std::vector<std::thread> th;
    for (int i = 0; i < threads; ++i) th.emplace_back([&, i]() { pin_worker(i); worker(); });
    for (auto& x : th) x.join();
  }
  auto t1 = std::chrono::steady_clock::now();
  if (!(in.flags & KT_EVAL_SKIP_CHECK)) {
    std::unordered_map<const Throttle*, int32_t> idx;
    for (int32_t t = 0; t < M; ++t) idx[k->colThrottles[t]] = t;
    if (a->pend_bitmap) std::memset(a->pend_bitmap, 0, sizeof(uint32_t) * (size_t)P * W);
    if (a->codes) std::memset(a->codes, 0, sizeof(uint32_t) * (size_t)P * 2 * W);
    std::atomic<int64_t> next{0};
    auto worker = [&]() {
      while (true) {
        int64_t p = next.fetch_add(1);
        if (p >= P) break;
        PreFilterResult r = k->w.PreFilter(k->colPending[p], (in.flags & KT_EVAL_ON_EQUAL) != 0);
        if (r.code == "Error") {
          // engine convention: a throttle with a selector error never matches; redo the two halves tolerantly
          if (a->admit) a->admit[p] = 1;
          failed = true;
          continue;
        }
        auto mark = [&](const std::vector<const Throttle*>& v, uint32_t code) {
          for (auto* t : v) {
            int32_t ti = idx[t];
            if (a->codes) a->codes[(size_t)p * 2 * W + (ti >> 4)] |= code << (2 * (ti & 15));
          }
        };
        for (const CheckResult* cr : {&r.thr, &r.clthr}) {
          for (auto* t : cr->affected) {
            int32_t ti = idx[t];
            if (a->pend_bitmap) a->pend_bitmap[(size_t)p * W + (ti >> 5)] |= 1u << (ti & 31);
          }
          mark(cr->active, KT_CHECK_ACTIVE);
          mark(cr->insufficient, KT_CHECK_INSUFFICIENT);
          mark(cr->exceeds, KT_CHECK_POD_REQUESTS_EXCEEDS_THRESHOLD);
        }
        if (a->admit) a->admit[p] = r.code == "Success";
      }
    };
    std::vector<std::thread> th;
    for (int i = 0; i < threads; ++i) th.emplace_back([&, i]() { pin_worker(i); worker(); });
    for (auto& x : th) x.join();
  }
  auto t2 = std::chrono::steady_clock::now();
  // reconcile outputs in the engine's layout
  for (int32_t t = 0; t < MR; ++t) {
    const Throttle& thr = *k->colThrottles[t];
    const ThrottleStatus& s = thr.status;
    auto put = [&](const ResourceAmount& ra, int64_t* vals, uint32_t* present, int64_t* cnt) {
      uint32_t pm = ra.hasCounts ? KT_COUNT_BIT : 0;
      for (int r = 0; r < R; ++r) {
        auto it = ra.requests.find("r" + std::to_string(r));
        int64_t v = 0;
        if (it != ra.requests.end()) { pm |= 1u << r; v = (int64_t)(it->second.nano / 1000000000); }
        if (vals) vals[(int64_t)r * M + t] = v;
      }
      if (present) present[t] = pm;
      if (cnt) cnt[t] = ra.hasCounts ? ra.pod : 0;
    };
    put(s.used, a->rec.used, a->rec.used_present, a->rec.used_cnt);
    put(s.calculatedThreshold.threshold, a->rec.calc_thr, a->rec.calc_present, a->rec.calc_cnt);
    if (a->rec.throttled) {
      uint32_t m = s.throttled.pod ? KT_COUNT_BIT : 0;
      for (int r = 0; r < R; ++r) {
        auto it = s.throttled.requests.find("r" + std::to_string(r));
        if (it != s.throttled.requests.end() && it->second) m |= 1u << r;
      }
      a->rec.throttled[t] = m;
    }
  }
  double rs = std::chrono::duration<double>(t1 - t0).count(), cs = std::chrono::duration<double>(t2 - t1).count();
  if (reconcile_seconds) *reconcile_seconds = rs;
  if (check_seconds) *check_seconds = cs;
  return failed ? -(rs + cs) - 1e-9 : rs + cs;
}

int ko_hardware_threads(void) { return (int)std::thread::hardware_concurrency(); }

}  // extern "C"
