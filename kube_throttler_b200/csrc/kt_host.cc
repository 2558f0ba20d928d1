// kt_host.cc -- the plugin surface (NewPlugin / PreFilter / Reserve / Unreserve) and both controllers'
// bookkeeping of everpeace/kube-throttler restated above the device engine (include/kt_host.h).
//
// Shape: the informer caches are kept COLUMN-first.  A pod is parsed once per event into its packed row
// (dictionary-encoded labels, ResourceAmountOfPod as exact quantities); rows live in a slotted table that
// mirrors the device columns one to one, so an informer event is a row scatter (kt_update_pod_rows) and a
// pass never rebuilds anything.  Throttles / namespaces are small and re-uploaded whole when they change.
// Nothing in this file decides whether a pod matches a selector or compares a quantity with a threshold:
// that is the device's job (kt_evaluate); this file packs, calls, and spells the results.
#include <algorithm>
#include <charconv>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/kt_b200.h"
#include "../../include/kt_host.h"
#include "kt_json.h"
#include "kt_quantity.h"

namespace {

using ktjson::Node;
using ktjson::Writer;
using kt::Quantity;

// ---- dictionaries --------------------------------------------------------------------------------
struct Dict {
  std::unordered_map<std::string, uint32_t> ids;
  std::vector<std::string> names;
  uint32_t id(const std::string& s) {
    auto it = ids.find(s);
    if (it != ids.end()) return it->second;
    const uint32_t v = (uint32_t)names.size();
    ids.emplace(s, v);
    names.push_back(s);
    return v;
  }
  int find(const std::string& s) const {
    auto it = ids.find(s);
    return it == ids.end() ? -1 : (int)it->second;
  }
  size_t size() const { return names.size(); }
};

// The label dictionaries hold what SELECTORS mention and nothing else: label keys share one id space (podSelector and
// namespaceSelector keys), values are numbered per key, so the ids are dense in both dimensions and the device takes its direct
// key / value tables (kt_tables.cc).  Pods and namespaces are encoded THROUGH them: a label whose key no selector mentions cannot
// influence any match and is dropped; a mentioned key with a value no requirement names becomes "some other value" (id 0 of every
// key -- In / NotIn never name it, Exists / DoesNotExist only look at the key).  A scheduler that lives for months sees an unbounded
// stream of label values (pod-template-hash, controller-uid, job-name): interning those grew the dictionaries, and the device's
// value tables, with every pod ever seen.  When a new throttle brings new vocabulary, the rows that carry it are packed again.
const char* const kOtherValue = "\x01other";  // not a legal label value: cannot collide with a real one
struct LabelDict {
  Dict keys;
  std::vector<Dict> vals;
  uint32_t key_id(const std::string& k, bool* added = nullptr) {
    const size_t n = keys.size();
    const uint32_t kid = keys.id(k);
    if (vals.size() <= kid) vals.resize(kid + 1);
    if (vals[kid].size() == 0) vals[kid].id(kOtherValue);
    if (added) *added = keys.size() != n;
    return kid;
  }
  uint32_t value_id(uint32_t kid, const std::string& v, bool* added = nullptr) {
    const size_t n = vals[kid].size();
    const uint32_t vid = vals[kid].id(v);
    if (added) *added = vals[kid].size() != n;
    return vid;
  }
  int64_t encode(const std::string& k, const std::string& v) const {  // KT_LABEL_EMPTY: no selector can see this label
    const int kid = keys.find(k);
    if (kid < 0) return KT_LABEL_EMPTY;
    const int vid = vals[(size_t)kid].find(v);
    return (int64_t)(((uint64_t)kid << 32) | (uint32_t)(vid < 0 ? 0 : vid));
  }
  size_t n_values() const {
    size_t n = 0;
    for (auto& d : vals) n += d.size();
    return n;
  }
};

// ---- time: time.Parse(time.RFC3339, s) with Go's error texts ---------------------------------------
struct GoTime {
  long long sec = 0;  // unix seconds
  int nsec = 0;
  bool zero = true;   // time.Time{} (year 1): "not set"
  __int128 ns() const { return (__int128)sec * 1000000000 + nsec; }
};
long long days_from_civil(long long y, unsigned m, unsigned d) {
  y -= m <= 2;
  const long long era = (y >= 0 ? y : y - 399) / 400;
  const unsigned yoe = (unsigned)(y - era * 400);
  const unsigned doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
  const unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + (long long)doe - 719468;
}
// metav1.Time marshals as UTC RFC3339 with second precision ("2006-01-02T15:04:05Z")
std::string format_rfc3339_utc(long long unix_sec) {
  long long days = unix_sec >= 0 ? unix_sec / 86400 : -((-unix_sec + 86399) / 86400);
  const long long rem = unix_sec - days * 86400;
  days += 719468;  // civil_from_days (H. Hinnant), the inverse of days_from_civil above
  const long long era = (days >= 0 ? days : days - 146096) / 146097;
  const unsigned doe = (unsigned)(days - era * 146097);
  const unsigned yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  long long y = (long long)yoe + era * 400;
  const unsigned doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const unsigned mp = (5 * doy + 2) / 153;
  const unsigned d = doy - (153 * mp + 2) / 5 + 1;
  const unsigned m = mp < 10 ? mp + 3 : mp - 9;
  y += m <= 2;
  char buf[64];
  std::snprintf(buf, sizeof buf, "%04lld-%02u-%02uT%02d:%02d:%02dZ", y, m, d, (int)(rem / 3600), (int)(rem % 3600 / 60), (int)(rem % 60));
  return buf;
}
// Layout-driven: the RFC3339 layout "2006-01-02T15:04:05Z07:00" is a list of chunks; the first chunk that
// fails to parse produces `cannot parse "<rest>" as "<chunk>"` exactly as time.Parse reports it.
std::string parse_rfc3339(const std::string& value, GoTime* out) {
  static const char* kLayout = "2006-01-02T15:04:05Z07:00";
  struct Chunk { const char* text; int digits; };  // digits > 0: fixed-width number; 0: literal
  static const Chunk chunks[] = {{"2006", 4}, {"-", 0}, {"01", 2}, {"-", 0}, {"02", 2}, {"T", 0}, {"15", 2}, {":", 0}, {"04", 2}, {":", 0}, {"05", 2}};
  int field[6] = {0, 0, 0, 0, 0, 0};
  int nf = 0;
  size_t p = 0;
  auto bad = [&](size_t at, const char* elem) {
    return "parsing time \"" + value + "\" as \"" + kLayout + "\": cannot parse \"" + value.substr(std::min(at, value.size())) + "\" as \"" + elem + "\"";
  };
  auto out_of_range = [&](const char* what) { return "parsing time \"" + value + "\": " + what + " out of range"; };
  for (const Chunk& c : chunks) {
    if (c.digits == 0) {
      if (p >= value.size() || value[p] != c.text[0]) return bad(p, c.text);
      ++p;
      continue;
    }
    if (p + c.digits > value.size()) return bad(p, c.text);
    int v = 0;
    for (int i = 0; i < c.digits; ++i) {
      const char ch = value[p + i];
      if (ch < '0' || ch > '9') return bad(p, c.text);
      v = v * 10 + (ch - '0');
    }
    p += c.digits;
    field[nf++] = v;
    if (nf == 2 && (v < 1 || v > 12)) return out_of_range("month");
    if (nf == 4 && v >= 24) return out_of_range("hour");
    if (nf == 5 && v >= 60) return out_of_range("minute");
    if (nf == 6 && v >= 60) return out_of_range("second");
  }
  int nsec = 0;
  if (p + 1 < value.size() && (value[p] == '.' || value[p] == ',') && value[p + 1] >= '0' && value[p + 1] <= '9') {
    ++p;
    int nd = 0;
    long long frac = 0;
    while (p < value.size() && value[p] >= '0' && value[p] <= '9') {
      if (nd < 9) { frac = frac * 10 + (value[p] - '0'); ++nd; }
      ++p;
    }
    for (; nd < 9; ++nd) frac *= 10;
    nsec = (int)frac;
  }
  long long offset = 0;
  const size_t zone_at = p;
  if (p < value.size() && value[p] == 'Z') {
    ++p;
  } else if (p < value.size() && (value[p] == '+' || value[p] == '-')) {
    const int sign = value[p] == '-' ? -1 : 1;
    auto two = [&](size_t at, int* v) {
      if (at + 2 > value.size() || value[at] < '0' || value[at] > '9' || value[at + 1] < '0' || value[at + 1] > '9') return false;
      *v = (value[at] - '0') * 10 + (value[at + 1] - '0');
      return true;
    };
    int oh = 0, om = 0;
    if (!two(p + 1, &oh) || p + 3 >= value.size() || value[p + 3] != ':' || !two(p + 4, &om)) return bad(zone_at, "Z07:00");
    p += 6;
    if (oh > 24) return out_of_range("time zone offset hour");
    if (om > 60) return out_of_range("time zone offset minute");
    offset = sign * (oh * 3600LL + om * 60LL);
  } else {
    return bad(zone_at, "Z07:00");
  }
  if (p != value.size()) return "parsing time \"" + value + "\": extra text: \"" + value.substr(p) + "\"";
  const int Y = field[0], M = field[1], D = field[2];
  static const int mdays[] = {31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
  const bool leap = (Y % 4 == 0 && Y % 100 != 0) || Y % 400 == 0;
  if (D < 1 || D > mdays[M - 1] + (M == 2 && leap ? 1 : 0)) return out_of_range("day");
  out->sec = days_from_civil(Y, (unsigned)M, (unsigned)D) * 86400LL + field[3] * 3600LL + field[4] * 60LL + field[5] - offset;
  out->nsec = nsec;
  out->zero = false;
  return "";
}
int64_t clamp_ns(__int128 v) {
  const __int128 lo = (__int128)INT64_MIN + 1, hi = (__int128)INT64_MAX - 1;
  return (int64_t)(v < lo ? lo : (v > hi ? hi : v));
}

// ---- label selector validation (metav1.LabelSelectorAsSelector -> labels.NewRequirement) -----------
// The messages are the ones a scheduler operator reads in the PreFilter Error status, so they are restated in full:
// k8s.io/apimachinery v0.26.4 pkg/labels/selector.go (NewRequirement, validateLabelKey/Value), pkg/util/validation
// (IsQualifiedName, IsDNS1123Subdomain, IsValidLabelValue, RegexError), pkg/util/validation/field (Invalid: %q / %#v of the
// value) and pkg/util/errors (aggregate: "[a, b]", duplicates dropped).  No reference test pins them.
bool is_alnum(char c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); }
bool qualified_name_re(const std::string& s) {  // ([A-Za-z0-9][-A-Za-z0-9_.]*)?[A-Za-z0-9]
  if (s.empty() || !is_alnum(s.front()) || !is_alnum(s.back())) return false;
  for (char c : s)
    if (!is_alnum(c) && c != '-' && c != '_' && c != '.') return false;
  return true;
}
bool dns1123_subdomain_re(const std::string& s) {  // [a-z0-9]([-a-z0-9]*[a-z0-9])?(\.[a-z0-9]([-a-z0-9]*[a-z0-9])?)*
  if (s.empty()) return false;
  size_t b = 0;
  while (true) {
    size_t e = s.find('.', b);
    const std::string lab = s.substr(b, e == std::string::npos ? std::string::npos : e - b);
    if (lab.empty()) return false;
    auto low = [](char c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'z'); };
    if (!low(lab.front()) || !low(lab.back())) return false;
    for (char c : lab)
      if (!low(c) && c != '-') return false;
    if (e == std::string::npos) return true;
    b = e + 1;
  }
}
std::string regex_error(const std::string& msg, const std::string& fmt, std::initializer_list<const char*> examples) {  // validation.RegexError
  std::string out = msg + " (e.g. ";
  bool first = true;
  for (const char* ex : examples) {
    if (!first) out += " or ";
    first = false;
    out += std::string("'") + ex + "', ";
  }
  return out + "regex used for validation is '" + fmt + "')";
}
const char* kQualifiedNameMsg = "must consist of alphanumeric characters, '-', '_' or '.', and must start and end with an alphanumeric character";
const char* kQualifiedNameFmt = "([A-Za-z0-9][-A-Za-z0-9_.]*)?[A-Za-z0-9]";
std::vector<std::string> is_qualified_name(const std::string& value) {  // validation.IsQualifiedName
  std::vector<std::string> errs;
  std::string name = value;
  const size_t slash = value.find('/');
  if (slash != std::string::npos) {
    if (value.find('/', slash + 1) != std::string::npos)
      return {"a qualified name " + regex_error(kQualifiedNameMsg, kQualifiedNameFmt, {"MyName", "my.name", "123-abc"}) +
              " with an optional DNS subdomain prefix and '/' (e.g. 'example.com/MyName')"};
    const std::string prefix = value.substr(0, slash);
    name = value.substr(slash + 1);
    if (prefix.empty()) errs.push_back("prefix part must be non-empty");
    else {
      if (prefix.size() > 253) errs.push_back("prefix part must be no more than 253 characters");
      if (!dns1123_subdomain_re(prefix))
        errs.push_back("prefix part " + regex_error("a lowercase RFC 1123 subdomain must consist of lower case alphanumeric characters, '-' or '.', and must start and end with an alphanumeric character",
                                                    "[a-z0-9]([-a-z0-9]*[a-z0-9])?(\\.[a-z0-9]([-a-z0-9]*[a-z0-9])?)*", {"example.com"}));
    }
  }
  if (name.empty()) errs.push_back("name part must be non-empty");
  else if (name.size() > 63) errs.push_back("name part must be no more than 63 characters");
  if (!qualified_name_re(name)) errs.push_back("name part " + regex_error(kQualifiedNameMsg, kQualifiedNameFmt, {"MyName", "my.name", "123-abc"}));
  return errs;
}
std::vector<std::string> is_valid_label_value(const std::string& v) {  // validation.IsValidLabelValue
  std::vector<std::string> errs;
  if (v.size() > 63) errs.push_back("must be no more than 63 characters");
  if (!v.empty() && !qualified_name_re(v))
    errs.push_back(regex_error("a valid label must be an empty string or consist of alphanumeric characters, '-', '_' or '.', and must start and end with an alphanumeric character",
                               "(([A-Za-z0-9][-A-Za-z0-9_.]*)?[A-Za-z0-9])?", {"MyValue", "my_value", "12345"}));
  return errs;
}
std::string go_quote(const std::string& v) {  // %q
  std::string o = "\"";
  for (unsigned char c : v) {
    if (c == '"') o += "\\\"";
    else if (c == '\\') o += "\\\\";
    else if (c == '\n') o += "\\n";
    else if (c == '\t') o += "\\t";
    else if (c == '\r') o += "\\r";
    else if (c < 0x20 || c == 0x7f) { char b[8]; std::snprintf(b, sizeof b, "\\x%02x", c); o += b; }
    else o += (char)c;
  }
  return o + "\"";
}
std::string go_sharp_v(const std::vector<std::string>& vals) {  // %#v of a []string
  if (vals.empty()) return "[]string(nil)";
  std::string o = "[]string{";
  for (size_t i = 0; i < vals.size(); ++i) o += (i ? ", " : "") + go_quote(vals[i]);
  return o + "}";
}
std::string join(const std::vector<std::string>& v, const char* sep) {
  std::string o;
  for (size_t i = 0; i < v.size(); ++i) o += (i ? sep : "") + v[i];
  return o;
}
// labels.NewRequirement's error for one requirement ("" when it is fine): every complaint, key first, aggregated
std::string requirement_error(const std::string& key, uint8_t op, bool equals, const std::vector<std::string>& vals) {
  std::vector<std::string> all;
  auto add = [&](const std::string& m) { if (std::find(all.begin(), all.end(), m) == all.end()) all.push_back(m); };
  std::vector<std::string> e = is_qualified_name(key);
  if (!e.empty()) add("key: Invalid value: " + go_quote(key) + ": " + join(e, "; "));
  if (!equals && (op == KT_OP_IN || op == KT_OP_NOTIN) && vals.empty())
    add("values: Invalid value: " + go_sharp_v(vals) + ": for 'in', 'notin' operators, values set can't be empty");
  if ((op == KT_OP_EXISTS || op == KT_OP_DOESNOTEXIST) && !vals.empty())
    add("values: Invalid value: " + go_sharp_v(vals) + ": values set must be empty for exists and does not exist");
  for (size_t i = 0; i < vals.size(); ++i) {
    e = is_valid_label_value(vals[i]);
    if (!e.empty()) add("values[" + std::to_string(i) + "][" + key + "]: Invalid value: " + go_quote(vals[i]) + ": " + join(e, "; "));
  }
  if (all.empty()) return "";
  return all.size() == 1 ? all[0] : "[" + join(all, ", ") + "]";
}

struct Requirement {
  std::string key;
  uint8_t op = KT_OP_IN;
  std::vector<std::string> values;
};
struct CompiledSelector {
  std::vector<Requirement> reqs;  // empty => Everything
  std::string error;              // non-empty => LabelSelectorAsSelector failed
};
CompiledSelector compile_selector(const Node& sel) {
  CompiledSelector out;
  if (!sel.is(Node::Obj)) return out;
  auto add = [&](const std::string& key, const std::string& opname, std::vector<std::string> values, bool equals) {
    if (!out.error.empty()) return;
    Requirement r;
    r.key = key;
    if (opname == "In") r.op = KT_OP_IN;
    else if (opname == "NotIn") r.op = KT_OP_NOTIN;
    else if (opname == "Exists") r.op = KT_OP_EXISTS;
    else if (opname == "DoesNotExist") r.op = KT_OP_DOESNOTEXIST;
    else { out.error = go_quote(opname) + " is not a valid label selector operator"; return; }
    out.error = requirement_error(key, r.op, equals, values);
    if (!out.error.empty()) return;
    r.values = std::move(values);
    out.reqs.push_back(std::move(r));
  };
  // matchLabels first, keys sorted (LabelSelectorAsSelector iterates a sorted key list), then matchExpressions in order
  std::map<std::string, std::string> ml;
  for (auto& kv : sel["matchLabels"].obj) ml[kv.first] = kv.second->str();
  for (auto& kv : ml) add(kv.first, "In", {kv.second}, true);  // selection.Equals: exactly one value
  for (auto& e : sel["matchExpressions"].arr) {
    std::vector<std::string> vals;
    for (auto& v : (*e)["values"].arr) vals.push_back(v->str());
    add((*e)["key"].str(), (*e)["operator"].str(), std::move(vals), false);
  }
  if (!out.error.empty()) out.reqs.clear();
  return out;
}

// ---- objects ----------------------------------------------------------------------------------------
struct ResAmount {  // ResourceAmount with exact quantities, keyed by resource column id
  bool has_counts = false;
  long long pod = 0;
  std::map<int, Quantity> requests;  // key present <=> Go map has the key
  bool requests_nil = true;
};

struct PodObj {
  std::string ns, name;
  std::vector<std::pair<std::string, std::string>> labels;
  std::string scheduler_name, node_name, phase;
  std::map<int, Quantity> request;  // PodRequestResourceList (resource id -> quantity); ResourceAmountOfPod adds Counts{1}
  int64_t row = -1;                 // slot in the running-pod table
  int64_t pend_row = -1;            // slot in the resident scheduling-queue table (pods that are ours to schedule and not bound yet)
  uint64_t seq = 0;                 // order of first appearance (the informer-cache order the oracle iterates in; Q8)
  bool live = false;
  std::string nn() const { return ns + "/" + name; }
};

struct Override {
  std::string begin, end;
  ResAmount threshold;
};
struct Term {
  CompiledSelector pod_sel, ns_sel;
};
struct ThrottleObj {
  int kind = KT_KIND_THROTTLE;
  std::string ns, name, uid, throttler_name;
  ResAmount threshold;
  std::vector<Override> overrides;
  std::vector<Term> terms;
  // status (the informer copy; reconcile writes it back)
  ResAmount st_calc;
  bool st_calc_at_set = false;
  long long st_calc_at = 0;
  std::vector<std::string> st_messages;
  bool st_thr_pod = false;
  std::map<int, bool> st_thr_req;
  bool st_thr_req_nil = true;
  ResAmount st_used;
  bool live = false;
  uint64_t seq = 0;        // creation order: device columns of deleted throttles are reused, lists keep the order the objects arrived in
  bool host_dirty = true;  // applied since its last reconcile: the host-only parts of its status (messages, spec gauges) may differ even
                           // when the device-side diff says its numbers do not
  bool metrics_pending = false;  // reconciled since its gauges were last written into the registry (see record_metrics)
  std::string nn() const { return ns + "/" + name; }
  std::string selector_error() const {  // the first podSelector that LabelSelectorAsSelector rejects
    for (auto& t : terms)
      if (!t.pod_sel.error.empty()) return t.pod_sel.error;
    return "";
  }
};

// label key of the internal "this namespace exists" marker: not a legal label key, so it cannot collide with a real one
const char* const kNsExistsKey = "\x01kt/exists";

struct NamespaceObj {
  std::string name;
  std::vector<std::pair<std::string, std::string>> labels;
  bool exists = false;  // a Namespace object was applied (pods may reference namespaces the informer has not seen)
};

// reservedResourceAmounts (reserved_resource_amounts.go): throttle -> pod -> ResourceAmountOfPod
struct ReservationCache {
  std::map<std::string, std::map<std::string, std::map<int, Quantity>>> by_thr;  // thrNN -> podNN -> request list
  bool add(const std::string& thr, const PodObj& pod) {
    auto& m = by_thr[thr];
    const bool existed = m.count(pod.nn()) != 0;
    m[pod.nn()] = pod.request;  // overwrites (podResourceAmountMap.add, :131-136)
    return !existed;
  }
  bool remove(const std::string& thr, const std::string& pod_nn) {
    auto it = by_thr.find(thr);
    if (it == by_thr.end()) return false;
    return it->second.erase(pod_nn) != 0;
  }
  // the pod leaves EVERY throttle's reservation: what the event handlers fall back on when the pass that would have named the
  // pod's affected throttles cannot run (a superset of them; a pod is only ever reserved on throttles it matched)
  bool remove_everywhere(const std::string& pod_nn) {
    bool any = false;
    for (auto& kv : by_thr) any = (kv.second.erase(pod_nn) != 0) || any;
    return any;
  }
};

struct ResourceColumn {
  std::string name;
  int scale_exp = 0;  // device value = quantity / 10^scale_exp
  Quantity::Format format = Quantity::DecimalSI;
};

[[noreturn]] void fail(const std::string& m) { throw std::runtime_error(m); }

thread_local std::string g_ret;
const char* ret(std::string s) {
  g_ret = std::move(s);
  return g_ret.c_str();
}
std::string err_json(const std::string& m) {
  Writer w;
  w.begin_obj().key("error").str(m).end_obj();
  return w.out;
}
thread_local std::string g_new_plugin_error;  // read back by kth_new_plugin_error() on the calling thread

}  // namespace

struct kth_plugin {
  std::mutex mu;
  std::string name, target_scheduler;
  int device = 0;
  kt_ctx* ctx = nullptr;
  kt_limits lim{};  // limits the current engine was created with

  LabelDict labels;
  Dict ns_dict;
  std::vector<NamespaceObj> namespaces;  // by ns id
  std::vector<ResourceColumn> cols;      // resource column table
  Dict col_dict;

  std::vector<PodObj> pods;  // slot == device row of the running-pod table
  std::unordered_map<std::string, int64_t> pod_index;
  // Row arenas: the device kernels walk a warp's 32 rows word by word (kt_kernels.cuh reconcile_tile), which is one or two
  // rounds when the rows share a namespace and one round per row when they do not.  The reference's pod informer is indexed
  // by namespace (plugin.go:81-84); here a namespace owns whole chunks of kArenaChunk consecutive rows, a new pod takes a free
  // slot of its namespace's chunks (or opens a new chunk), a deleted pod's slot goes back to ITS namespace -- so rows stay
  // namespace-clustered under any churn, at the price of < kArenaChunk tombstone rows per namespace.
  static constexpr int64_t kArenaChunk = 32;
  std::unordered_map<std::string, std::vector<int64_t>> ns_free_rows;
  int64_t alloc_row(const std::string& ns) {
    std::vector<int64_t>& f = ns_free_rows[ns];
    if (f.empty()) {
      const int64_t base = (int64_t)pods.size();
      pods.resize((size_t)(base + kArenaChunk));
      for (int64_t i = 0; i < kArenaChunk; ++i) pods[(size_t)(base + i)].row = base + i;
      for (int64_t i = kArenaChunk - 1; i >= 0; --i) f.push_back(base + i);  // handed out front to back
    }
    const int64_t row = f.back();
    f.pop_back();
    return row;
  }
  std::set<int64_t> dirty_rows;
  uint64_t next_pod_seq = 1;
  int64_t row_capacity = 0;  // rows the device table currently holds
  bool pods_full_upload = true;

  std::vector<ThrottleObj> throttles;  // column order == device order (both kinds interleaved, insertion order)
  std::unordered_map<std::string, int> thr_index;  // "T:ns/name" | "C:/name"
  // Device columns of deleted throttles are handed out again (a scheduler that lives for months sees throttles come and go: M,
  // the table compile and every pass would only ever grow otherwise).  Whatever lists throttles for the caller -- affected
  // throttles of a pod (the order of the names inside a PreFilter reason), the broken-selector walk (WHICH error a pod gets),
  // reconcile's changed list -- is in creation order, as the reference's lister-backed slices are, not in column order.
  std::vector<int> free_thr;
  long long words_stat = -1;  // kth_queue_stats: words per namespace of the current layout (-1: not computed)
  uint64_t thr_seq = 0;
  bool thr_reused = false;  // some column holds a younger throttle than a higher one: column order is not creation order any more
  template <class V>
  void creation_order(V& cols_list) const {  // sort a list of throttle columns by creation
    if (thr_reused) std::stable_sort(cols_list.begin(), cols_list.end(), [&](size_t a, size_t b) { return throttles[a].seq < throttles[b].seq; });
  }
  bool throttles_dirty = true, namespaces_dirty = true, status_dirty = true, reserved_dirty = true;
  std::vector<size_t> broken;  // columns of the throttles with a podSelector that does not convert (controller_error)
  bool broken_valid = false;

  ReservationCache cache[2];  // one per controller (controller.go:34-50)

  // ---- the scheduling queue, resident on the device ------------------------------------------------------------------
  // Every pod the informer delivered that is ours to schedule (schedulerName == target, no nodeName yet, not finished) also
  // has a row in the device's PENDING table, maintained by the pod events like the running table.  PreFilter for such a pod
  // is addressed by key (kth_pre_filter_key): nothing is parsed, packed or uploaded for it, and ONE pass over the table
  // answers for the whole queue.  Rows [0, pend_capacity) are the queue, rows behind them are scratch rows for pods that
  // are NOT in the informer cache (the manifest arguments of kth_pre_filter / kth_reserve / kth_pre_filter_batch).
  std::vector<int64_t> pend_pod;   // queue row -> pods[] slot, -1: free
  std::vector<int64_t> pend_free;
  std::set<int64_t> pend_dirty;    // queue rows to (re)pack
  int64_t pend_capacity = 0, scratch_capacity = 0, scratch_used = 0;
  bool pend_full_upload = true;
  // Verdicts of the last pass over the queue, kept until something they depend on changes: a PreFilter verdict depends on the
  // pod's own row, the throttle set / selectors / namespaces (anything that recompiles tables: everything is void), and -- per
  // throttle -- the informer copy of its status and its reservations.  The last two are tracked per throttle (`dirty`): a
  // cached verdict stays good as long as none of the pod's affected throttles is dirty, so the scheduler's
  // PreFilter -> Reserve -> PreFilter(next pod) cycle only pays a device pass when consecutive pods share a throttle.
  struct QueueCache {
    bool valid = false;
    int Wp = 0;
    std::vector<uint8_t> admit, row_ok;             // [pend_capacity]; row_ok: the row's verdict belongs to the pod now in the row
    std::vector<uint32_t> bitmap;                   // [pend_capacity][Wp] affectedThrottles rows
    std::unordered_map<int64_t, std::vector<std::pair<uint32_t, uint32_t>>> codes;  // row -> non-zero {code word index, word}
    std::vector<uint32_t> dirty;                    // [Wp] throttles whose status / reservations changed since the pass
    uint64_t passes = 0, hits = 0;
  } queue;
  void queue_void() { queue.valid = false; }
  void throttle_state_changed(size_t t) {  // status or reservations of throttle column t
    if (queue.valid && (t >> 5) < queue.dirty.size()) queue.dirty[t >> 5] |= 1u << (t & 31);
  }
  void reservation_changed(size_t t) { reserved_dirty = true; throttle_state_changed(t); }
  bool apply_committed = false;  // kth_apply: the object was stored; whatever fails afterwards must not roll its resource names back
  std::string apply_warning;     // kth_apply: a committed object whose follow-up pass failed
  int max_labels = 0, max_ns_labels = 0;

  // ---- resource columns / scales ----------------------------------------------------------------
  int column(const std::string& rname) {
    int c = col_dict.find(rname);
    if (c >= 0) return c;
    // refuse BEFORE interning: the object that brought the name is rejected, the plugin stays usable
    if ((int)cols.size() >= KT_MAX_RESOURCES) fail("more than " + std::to_string(KT_MAX_RESOURCES) + " distinct resource names (" + rname + ")");
    c = (int)col_dict.id(rname);
    ResourceColumn rc;
    rc.name = rname;
    rc.scale_exp = rname == "cpu" ? -3 : 0;  // milli-cpu, whole units / bytes elsewhere; refined on demand
    cols.push_back(rc);
    if (ctx && (int)cols.size() > lim.n_resources) drop_engine();
    return c;
  }
  // An object that is refused (a limit, a malformed quantity) must not leave resource names behind that only it mentioned:
  // kth_apply undoes the interning that happened since it started.
  void rollback_columns(size_t n0) {
    if (cols.size() > n0) totals_valid = false;
    while (cols.size() > n0) {
      col_dict.ids.erase(col_dict.names.back());
      col_dict.names.pop_back();
      cols.pop_back();
    }
  }
  void note_quantity(int c, const Quantity& q) {
    const int need = kt::quantity_min_exp(q);
    if (need < cols[c].scale_exp) {  // a finer value than the column holds: every row of the column is re-packed
      cols[c].scale_exp = need;
      totals_valid = false;  // the running column totals were counted in the coarser unit
      pods_full_upload = pend_full_upload = throttles_dirty = status_dirty = reserved_dirty = true;
    }
    if (q.format == Quantity::BinarySI) cols[c].format = Quantity::BinarySI;
  }
  int64_t at_scale(int c, const Quantity& q) const {
    bool ok;
    const int64_t v = kt::quantity_at_scale(q, cols[c].scale_exp, &ok);
    if (!ok) fail("resource '" + cols[c].name + "': value " + kt::decimal_string(q) + " does not fit the int64 column at scale 1e" + std::to_string(cols[c].scale_exp));
    return v;
  }
  // PreFilter of a manifest keeps no state: a resource name nobody has a column for -- no throttle's threshold, override or
  // status mentions it, no pod of the informer requests it -- cannot influence the check (IsThrottledFor only looks at threshold
  // resources) and is not given one; a stream of pending pods with ever new extended-resource names must not use up the
  // KT_MAX_RESOURCES columns (or re-create the engine) for nothing.  Reserve and the informer events do intern: reservations
  // and status.used carry every name.
  bool check_only_names = false;
  std::map<int, Quantity> resource_list(const Node& n) {  // corev1.ResourceList
    std::map<int, Quantity> out;
    for (auto& kv : n.obj) {
      const int c = check_only_names ? col_dict.find(kv.first) : column(kv.first);
      if (c < 0) {
        (void)kt::parse_quantity(kv.second->scalar());  // a malformed quantity is still an error
        continue;
      }
      const Quantity q = kt::parse_quantity(kv.second->scalar());
      note_quantity(c, q);
      out[c] = q;
    }
    return out;
  }
  ResAmount res_amount(const Node& n) {
    ResAmount a;
    if (!n.is(Node::Obj)) return a;
    const Node& rc = n["resourceCounts"];
    if (rc.is(Node::Obj)) { a.has_counts = true; a.pod = rc["pod"].integer(0); }
    const Node& rr = n["resourceRequests"];
    if (rr.is(Node::Obj)) { a.requests_nil = false; a.requests = resource_list(rr); }
    return a;
  }

  // ---- PodRequestResourceList (pkg/resourcelist/resourcelist.go:27-46) ------------------------------
  std::map<int, Quantity> pod_request_resource_list(const Node& spec) {
    std::map<int, Quantity> ic, c;
    for (auto& ctr : spec["initContainers"].arr)  // icRes.SetMax(requests): rhs-only names are inserted as they are
      for (auto& kv : resource_list((*ctr)["resources"]["requests"])) {
        auto it = ic.find(kv.first);
        if (it == ic.end()) ic[kv.first] = kv.second;
        else if (kt::quantity_cmp(kv.second, it->second) > 0) it->second = kv.second;
      }
    for (auto& ctr : spec["containers"].arr)  // cRes.Add(requests)
      for (auto& kv : resource_list((*ctr)["resources"]["requests"])) {
        auto it = c.find(kv.first);
        if (it == c.end()) c[kv.first] = kv.second;
        else it->second = kt::quantity_add(it->second, kv.second);
      }
    for (auto& kv : ic) {  // cRes.SetMax(icRes)
      auto it = c.find(kv.first);
      if (it == c.end()) c[kv.first] = kv.second;
      else if (kt::quantity_cmp(kv.second, it->second) > 0) it->second = kv.second;
    }
    if (spec["overhead"].is(Node::Obj))  // pod.Spec.Overhead != nil
      for (auto& kv : resource_list(spec["overhead"])) {
        auto it = c.find(kv.first);
        if (it == c.end()) c[kv.first] = kv.second;
        else it->second = kt::quantity_add(it->second, kv.second);
      }
    for (auto& kv : c) note_quantity(kv.first, kv.second);
    return c;
  }
  PodObj pod_from(const Node& v) {
    PodObj p;
    const Node& md = v["metadata"];
    p.ns = md["namespace"].str();
    p.name = md["name"].str();
    for (auto& kv : md["labels"].obj) p.labels.emplace_back(kv.first, kv.second->str());
    const Node& spec = v["spec"];
    p.scheduler_name = spec["schedulerName"].str();
    p.node_name = spec["nodeName"].str();
    p.phase = v["status"]["phase"].str();
    p.request = pod_request_resource_list(spec);
    p.live = true;
    if ((int)p.labels.size() > max_labels) {
      if ((int)p.labels.size() > KT_MAX_LABEL_SLOTS) fail("pod " + p.nn() + " has more than " + std::to_string(KT_MAX_LABEL_SLOTS) + " labels");
      max_labels = (int)p.labels.size();
      if (ctx && max_labels > lim.label_slots) drop_engine();
    }
    return p;
  }
  uint32_t pod_flags(const PodObj& p) const {
    uint32_t f = 0;
    if (p.scheduler_name == target_scheduler) f |= KT_POD_SCHEDULER_MATCH;       // shouldCountIn, throttle_controller.go:217-219
    if (!p.node_name.empty()) f |= KT_POD_SCHEDULED;                            // isScheduled, pod_util.go:22-24
    if (p.phase != "Succeeded" && p.phase != "Failed") f |= KT_POD_NOT_FINISHED;  // isNotFinished, pod_util.go:26-28
    return f;
  }
  bool should_count_in(const PodObj& p) const { return p.scheduler_name == target_scheduler && !p.node_name.empty(); }
  // in the scheduling queue: ours to schedule, not bound, not finished
  bool is_queued(const PodObj& p) const {
    return p.live && p.scheduler_name == target_scheduler && p.node_name.empty() && p.phase != "Succeeded" && p.phase != "Failed";
  }
  // after pods[slot] changed: keep the resident queue table in step
  void queue_update(int64_t slot) {
    PodObj& p = pods[(size_t)slot];
    if (is_queued(p)) {
      if (p.pend_row < 0) {
        if (!pend_free.empty()) { p.pend_row = pend_free.back(); pend_free.pop_back(); }
        else { p.pend_row = (int64_t)pend_pod.size(); pend_pod.push_back(-1); }
        pend_pod[(size_t)p.pend_row] = slot;
      }
      pend_dirty.insert(p.pend_row);
      if ((size_t)p.pend_row < queue.row_ok.size()) queue.row_ok[(size_t)p.pend_row] = 0;
    } else if (p.pend_row >= 0) {
      queue_release(p.pend_row);
      p.pend_row = -1;
    }
  }
  void queue_release(int64_t row) {
    pend_pod[(size_t)row] = -1;
    pend_free.push_back(row);
    pend_dirty.insert(row);
    if ((size_t)row < queue.row_ok.size()) queue.row_ok[(size_t)row] = 0;
  }

  int32_t ns_id(const std::string& ns_name) {
    const uint32_t id = ns_dict.id(ns_name);
    if (namespaces.size() <= id) {
      namespaces.resize(id + 1);
      namespaces[id].name = ns_name;
      namespaces_dirty = throttles_dirty = true;  // Throttle namespace equality is part of the compiled tables
    }
    return (int32_t)id;
  }

  // ---- engine --------------------------------------------------------------------------------------
  void drop_engine() {
    if (ctx) kt_destroy(ctx);
    ctx = nullptr;
    sparse_cap = 0;
    queue.valid = false;
    pods_full_upload = pend_full_upload = throttles_dirty = namespaces_dirty = status_dirty = reserved_dirty = true;
  }
  void check(int rc, const char* what) {
    if (rc != KT_OK) fail(std::string(what) + ": " + (ctx ? kt_last_error(ctx) : "no engine") + " (" + std::to_string(rc) + ")");
  }
  static int round_up(int v, std::initializer_list<int> steps) {
    for (int s : steps)
      if (v <= s) return s;
    return *(steps.end() - 1);
  }
  void ensure_engine() {
    if (ctx) return;
    lim.abi_version = KT_ABI_VERSION;
    lim.n_resources = round_up(std::max<int>(1, (int)cols.size()), {4, 8, 16, 31});
    lim.label_slots = round_up(std::max(1, max_labels), {8, 16, 32});
    lim.ns_label_slots = round_up(std::max(1, max_ns_labels + 1), {4, 8, 16, 32});  // + the internal "exists" label
    const int rc = kt_create(&ctx, device, &lim);
    if (rc != KT_OK) { ctx = nullptr; fail("kt_create failed (" + std::to_string(rc) + "): no usable CUDA device -- there is no CPU path"); }
  }

  // pack one pod into compact single-row columns appended to the given vectors
  void pack_pod(const PodObj& p, std::vector<int64_t>& lab, std::vector<int64_t>& req, std::vector<uint32_t>& present, std::vector<uint32_t>& flags,
                std::vector<int32_t>& nsid, size_t k, size_t i) {
    const int L = lim.label_slots, R = lim.n_resources;
    for (int s = 0; s < L; ++s) lab[(size_t)s * k + i] = KT_LABEL_EMPTY;
    for (int r = 0; r < R; ++r) req[(size_t)r * k + i] = 0;
    present[i] = 0;
    flags[i] = 0;
    nsid[i] = 0;
    if (!p.live) return;  // tombstone: never counted, matches nothing
    int s = 0;
    for (auto& kv : p.labels) {
      const int64_t code = labels.encode(kv.first, kv.second);
      if (code != KT_LABEL_EMPTY) lab[(size_t)(s++) * k + i] = code;
    }
    for (auto& kv : p.request) {
      req[(size_t)kv.first * k + i] = at_scale(kv.first, kv.second);
      present[i] |= 1u << kv.first;
    }
    flags[i] = pod_flags(p);
    nsid[i] = ns_id(p.ns);
  }

  void sync_pods() {
    ensure_engine();
    const int L = lim.label_slots, R = lim.n_resources;
    if ((int64_t)pods.size() > row_capacity) pods_full_upload = true;
    if (pods_full_upload) {
      int64_t cap = std::max<int64_t>(64, row_capacity);
      while (cap < (int64_t)pods.size()) cap *= 2;
      const size_t k = (size_t)cap;
      std::vector<int64_t> lab((size_t)L * k), req((size_t)R * k);
      std::vector<uint32_t> present(k), flags(k);
      std::vector<int32_t> nsid(k);
      PodObj tomb;
      for (size_t i = 0; i < k; ++i) pack_pod(i < pods.size() ? pods[i] : tomb, lab, req, present, flags, nsid, k, i);
      overflow_check();
      check(kt_upload_pods(ctx, KT_PODS_RUNNING, cap, lab.data(), req.data(), present.data(), flags.data(), nsid.data()), "kt_upload_pods");
      row_capacity = cap;
      pods_full_upload = false;
      dirty_rows.clear();
    } else if (!dirty_rows.empty()) {
      const size_t k = dirty_rows.size();
      std::vector<int64_t> rows(dirty_rows.begin(), dirty_rows.end());
      std::vector<int64_t> lab((size_t)L * k), req((size_t)R * k);
      std::vector<uint32_t> present(k), flags(k);
      std::vector<int32_t> nsid(k);
      for (size_t i = 0; i < k; ++i) pack_pod(pods[(size_t)rows[i]], lab, req, present, flags, nsid, k, i);
      overflow_check();
      check(kt_update_pod_rows(ctx, KT_PODS_RUNNING, (int64_t)k, rows.data(), lab.data(), req.data(), present.data(), flags.data(), nsid.data()),
            "kt_update_pod_rows");
      dirty_rows.clear();
    }
  }
  // int64 adds (and the NCCL sum) wrap silently: prove per column that they cannot (DESIGN.md "Quantity columns").
  // The per-column totals of |value| are kept up to date by the pod events (totals_add), so a sync after a few events does
  // not walk the whole pod table again; they are recounted only after a column changed its unit.
  std::vector<__int128> col_abs;
  bool totals_valid = false;
  void totals_add(const PodObj& p, int sign) {
    if (!totals_valid || !p.live) return;
    if (col_abs.size() < cols.size()) col_abs.resize(cols.size(), 0);
    for (auto& kv : p.request) {
      bool ok;
      const int64_t v = kt::quantity_at_scale(kv.second, cols[(size_t)kv.first].scale_exp, &ok);
      if (!ok) { totals_valid = false; return; }  // the full recount reports it
      col_abs[(size_t)kv.first] += (v < 0 ? -(__int128)v : (__int128)v) * sign;
    }
  }
  void overflow_check() {
    if (!totals_valid) {
      col_abs.assign(cols.size(), 0);
      for (auto& p : pods)
        if (p.live)
          for (auto& kv : p.request) {
            const int64_t v = at_scale(kv.first, kv.second);
            col_abs[(size_t)kv.first] += v < 0 ? -(__int128)v : v;
          }
      totals_valid = true;
    }
    for (size_t c = 0; c < cols.size() && c < col_abs.size(); ++c)
      if (col_abs[c] >= ((__int128)1 << 62)) fail("resource '" + cols[c].name + "': the column sum can overflow int64 at scale 1e" + std::to_string(cols[c].scale_exp));
  }

  void sync_namespaces() {
    ensure_engine();
    if (!namespaces_dirty) return;
    queue_void();  // (see sync_throttles)
    words_stat = -1;
    const int LN = lim.ns_label_slots;
    const size_t n = namespaces.size();
    std::vector<int64_t> lab((size_t)LN * std::max<size_t>(n, 1), KT_LABEL_EMPTY);
    for (size_t i = 0; i < n; ++i) {
      int s = 0;
      for (auto& kv : namespaces[i].labels) {
        const int64_t code = labels.encode(kv.first, kv.second);
        if (code != KT_LABEL_EMPTY) lab[(size_t)(s++) * n + i] = code;
      }
      // A namespace the lister does not hold (never seen, or deleted) is not in the list affectedPods walks
      // (clusterthrottle_controller.go:227) -- no ClusterThrottle term may match it, not even one whose namespaceSelector is
      // empty.  Existing namespaces carry one internal label (a key no real label can have) that every term requires.
      if (namespaces[i].exists && labels.encode(kNsExistsKey, "1") != KT_LABEL_EMPTY) lab[(size_t)(s++) * n + i] = labels.encode(kNsExistsKey, "1");
    }
    check(kt_upload_namespaces(ctx, (int32_t)n, lab.data()), "kt_upload_namespaces");
    namespaces_dirty = false;
  }

  // ---- device columns in NAMESPACE order ----------------------------------------------------------------------------
  // A pod only visits the 32-throttle words in which some throttle can apply to its namespace, and every word costs a round
  // of table gathers and segmented sums: what a pass costs is the number of words per namespace.  Columns in the order the
  // objects happened to arrive scatter a namespace's throttles over all the words (BASELINE C2 created in random order: 15.6
  // words per pod instead of 1.7; C3: 31.7 instead of 8.9 -- tools/words_per_namespace.py).  So, whenever the throttle set
  // changes, the columns are laid out again: Throttles by namespace, ClusterThrottles by the SET of namespaces their
  // namespaceSelectors admit (the sets as strings of one character per namespace, in lexicographic order: equal sets adjacent,
  // sets that share their first namespaces near each other -- C3: 8.9 words per pod; largest-sets-first 11.1, a greedy
  // nearest-neighbour chain 10.0), creation order inside a group; columns of deleted throttles disappear.  Nothing the caller sees depends on column order (creation_order above); everything per column on
  // the device is uploaded again after a throttle change anyway.  (The pod rows get the same treatment: row arenas.)
  static std::string ns_selector_signature(const ThrottleObj& o) {
    std::string sig;
    for (auto& t : o.terms) {
      if (!t.ns_sel.error.empty()) { sig += "!|"; continue; }  // Q9: swallowed, the term matches no namespace
      for (auto& r : t.ns_sel.reqs) {
        sig += r.key;
        sig += (char)('0' + r.op);
        for (auto& v : r.values) { sig += v; sig += ','; }
        sig += ';';
      }
      sig += '|';
    }
    return sig;
  }
  std::string namespace_set_of(const ThrottleObj& o) const {  // one character per namespace id: which namespaces some term admits
    std::string set(namespaces.size(), '0');
    for (size_t i = 0; i < namespaces.size(); ++i) {
      if (!namespaces[i].exists) continue;
      for (auto& t : o.terms)
        if (t.ns_sel.error.empty() && ns_selector_matches(t.ns_sel, namespaces[i])) { set[i] = '1'; break; }
    }
    return set;
  }
  void reorder_columns() {
    struct Key {
      int kind;
      std::string set;
      uint64_t seq;
      size_t idx;
    };
    std::vector<Key> keys;
    std::map<std::string, std::string> set_of;  // distinct ClusterThrottle signatures: evaluated once
    bool dead = false;
    for (size_t t = 0; t < throttles.size(); ++t) {
      const ThrottleObj& o = throttles[t];
      if (!o.live) { dead = true; continue; }
      Key k{o.kind == KT_KIND_THROTTLE ? 0 : 1, std::string(), o.seq, t};
      if (o.kind == KT_KIND_THROTTLE) {
        k.set = o.ns;
      } else {
        const std::string sig = ns_selector_signature(o);
        auto it = set_of.find(sig);
        if (it == set_of.end()) it = set_of.emplace(sig, namespace_set_of(o)).first;
        k.set = it->second;
      }
      keys.push_back(std::move(k));
    }
    std::stable_sort(keys.begin(), keys.end(), [](const Key& a, const Key& b) {
      if (a.kind != b.kind) return a.kind < b.kind;
      if (a.set != b.set) return a.set < b.set;
      return a.seq < b.seq;
    });
    bool same = !dead;
    for (size_t i = 0; same && i < keys.size(); ++i) same = keys[i].idx == i;
    if (same) return;
    std::vector<ThrottleObj> laid_out;
    laid_out.reserve(keys.size());
    for (auto& k : keys) laid_out.push_back(std::move(throttles[k.idx]));
    throttles = std::move(laid_out);
    thr_index.clear();
    free_thr.clear();
    thr_reused = false;
    for (size_t t = 0; t < throttles.size(); ++t) {
      thr_index[std::string(throttles[t].kind == KT_KIND_THROTTLE ? "T:" : "C:") + throttles[t].nn()] = (int)t;
      if (t && throttles[t].seq < throttles[t - 1].seq) thr_reused = true;  // column order is not creation order
    }
    broken_valid = false;
    queue_void();
    status_dirty = reserved_dirty = true;
  }

  // Throttle specs -> kt_throttle_cols + kt_selector_table.  Terms after the first invalid podSelector are
  // unreachable in the reference (MatchesToPod returns the error first), so they are not compiled.
  void sync_throttles() {
    ensure_engine();
    if (!throttles_dirty) return;
    // The cached verdicts of the resident queue were computed with the old tables: whoever brings the new ones to the device --
    // a PreFilter pass or, before it, a reconcile -- voids them.  (Found by the resident-queue event stream of the second session
    // of round 2: throttle edit, reconcile, PreFilter by key answered from the cache of the OLD throttle set.)
    queue_void();
    words_stat = -1;
    reorder_columns();
    const int R = lim.n_resources;
    const size_t m = throttles.size();
    std::vector<uint8_t> kind(m), flags(m);
    std::vector<int32_t> nsid(m), ovr_off(m + 1, 0);
    std::vector<int64_t> thr((size_t)R * std::max<size_t>(m, 1), 0), thr_cnt(m, 0);
    std::vector<uint32_t> thr_present(m, 0);
    std::vector<int64_t> ovr_begin, ovr_end, ovr_cnt;
    std::vector<uint8_t> ovr_flags;
    std::vector<uint32_t> ovr_present;
    std::vector<std::vector<int64_t>> ovr_vals;  // per override: R values
    std::vector<int32_t> term_off(m + 1, 0), pod_req_off{0}, ns_req_off, req_val_off{0};
    std::vector<uint8_t> term_flags, req_op;
    std::vector<uint32_t> req_key, req_vals;
    std::vector<std::vector<Requirement>> ns_reqs_of_term;
    auto push_reqs = [&](const std::vector<Requirement>& reqs) {
      for (auto& r : reqs) {
        const uint32_t kid = labels.key_id(r.key);  // (all of it interned by sync_vocabulary already)
        req_key.push_back(kid);
        req_op.push_back(r.op);
        for (auto& v : r.values) req_vals.push_back(labels.value_id(kid, v));
        req_val_off.push_back((int32_t)req_vals.size());
      }
    };
    auto amount_cols = [&](const ResAmount& a, int64_t* vals, size_t stride, uint32_t* present, int64_t* cnt) {
      *present = 0;
      *cnt = 0;
      if (a.has_counts) { *present |= KT_COUNT_BIT; *cnt = a.pod; }
      for (auto& kv : a.requests) {
        vals[(size_t)kv.first * stride] = at_scale(kv.first, kv.second);
        *present |= 1u << kv.first;
      }
    };
    for (size_t t = 0; t < m; ++t) {
      const ThrottleObj& o = throttles[t];
      kind[t] = (uint8_t)o.kind;
      nsid[t] = o.kind == KT_KIND_THROTTLE ? ns_id(o.ns) : -1;
      flags[t] = 0;
      if (o.live && o.throttler_name == name) flags[t] |= KT_THR_RESPONSIBLE;  // isResponsibleFor, throttle_controller.go:213-215
      amount_cols(o.threshold, &thr[t], m, &thr_present[t], &thr_cnt[t]);
      for (size_t i = 0; i < o.overrides.size(); ++i) {
        const Override& ov = o.overrides[i];
        GoTime b, e;
        uint8_t f = 0;
        if (!ov.begin.empty() && !parse_rfc3339(ov.begin, &b).empty()) f = KT_OVR_PARSE_ERROR;
        if (!ov.end.empty() && !parse_rfc3339(ov.end, &e).empty()) f = KT_OVR_PARSE_ERROR;
        ovr_begin.push_back(b.zero ? KT_TIME_OPEN_BEGIN : clamp_ns(b.ns()));
        ovr_end.push_back(e.zero ? KT_TIME_OPEN_END : clamp_ns(e.ns()));
        ovr_flags.push_back(f);
        std::vector<int64_t> vals((size_t)R, 0);
        uint32_t pr;
        int64_t cnt;
        amount_cols(ov.threshold, vals.data(), 1, &pr, &cnt);
        ovr_vals.push_back(std::move(vals));
        ovr_present.push_back(pr);
        ovr_cnt.push_back(cnt);
      }
      ovr_off[t + 1] = (int32_t)ovr_begin.size();
      for (auto& term : o.terms) {
        // a podSelector that does not convert: the term matches nobody and shadows the LATER terms for exactly the pods that
        // reach it (KT_TERM_POD_INVALID; the table compiler scopes that by namespace / namespaceSelector)
        term_flags.push_back((term.ns_sel.error.empty() ? 0 : KT_TERM_NS_INVALID) |  // Q9: swallowed, the term is false
                             (term.pod_sel.error.empty() ? 0 : KT_TERM_POD_INVALID));
        push_reqs(term.pod_sel.reqs);  // (none when the selector is broken)
        pod_req_off.push_back((int32_t)req_key.size());
        std::vector<Requirement> nsr;
        if (o.kind == KT_KIND_CLUSTERTHROTTLE && term.ns_sel.error.empty()) {
          nsr = term.ns_sel.reqs;
          Requirement ex;  // the namespace must be one the lister holds (sync_namespaces)
          ex.key = kNsExistsKey;
          ex.op = KT_OP_EXISTS;
          nsr.push_back(std::move(ex));
        }
        ns_reqs_of_term.push_back(std::move(nsr));
      }
      term_off[t + 1] = (int32_t)term_flags.size();
    }
    // requirement pool layout: all podSelector requirements (term order), then all namespaceSelector ones
    ns_req_off.push_back((int32_t)req_key.size());
    for (auto& reqs : ns_reqs_of_term) {
      push_reqs(reqs);
      ns_req_off.push_back((int32_t)req_key.size());
    }
    const size_t n_ovr = ovr_begin.size();
    std::vector<int64_t> ovr_thr((size_t)R * std::max<size_t>(n_ovr, 1), 0);
    for (size_t i = 0; i < n_ovr; ++i)
      for (int r = 0; r < R; ++r) ovr_thr[(size_t)r * n_ovr + i] = ovr_vals[i][(size_t)r];
    kt_throttle_cols tc{};
    tc.kind = kind.data(); tc.ns_id = nsid.data(); tc.flags = flags.data(); tc.thr = thr.data(); tc.thr_present = thr_present.data();
    tc.thr_cnt = thr_cnt.data(); tc.ovr_off = ovr_off.data(); tc.n_ovr = (int32_t)n_ovr; tc.ovr_begin = ovr_begin.data(); tc.ovr_end = ovr_end.data();
    tc.ovr_flags = ovr_flags.data(); tc.ovr_thr = ovr_thr.data(); tc.ovr_present = ovr_present.data(); tc.ovr_cnt = ovr_cnt.data();
    kt_selector_table st{};
    st.n_terms = (int32_t)term_flags.size(); st.n_reqs = (int32_t)req_key.size(); st.n_vals = (int32_t)req_vals.size();
    st.term_off = term_off.data(); st.term_flags = term_flags.data(); st.pod_req_off = pod_req_off.data(); st.ns_req_off = ns_req_off.data();
    st.req_key = req_key.data(); st.req_op = req_op.data(); st.req_val_off = req_val_off.data(); st.req_vals = req_vals.data();
    sync_namespaces();  // Throttle rows may have introduced namespace ids
    check(kt_upload_throttles(ctx, (int32_t)m, &tc, &st), "kt_upload_throttles");
    throttles_dirty = false;
    status_dirty = reserved_dirty = true;  // kt_upload_throttles forgets both
  }

  void sync_status() {
    if (!status_dirty) return;
    const int R = lim.n_resources;
    const size_t m = throttles.size();
    if (m == 0) { status_dirty = false; return; }
    std::vector<uint8_t> calculated(m, 0);
    std::vector<int64_t> calc_thr((size_t)R * m, 0), calc_cnt(m, 0), used((size_t)R * m, 0), used_cnt(m, 0);
    std::vector<uint32_t> calc_present(m, 0), used_present(m, 0), throttled(m, 0);
    for (size_t t = 0; t < m; ++t) {
      const ThrottleObj& o = throttles[t];
      calculated[t] = o.st_calc_at_set;  // !CalculatedAt.Time.IsZero() (throttle_types.go:129-132)
      if (o.st_calc.has_counts) { calc_present[t] |= KT_COUNT_BIT; calc_cnt[t] = o.st_calc.pod; }
      for (auto& kv : o.st_calc.requests) { calc_thr[(size_t)kv.first * m + t] = at_scale(kv.first, kv.second); calc_present[t] |= 1u << kv.first; }
      if (o.st_used.has_counts) { used_present[t] |= KT_COUNT_BIT; used_cnt[t] = o.st_used.pod; }
      for (auto& kv : o.st_used.requests) { used[(size_t)kv.first * m + t] = at_scale(kv.first, kv.second); used_present[t] |= 1u << kv.first; }
      if (o.st_thr_pod) throttled[t] |= KT_COUNT_BIT;
      for (auto& kv : o.st_thr_req)
        if (kv.second) throttled[t] |= 1u << kv.first;
    }
    kt_status_cols sc{calculated.data(), calc_thr.data(), calc_present.data(), calc_cnt.data(), used.data(), used_present.data(), used_cnt.data(), throttled.data()};
    check(kt_upload_status(ctx, &sc), "kt_upload_status");
    status_dirty = false;
  }

  void sync_reserved() {
    if (!reserved_dirty) return;
    const int R = lim.n_resources;
    const size_t m = throttles.size();
    if (m == 0) { reserved_dirty = false; return; }
    std::vector<int64_t> reserved((size_t)R * m, 0), cnt(m, 0);
    std::vector<uint32_t> present(m, 0);
    bool any = false;
    for (size_t t = 0; t < m; ++t) {
      const ThrottleObj& o = throttles[t];
      auto it = cache[o.kind].by_thr.find(o.nn());
      if (it == cache[o.kind].by_thr.end() || it->second.empty()) continue;
      any = true;
      present[t] |= KT_COUNT_BIT;  // every reserved ResourceAmountOfPod carries Counts{Pod: 1}
      cnt[t] = (int64_t)it->second.size();
      for (auto& pod : it->second)
        for (auto& kv : pod.second) {
          reserved[(size_t)kv.first * m + t] += at_scale(kv.first, kv.second);
          present[t] |= 1u << kv.first;
        }
    }
    if (any) check(kt_set_reserved(ctx, reserved.data(), present.data(), cnt.data()), "kt_set_reserved");
    else check(kt_set_reserved(ctx, nullptr, nullptr, nullptr), "kt_set_reserved");
    reserved_dirty = false;
  }
  // What the selectors mention goes into the label dictionaries BEFORE any row is packed; rows that carry newly mentioned keys or
  // values (they were packed as "invisible" / "some other value") are packed again.
  void sync_vocabulary() {
    if (!throttles_dirty) return;
    std::unordered_set<std::string> new_keys;
    std::unordered_map<std::string, std::unordered_set<std::string>> new_vals;
    auto intern = [&](const std::vector<Requirement>& reqs) {
      for (auto& r : reqs) {
        bool added = false;
        const uint32_t kid = labels.key_id(r.key, &added);
        if (added) new_keys.insert(r.key);
        for (auto& v : r.values) {
          labels.value_id(kid, v, &added);
          if (added) new_vals[r.key].insert(v);
        }
      }
    };
    bool cluster_terms = false;
    for (auto& o : throttles)
      for (auto& term : o.terms) {
        intern(term.pod_sel.reqs);
        if (o.kind == KT_KIND_CLUSTERTHROTTLE) { intern(term.ns_sel.reqs); cluster_terms = true; }
      }
    if (cluster_terms) {
      bool added = false;
      labels.key_id(kNsExistsKey, &added);
      if (added) new_keys.insert(kNsExistsKey);
    }
    if (new_keys.empty() && new_vals.empty()) return;
    auto carries_news = [&](const std::vector<std::pair<std::string, std::string>>& labs) {
      for (auto& kv : labs) {
        if (new_keys.count(kv.first)) return true;
        auto it = new_vals.find(kv.first);
        if (it != new_vals.end() && it->second.count(kv.second)) return true;
      }
      return false;
    };
    for (auto& p : pods) {
      if (!p.live || !carries_news(p.labels)) continue;
      if (p.row >= 0) dirty_rows.insert(p.row);
      if (p.pend_row >= 0) pend_dirty.insert(p.pend_row);
    }
    namespaces_dirty = true;  // (a handful of rows: packed whole)
  }
  void sync_all() {
    sync_vocabulary();
    sync_pods();
    sync_namespaces();
    sync_throttles();
  }

  // ---- results -> objects ------------------------------------------------------------------------------
  Quantity from_scale(int c, int64_t v) const {
    Quantity q;
    q.mant = v;
    q.exp = cols[c].scale_exp;
    q.format = cols[c].format;
    q.canon();
    return q;
  }
  void amount_json(Writer& w, const ResAmount& a) const {
    w.begin_obj();
    if (a.has_counts) { w.key("resourceCounts").begin_obj().key("pod").num(a.pod).end_obj(); }
    if (!a.requests_nil) {
      w.key("resourceRequests").begin_obj();
      for (auto& kv : a.requests) w.key(cols[kv.first].name).str(kt::decimal_string(kv.second));
      w.end_obj();
    }
    w.end_obj();
  }
  static bool amount_equal(const ResAmount& a, const ResAmount& b) {  // apiequality.Semantic.DeepEqual on ResourceAmount
    if (a.has_counts != b.has_counts || (a.has_counts && a.pod != b.pod)) return false;
    if (a.requests.size() != b.requests.size()) return false;  // nil and empty maps are equal
    for (auto& kv : a.requests) {
      auto it = b.requests.find(kv.first);
      if (it == b.requests.end() || kt::quantity_cmp(kv.second, it->second) != 0) return false;
    }
    return true;
  }

  // CalculateThreshold's Messages (throttle_types.go:78-84): "index %d: Failed to parse Begin|End: <time.Parse error>"
  static std::vector<std::string> override_messages(const ThrottleObj& o) {
    std::vector<std::string> msgs;
    for (size_t i = 0; i < o.overrides.size(); ++i) {
      GoTime t;
      std::string e;
      if (!o.overrides[i].begin.empty() && !(e = parse_rfc3339(o.overrides[i].begin, &t)).empty()) {
        msgs.push_back("index " + std::to_string(i) + ": Failed to parse Begin: " + e);
        continue;
      }
      if (!o.overrides[i].end.empty() && !(e = parse_rfc3339(o.overrides[i].end, &t)).empty())
        msgs.push_back("index " + std::to_string(i) + ": Failed to parse End: " + e);
    }
    return msgs;
  }

  // NextOverrideHappensIn (throttle_types.go:37-63): the nearest override boundary after `now`, i.e. when the throttle
  // must be reconciled again although no object changed (the reference enqueues it with enqueueAfter, :201-208).
  // An override whose Begin does not parse is skipped entirely; one whose End does not parse still contributes its Begin.
  static bool next_override_happens_in(const ThrottleObj& o, const GoTime& now, __int128* nanos) {
    bool have = false;
    auto consider = [&](const GoTime& t) {
      if (t.zero) return;  // time.Time{} is never After(now)
      const __int128 d = t.ns() - now.ns();
      if (d > 0 && (!have || d < *nanos)) { *nanos = d; have = true; }
    };
    for (auto& ov : o.overrides) {
      GoTime b, e;
      if (!ov.begin.empty() && !parse_rfc3339(ov.begin, &b).empty()) continue;
      consider(b);
      if (!ov.end.empty() && !parse_rfc3339(ov.end, &e).empty()) continue;
      consider(e);
    }
    return have;
  }

  // ---- reconcile: every throttle in one device pass ------------------------------------------------
  // ---- gauges (throttle_metrics.go / clusterthrottle_metrics.go / metrics_recorder.go) --------------------------
  // A GaugeVec keeps every series it was ever given: reconcile records the throttle it just handled, nothing is deleted
  // when a throttle or one of its resource names goes away.  family -> (label pairs sorted by name, rendered) -> value.
  // Rendering ~20 label sets per throttle is 3 us of string work -- a hundred times the device pass for 1000 throttles -- so
  // reconcile only MARKS the throttle (metrics_pending); the registry is brought up to date when somebody looks at it
  // (kth_metrics) and, so that the values are the ones of the last reconcile and nothing newer, right before the object
  // changes under it (a spec or status update, a delete).
  std::map<std::string, std::map<std::string, double>> gauges;
  static std::string label_escape(const std::string& v) {
    std::string o;
    for (char c : v) {
      if (c == '\\') o += "\\\\";
      else if (c == '"') o += "\\\"";
      else if (c == '\n') o += "\\n";
      else o += c;
    }
    return o;
  }
  void record_metrics(const ThrottleObj& o) {
    const bool cluster = o.kind == KT_KIND_CLUSTERTHROTTLE;
    const std::string prefix = cluster ? "clusterthrottle_" : "throttle_";
    auto series = [&](const std::string& resource) {  // client_golang sorts the label pairs by name
      std::string l = "name=\"" + label_escape(o.name) + "\"";
      if (!cluster) l += ",namespace=\"" + label_escape(o.ns) + "\"";
      l += ",resource=\"" + label_escape(resource) + "\",uid=\"" + label_escape(o.uid) + "\"";
      return l;
    };
    auto counts = [&](const std::string& fam, bool has, long long pod) {  // recordResourceCounts: nil -> 0
      gauges[prefix + fam][series("pod")] = has ? (double)pod : 0.0;
    };
    auto requests = [&](const std::string& fam, const ResAmount& a) {  // recordResourceRequests: cpu in milli, the rest in units
      for (auto& kv : a.requests) {
        const std::string& rn = cols[(size_t)kv.first].name;
        gauges[prefix + fam][series(rn)] = (double)kt::quantity_scaled_value(kv.second, rn == "cpu" ? -3 : 0);
      }
    };
    counts("spec_threshold_resourceCounts", o.threshold.has_counts, o.threshold.pod);
    requests("spec_threshold_resourceRequests", o.threshold);
    gauges[prefix + "status_throttled_resourceCounts"][series("pod")] = o.st_thr_pod ? 1.0 : 0.0;
    if (!o.st_thr_req_nil)
      for (auto& kv : o.st_thr_req) gauges[prefix + "status_throttled_resourceRequests"][series(cols[(size_t)kv.first].name)] = kv.second ? 1.0 : 0.0;
    counts("status_used_resourceCounts", o.st_used.has_counts, o.st_used.pod);
    requests("status_used_resourceRequests", o.st_used);
    counts("status_calculated_threshold_resourceCounts", o.st_calc.has_counts, o.st_calc.pod);
    requests("status_calculated_threshold_resourceRequests", o.st_calc);
  }
  // expfmt's writeFloat: shortcuts for 0, 1 and -1, else strconv.AppendFloat(f, 'g', -1, 64) -- the shortest digits that
  // round-trip, in %e form when the decimal exponent is < -4 or >= 6 (Go's 'g' decides with precision 6 in shortest mode,
  // so 1000000 prints as 1e+06 and 536870912 as 5.36870912e+08), else in %f form with no padding.
  static std::string go_float(double f) {
    if (f == 0) return "0";
    if (f == 1) return "1";
    if (f == -1) return "-1";
    if (f != f) return "NaN";
    if (f > 1.7976931348623157e308) return "+Inf";
    if (f < -1.7976931348623157e308) return "-Inf";
    char buf[64];
    auto r = std::to_chars(buf, buf + sizeof buf, f, std::chars_format::scientific);  // shortest round-trip digits, d.ddde[+-]XX
    std::string sci(buf, r.ptr);
    const size_t epos = sci.find('e');
    std::string mant = sci.substr(0, epos);
    const int exp = std::atoi(sci.c_str() + epos + 1);
    const bool neg = mant[0] == '-';
    if (neg) mant.erase(0, 1);
    std::string digits;
    for (char c : mant)
      if (c != '.') digits += c;
    std::string out = neg ? "-" : "";
    if (exp < -4 || exp >= 6) {  // %e with the shortest digits and an exponent of at least two digits
      out += digits.substr(0, 1);
      if (digits.size() > 1) out += "." + digits.substr(1);
      out += exp < 0 ? "e-" : "e+";
      const int a = exp < 0 ? -exp : exp;
      if (a < 10) out += "0";
      out += std::to_string(a);
      return out;
    }
    if (exp >= 0) {  // %f with just the digits needed
      if ((int)digits.size() <= exp + 1) return out + digits + std::string((size_t)(exp + 1) - digits.size(), '0');
      return out + digits.substr(0, (size_t)exp + 1) + "." + digits.substr((size_t)exp + 1);
    }
    return out + "0." + std::string((size_t)(-exp - 1), '0') + digits;
  }
  void flush_metrics() {
    for (auto& o : throttles)
      if (o.metrics_pending) { record_metrics(o); o.metrics_pending = false; }
  }
  std::string metrics_text() const {
    static const std::pair<const char*, const char*> kHelp[] = {
        {"spec_threshold_resourceCounts", "threshold on specific resourceCounts of the %s"},
        {"spec_threshold_resourceRequests", "threshold on specific resourceRequests of the %s"},
        {"status_calculated_threshold_resourceCounts", "calculated threshold on specific resourceCounts of the %s"},
        {"status_calculated_threshold_resourceRequests", "calculated threshold on specific resourceRequests of the %s"},
        {"status_throttled_resourceCounts", "resourceCounts of the %s is throttled or not on specific resource (1=throttled, 0=not throttled)"},
        {"status_throttled_resourceRequests", "resourceRequests of the %s is throttled or not on specific resource (1=throttled, 0=not throttled)"},
        {"status_used_resourceCounts", "used resource counts of the %s"},
        {"status_used_resourceRequests", "used amount of resource requests of the %s"},
    };
    std::string out;
    for (const char* prefix : {"clusterthrottle_", "throttle_"})  // families in name order, as Gather returns them
      for (auto& h : kHelp) {
        auto it = gauges.find(std::string(prefix) + h.first);
        if (it == gauges.end() || it->second.empty()) continue;
        std::string help = h.second;
        help.replace(help.find("%s"), 2, "throttle");  // both recorders say "throttle" (clusterthrottle_metrics.go:44-100)
        out += "# HELP " + it->first + " " + help + "\n# TYPE " + it->first + " gauge\n";
        for (auto& sv : it->second) out += it->first + "{" + sv.first + "} " + go_float(sv.second) + "\n";
      }
    return out;
  }

  std::string reconcile_all(const std::string& now_s) {
    GoTime now;
    std::string e = parse_rfc3339(now_s, &now);
    if (!e.empty()) fail(e);
    sync_all();
    const size_t m = throttles.size();
    Writer w;
    w.begin_obj();
    if (m == 0) { w.key("reconciled").num(0).key("changed").begin_arr().end_arr().key("requeueAfterNanos").begin_obj().end_obj().end_obj(); return w.out; }
    // The informer copy of every status is on the device (sync_status: a no-op unless some status changed since the last
    // upload), so the pass itself diffs what it computes against it (throttle_controller.go:157 DeepEqual): only the throttles it
    // lists -- plus those applied since their last reconcile, whose host-only status parts may differ -- are looked at and
    // downloaded below (SURVEY 8f.3: the download and the host's work are proportional to what changed, not to M).
    sync_status();
    check(kt_evaluate(ctx, clamp_ns(now.ns()), KT_EVAL_FRESH_STATUS | KT_EVAL_SKIP_CHECK), "kt_evaluate");
    const int R = lim.n_resources;
    std::vector<int32_t> todo_idx(m);
    std::vector<int32_t> pos(m, -1);  // throttle column -> its row in the gathered status columns
    size_t k = 0;
    {
      int64_t n_changed = 0;
      check(kt_get_changed(ctx, todo_idx.data(), (int64_t)m, &n_changed, nullptr), "kt_get_changed");
      std::vector<char> mark(m, 0);
      for (int64_t i = 0; i < n_changed && i < (int64_t)m; ++i) mark[(size_t)todo_idx[(size_t)i]] = 1;
      for (size_t t = 0; t < m; ++t)
        if (throttles[t].host_dirty && throttles[t].live) mark[t] = 1;
      for (size_t t = 0; t < m; ++t)
        if (mark[t]) { pos[t] = (int32_t)k; todo_idx[k++] = (int32_t)t; }
    }
    std::vector<int64_t> used((size_t)R * std::max<size_t>(k, 1)), used_cnt(k), calc_thr((size_t)R * std::max<size_t>(k, 1)), calc_cnt(k);
    std::vector<uint32_t> used_present(k), throttled(k), calc_present(k);
    std::vector<uint8_t> ovr_active(k);
    kt_reconcile_out ro{used.data(), used_present.data(), used_cnt.data(), throttled.data(), calc_thr.data(), calc_present.data(), calc_cnt.data(), ovr_active.data()};
    if (k) check(kt_get_reconcile_rows(ctx, (int64_t)k, todo_idx.data(), &ro), "kt_get_reconcile_rows");
    // pods that are reserved somewhere: their match rows decide what reconcile un-reserves (:135-155)
    std::vector<int64_t> rows;
    std::vector<std::string> row_pod;
    {
      std::set<std::string> seen;
      for (int k = 0; k < 2; ++k)
        for (auto& thr : cache[k].by_thr)
          for (auto& pod : thr.second) {
            auto it = pod_index.find(pod.first);
            if (it != pod_index.end() && seen.insert(pod.first).second) { rows.push_back(it->second); row_pod.push_back(pod.first); }
          }
    }
    const int Wp = kt_match_words(ctx);
    std::vector<uint32_t> words(rows.size() * (size_t)Wp);
    if (!rows.empty()) check(kt_get_match_rows(ctx, KT_PODS_RUNNING, (int64_t)rows.size(), rows.data(), words.data()), "kt_get_match_rows");
    // Q8 (throttle_controller.go:241, `terminatedPods = append(nonterminatedPods, pod)`): the THROTTLE controller's list of
    // terminated affected pods ends up holding only the LAST terminated match of the namespace, so of the finished pods that
    // still hold a reservation only that one is un-reserved; the others keep it until the pod is deleted.  (Which pod is "last"
    // is the informer's map order in the reference; the oracle and this code take the order of first appearance.)  Needed only
    // when a finished pod holds a reservation: then the match rows of the finished counted pods say who is last per throttle.
    std::vector<char> row_finished(rows.size(), 0);
    bool any_finished_reserved = false;
    for (size_t i = 0; i < rows.size(); ++i) {
      const PodObj& p = pods[(size_t)rows[i]];
      row_finished[i] = p.live && !(pod_flags(p) & KT_POD_NOT_FINISHED);
      any_finished_reserved |= row_finished[i] != 0;
    }
    std::vector<int64_t> fin_rows;
    std::vector<uint32_t> fin_words;
    if (any_finished_reserved) {
      for (auto& p : pods)
        if (p.live && should_count_in(p) && !(pod_flags(p) & KT_POD_NOT_FINISHED)) fin_rows.push_back(p.row);
      fin_words.resize(fin_rows.size() * (size_t)Wp);
      if (!fin_rows.empty()) check(kt_get_match_rows(ctx, KT_PODS_RUNNING, (int64_t)fin_rows.size(), fin_rows.data(), fin_words.data()), "kt_get_match_rows");
    }
    auto last_finished_match = [&](size_t t, const std::string& ns) -> int64_t {  // row of the last finished pod of ns that matches t
      int64_t best = -1;
      uint64_t best_seq = 0;
      for (size_t i = 0; i < fin_rows.size(); ++i) {
        const PodObj& p = pods[(size_t)fin_rows[i]];
        if (p.ns != ns || !((fin_words[i * (size_t)Wp + (t >> 5)] >> (t & 31)) & 1)) continue;
        if (best < 0 || p.seq > best_seq) { best = p.row; best_seq = p.seq; }
      }
      return best;
    };

    // A Throttle with a podSelector term that does not convert: affectedPods (throttle_controller.go:221-246) only fails -- and
    // the reconcile with it -- when some counted pod of the namespace actually REACHES that term, i.e. matches none of the
    // valid terms before it (those are what the device column holds, sync_throttles).  The rows of the namespace's counted
    // pods tell.  ClusterThrottles: see DESIGN.md "Known deviations" (their terms carry their own namespace scope).
    std::vector<char> selector_fails(m, 0);
    for (size_t t = 0; t < m; ++t) {
      const ThrottleObj& o = throttles[t];
      if (!o.live || o.throttler_name != name || o.selector_error().empty()) continue;
      // the counted pods a broken term is in the way of: the Throttle's namespace, or -- per term -- the namespaces a
      // ClusterThrottle term's namespaceSelector matches (clusterthrottle_controller.go:224-270 walks exactly those pods)
      std::vector<int64_t> ns_rows;
      std::map<std::string, bool> ns_reaches;
      for (auto& p : pods) {
        if (!p.live || !should_count_in(p)) continue;
        if (o.kind == KT_KIND_THROTTLE) {
          if (p.ns != o.ns) continue;
        } else {
          auto f = ns_reaches.find(p.ns);
          if (f == ns_reaches.end()) f = ns_reaches.emplace(p.ns, !reachable_selector_error(o, p.ns).empty()).first;
          if (!f->second) continue;
        }
        ns_rows.push_back(p.row);
      }
      if (ns_rows.empty()) continue;  // nobody to ask the selector about: no error
      std::vector<uint32_t> w((size_t)ns_rows.size() * (size_t)Wp);
      check(kt_get_match_rows(ctx, KT_PODS_RUNNING, (int64_t)ns_rows.size(), ns_rows.data(), w.data()), "kt_get_match_rows");
      for (size_t i = 0; i < ns_rows.size() && !selector_fails[t]; ++i)
        if (!((w[i * (size_t)Wp + (t >> 5)] >> (t & 31)) & 1)) selector_fails[t] = 1;
    }

    int reconciled = 0;
    std::vector<std::string> changed;
    std::vector<std::pair<std::string, long long>> requeue;
    std::vector<size_t> thr_order(m);
    for (size_t t = 0; t < m; ++t) thr_order[t] = t;
    creation_order(thr_order);
    for (size_t t : thr_order) {
      ThrottleObj& o = throttles[t];
      if (!o.live || o.throttler_name != name) continue;   // only responsible throttles are ever enqueued (:403-425)
      if (selector_fails[t]) continue;                      // affectedPods fails -> reconcile returns the error, status untouched
      ++reconciled;
      const int32_t q = pos[t];  // >= 0: the device says its status changes (or the object was applied since its last reconcile)
      if (q >= 0) {
      o.host_dirty = false;
      ResAmount nu;  // used := ResourceAmount{}; used = used.Add(ResourceAmountOfPod(p)) ...
      if (used_present[q] & KT_COUNT_BIT) {
        nu.has_counts = true;
        nu.pod = used_cnt[q];
        nu.requests_nil = false;
        for (int r = 0; r < (int)cols.size(); ++r)
          if ((used_present[q] >> r) & 1) nu.requests[r] = from_scale(r, used[(size_t)r * k + q]);
      }
      ResAmount nc;  // CalculateThreshold(now).Threshold
      nc.has_counts = calc_present[q] & KT_COUNT_BIT;
      nc.pod = nc.has_counts ? calc_cnt[q] : 0;
      nc.requests_nil = false;
      for (int r = 0; r < (int)cols.size(); ++r)
        if ((calc_present[q] >> r) & 1) nc.requests[r] = from_scale(r, calc_thr[(size_t)r * k + q]);
      if (!ovr_active[q]) nc = o.threshold;  // no active override: spec.threshold itself (keeps nil-ness and spelling)
      const std::vector<std::string> msgs = override_messages(o);
      bool status_changed = false;
      if (!amount_equal(o.st_calc, nc) || o.st_messages != msgs) {  // Q6: otherwise the old calculatedAt is kept
        o.st_calc = nc;
        o.st_calc_at_set = true;
        o.st_calc_at = now.sec;
        o.st_messages = msgs;
        status_changed = true;
      }
      // newStatus.Throttled = CalculatedThreshold.Threshold.IsThrottled(Used, true): one entry per threshold resource
      const bool thr_pod = throttled[q] & KT_COUNT_BIT;
      std::map<int, bool> thr_req;
      for (auto& kv : o.st_calc.requests) thr_req[kv.first] = (throttled[q] >> kv.first) & 1;
      const bool thr_nil = o.st_calc.requests.empty();
      if (thr_pod != o.st_thr_pod || thr_req != o.st_thr_req) status_changed = true;
      // apiequality.Semantic.DeepEqual (throttle_controller.go:157): an empty map IS a nil map -- a status that differs from the
      // informer copy in nil-ness only is not written, and the copy keeps its own (found by a third random event stream, with
      // statuses arriving through the informer: `used: {resourceRequests: {}}` on a throttle that matches no pod)
      if (!amount_equal(o.st_used, nu)) status_changed = true;
      if (status_changed) {  // UpdateStatus(newStatus): the whole of it replaces the copy
        o.st_thr_pod = thr_pod;
        o.st_thr_req = thr_req;
        o.st_thr_req_nil = thr_nil;
        o.st_used = nu;
      }
      o.metrics_pending = true;  // both branches of the status comparison record (throttle_controller.go:159,187); see record_metrics
      if (status_changed) {
        changed.push_back(o.nn());
        throttle_state_changed(t);  // PreFilter reads this status: cached verdicts of the pods it affects are void
        status_dirty = true;
      }
      }  // (q >= 0)
      __int128 after = 0;
      if (next_override_happens_in(o, now, &after)) requeue.emplace_back(o.nn(), (long long)(after > INT64_MAX ? INT64_MAX : after));
      // unreserveAffectedPods: every affected pod the informer has observed leaves the reservation cache -- except, for a
      // Throttle, the finished ones the reference's list loses (Q8)
      auto it = cache[o.kind].by_thr.find(o.nn());
      if (it != cache[o.kind].by_thr.end()) {
        int64_t last_fin = -2;  // computed on first need
        for (size_t i = 0; i < rows.size(); ++i) {
          if (!((words[i * (size_t)Wp + (t >> 5)] >> (t & 31)) & 1)) continue;
          if (o.kind == KT_KIND_THROTTLE && row_finished[i]) {
            if (last_fin == -2) last_fin = last_finished_match(t, o.ns);
            if (rows[i] != last_fin) continue;
          }
          if (it->second.erase(row_pod[i])) reservation_changed(t);
        }
      }
    }
    w.key("reconciled").num(reconciled).key("changed").begin_arr();
    for (auto& c : changed) w.str(c);
    w.end_arr();
    w.key("requeueAfterNanos").begin_obj();  // enqueueAfter(thr, *nextOverrideHappensIn)
    for (auto& r : requeue) w.key(r.first).num(r.second);
    w.end_obj().end_obj();
    return w.out;
  }

  // ---- pending pods: one device pass for a batch ----------------------------------------------------------
  struct RowView {  // one pending pod's share of a pass: affectedThrottles row, 2-bit check codes, admit bit
    const uint32_t* bitmap;
    const uint32_t* codes;
    uint8_t admit;
    int Wp;
  };
  struct PendingResult {
    std::vector<uint32_t> bitmap, codes;
    std::vector<uint8_t> admit;
    int Wp = 0;
    RowView row(size_t i) const { return RowView{bitmap.data() + i * (size_t)Wp, codes.data() + i * 2 * (size_t)Wp, admit.empty() ? (uint8_t)1 : admit[i], Wp}; }
  };
  // The device's PENDING table = the resident queue rows + `k` scratch rows holding `batch` (pods that are not in the informer
  // cache).  Brings it up to date with row deltas; a full upload only when a capacity grows or the packing changed.
  void sync_pending(const std::vector<PodObj>& batch) {
    const int L = lim.label_slots, R = lim.n_resources;
    const int64_t k = (int64_t)batch.size();
    int64_t want_q = std::max<int64_t>(64, pend_capacity), want_s = std::max<int64_t>(16, scratch_capacity);
    while (want_q < (int64_t)pend_pod.size()) want_q *= 2;
    while (want_s < k) want_s *= 2;
    if (want_q != pend_capacity || want_s != scratch_capacity) pend_full_upload = true;
    PodObj tomb;
    auto queue_pod = [&](int64_t row) -> const PodObj& {
      const int64_t slot = row < (int64_t)pend_pod.size() ? pend_pod[(size_t)row] : -1;
      return slot >= 0 ? pods[(size_t)slot] : tomb;
    };
    if (pend_full_upload) {
      const size_t n = (size_t)(want_q + want_s);
      std::vector<int64_t> lab((size_t)L * n), req((size_t)R * n);
      std::vector<uint32_t> present(n), flags(n);
      std::vector<int32_t> nsid(n);
      for (int64_t i = 0; i < want_q; ++i) pack_pod(queue_pod(i), lab, req, present, flags, nsid, n, (size_t)i);
      for (int64_t i = 0; i < want_s; ++i) pack_pod(i < k ? batch[(size_t)i] : tomb, lab, req, present, flags, nsid, n, (size_t)(want_q + i));
      if (namespaces_dirty || throttles_dirty) { sync_all(); sync_status(); sync_reserved(); }  // packing introduced new namespace ids
      check(kt_upload_pods(ctx, KT_PODS_PENDING, (int64_t)n, lab.data(), req.data(), present.data(), flags.data(), nsid.data()), "kt_upload_pods(pending)");
      pend_capacity = want_q;
      scratch_capacity = want_s;
      pend_full_upload = false;
      pend_dirty.clear();
      queue.valid = false;
    } else {
      std::vector<int64_t> rows(pend_dirty.begin(), pend_dirty.end());
      const int64_t n_scratch = std::max(k, scratch_used);  // this batch, and what the last one left behind
      for (int64_t i = 0; i < n_scratch; ++i) rows.push_back(pend_capacity + i);
      const size_t n = rows.size();
      if (n) {
        std::vector<int64_t> lab((size_t)L * n), req((size_t)R * n);
        std::vector<uint32_t> present(n), flags(n);
        std::vector<int32_t> nsid(n);
        for (size_t i = 0; i < n; ++i) {
          const int64_t row = rows[i];
          pack_pod(row < pend_capacity ? queue_pod(row) : (row - pend_capacity < k ? batch[(size_t)(row - pend_capacity)] : tomb), lab, req, present, flags, nsid, n, i);
        }
        if (namespaces_dirty || throttles_dirty) { sync_all(); sync_status(); sync_reserved(); }
        check(kt_update_pod_rows(ctx, KT_PODS_PENDING, (int64_t)n, rows.data(), lab.data(), req.data(), present.data(), flags.data(), nsid.data()),
              "kt_update_pod_rows(pending)");
      }
      pend_dirty.clear();
    }
    scratch_used = k;
  }
  // One pass over the PENDING table (queue + scratch rows): PreFilter reads the informer copy of .status; reconcile is a
  // separate event (KT_EVAL_GIVEN_STATUS).  Afterwards the device holds the verdicts of every queue row at this state.
  void run_pending_pass(const std::vector<PodObj>& batch, uint32_t extra_flags) {
    const bool tables_change = throttles_dirty || namespaces_dirty;
    sync_all();
    sync_status();
    sync_reserved();
    if (tables_change) queue.valid = false;
    sync_pending(batch);
    if (throttles.empty()) return;
    check(kt_evaluate(ctx, 0, KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE | extra_flags), "kt_evaluate");
  }
  // Bring the host copy of the queue's verdicts up to date (admit bits, affectedThrottles rows, non-zero check codes).
  void fetch_queue_results() {
    const int Wp = kt_match_words(ctx);
    const size_t n = (size_t)pend_capacity, all = (size_t)(pend_capacity + scratch_capacity);
    queue.Wp = Wp;
    queue.codes.clear();
    queue.dirty.assign((size_t)Wp, 0);
    queue.admit.assign(all, 1);
    queue.bitmap.assign(all * (size_t)Wp, 0);
    if (!throttles.empty()) {
      std::vector<uint32_t> ent((size_t)sparse_cap * 3);
      int64_t cnt = 0;
      check(kt_get_check_sparse(ctx, queue.admit.data(), ent.data(), (int64_t)sparse_cap, &cnt), "kt_get_check_sparse");
      if (cnt > (int64_t)sparse_cap) {  // more rejected pairs than the list holds: the dense rows
        std::vector<uint32_t> dense(all * 2 * (size_t)Wp);
        check(kt_get_check(ctx, dense.data(), nullptr), "kt_get_check");
        for (size_t row = 0; row < n; ++row)
          for (size_t j = 0; j < 2 * (size_t)Wp; ++j)
            if (dense[row * 2 * Wp + j]) queue.codes[(int64_t)row].emplace_back((uint32_t)j, dense[row * 2 * Wp + j]);
      } else {
        for (int64_t i = 0; i < cnt; ++i)
          if (ent[3 * i] < n) queue.codes[(int64_t)ent[3 * i]].emplace_back(ent[3 * i + 1], ent[3 * i + 2]);
      }
      check(kt_get_match_bitmap(ctx, KT_PODS_PENDING, queue.bitmap.data()), "kt_get_match_bitmap");
    }
    queue.admit.resize(n);
    queue.bitmap.resize(n * (size_t)Wp);
    queue.row_ok.assign(n, 1);
    queue.valid = true;
    ++queue.passes;
  }
  uint32_t sparse_cap = 0;
  void ensure_sparse() {
    const uint32_t want = (uint32_t)std::min<int64_t>(4 * (pend_capacity + scratch_capacity) + 1024, (int64_t)1 << 26);
    if (want > sparse_cap) {
      check(kt_set_sparse_check(ctx, (int64_t)want), "kt_set_sparse_check");
      sparse_cap = want;
    }
  }
  // Is the cached verdict of queue row `row` still the truth?
  bool queue_row_current(int64_t row) const {
    if (!queue.valid || throttles_dirty || namespaces_dirty || pend_full_upload) return false;
    if (row < 0 || (size_t)row >= queue.row_ok.size() || !queue.row_ok[(size_t)row] || pend_dirty.count(row)) return false;
    const uint32_t* bm = &queue.bitmap[(size_t)row * (size_t)queue.Wp];
    for (int w = 0; w < queue.Wp; ++w)
      if (bm[w] & queue.dirty[(size_t)w]) return false;
    return true;
  }
  // One pass for the whole resident queue, results cached on the host.
  void refresh_queue() {
    run_pending_pass({}, 0);
    if (!throttles.empty()) {
      const uint32_t before = sparse_cap;
      ensure_sparse();
      if (sparse_cap != before) check(kt_evaluate(ctx, 0, KT_EVAL_GIVEN_STATUS | KT_EVAL_SKIP_RECONCILE), "kt_evaluate");  // the list exists from this pass on
    }
    fetch_queue_results();
  }

  PendingResult check_pending(const std::vector<PodObj>& batch, uint32_t extra_flags) {
    const size_t k = batch.size();
    run_pending_pass(batch, extra_flags);
    PendingResult out;
    out.Wp = kt_match_words(ctx);
    out.bitmap.assign(k * (size_t)out.Wp, 0);
    out.codes.assign(k * 2 * (size_t)out.Wp, 0);
    out.admit.assign(k, 1);
    if (throttles.empty() || k == 0) return out;
    std::vector<int64_t> rows(k);
    for (size_t i = 0; i < k; ++i) rows[i] = pend_capacity + (int64_t)i;
    check(kt_get_check_rows(ctx, (int64_t)k, rows.data(), out.codes.data(), out.admit.data()), "kt_get_check_rows");
    check(kt_get_match_rows(ctx, KT_PODS_PENDING, (int64_t)k, rows.data(), out.bitmap.data()), "kt_get_match_rows");
    return out;
  }
  // PreFilter of a pod of the resident queue: from the cached verdicts when they are current, else after ONE pass that
  // refreshes the whole queue's.
  PendingResult queue_result(int64_t row) {
    if (!queue_row_current(row)) refresh_queue();
    else ++queue.hits;
    PendingResult out;
    out.Wp = queue.Wp;
    out.bitmap.assign(&queue.bitmap[(size_t)row * (size_t)queue.Wp], &queue.bitmap[(size_t)row * (size_t)queue.Wp] + queue.Wp);
    out.codes.assign(2 * (size_t)queue.Wp, 0);
    out.admit.assign(1, queue.admit[(size_t)row]);
    auto it = queue.codes.find(row);
    if (it != queue.codes.end())
      for (auto& e : it->second) out.codes[e.first] = e.second;
    return out;
  }
  std::vector<int> affected(const PendingResult& r, size_t i, int kind) const { return affected(r.row(i), kind); }
  std::vector<int> affected(const RowView& r, int kind) const {  // the set bits of the pod's match row, in column order
    std::vector<int> out;
    const uint32_t* row = r.bitmap;
    for (int w = 0; w < r.Wp; ++w)
      for (uint32_t bits = row[w]; bits; bits &= bits - 1) {
        const size_t t = (size_t)w * 32 + (size_t)__builtin_ctz(bits);
        if (t < throttles.size() && throttles[t].kind == kind) out.push_back((int)t);
      }
    creation_order(out);
    return out;
  }
  // affectedThrottles / affectedClusterThrottles error paths that never reach the device:
  // an invalid podSelector (MatchesToPod returns the error) and a namespace the informer does not know.
  std::string controller_error(const PodObj& pod, const PendingResult& r, size_t i, int kind) { return controller_error(pod, r.row(i), kind); }
  std::string controller_error(const PodObj& pod, const RowView& r, int kind) {
    if (kind == KT_KIND_CLUSTERTHROTTLE) {
      const int id = ns_dict.find(pod.ns);
      if (id < 0 || !namespaces[(size_t)id].exists) return "namespace \"" + pod.ns + "\" not found";  // namespaceInformer.Lister().Get (clusterthrottle_controller.go:273-276)
    }
    if (!broken_valid) {  // the throttles whose podSelector does not convert: usually none, so not a walk over all of them per pod
      broken.clear();
      for (size_t t = 0; t < throttles.size(); ++t)
        if (throttles[t].live && !throttles[t].selector_error().empty()) broken.push_back(t);
      creation_order(broken);
      broken_valid = true;
    }
    for (size_t t : broken) {
      const ThrottleObj& o = throttles[t];
      if (!o.live || o.kind != kind || o.throttler_name != name) continue;
      if (kind == KT_KIND_THROTTLE && o.ns != pod.ns) continue;
      const std::string e = reachable_selector_error(o, pod.ns);
      if (e.empty()) continue;  // no broken term is in this pod's way (ClusterThrottle terms carry their own namespace scope)
      if ((r.bitmap[t >> 5] >> (t & 31)) & 1) continue;  // an earlier, valid term already matched
      return e;
    }
    return "";
  }
  // labels.Selector.Matches on a namespace's labels (the compiled namespaceSelector of a ClusterThrottle term).  Namespaces, not
  // pods: the same evaluation the table compiler does for the device's per-namespace masks (kt_tables.cc ns_term_matches).
  static bool ns_selector_matches(const CompiledSelector& sel, const NamespaceObj& ns) {
    for (auto& rq : sel.reqs) {
      const std::string* val = nullptr;
      for (auto& kv : ns.labels)
        if (kv.first == rq.key) { val = &kv.second; break; }
      const bool in_set = val && std::find(rq.values.begin(), rq.values.end(), *val) != rq.values.end();
      bool ok = false;
      switch (rq.op) {
        case KT_OP_IN: ok = val && in_set; break;
        case KT_OP_NOTIN: ok = !val || !in_set; break;
        case KT_OP_EXISTS: ok = val != nullptr; break;
        default: ok = val == nullptr; break;  // DoesNotExist
      }
      if (!ok) return false;
    }
    return true;
  }
  // The podSelector conversion error a pod of namespace `ns` runs into when MatchesToPod walks o's terms in order, "" if it
  // reaches none: every broken term of a Throttle is in the way of its namespace's pods (throttle_selector.go:30-42); a
  // ClusterThrottle term checks its namespaceSelector FIRST and is skipped where that does not match -- or does not convert,
  // Q9 -- (clusterthrottle_selector.go:71-87).  Whether a valid term BEFORE it already matched the pod is the device's bit.
  std::string reachable_selector_error(const ThrottleObj& o, const std::string& ns) const {
    const NamespaceObj* nso = nullptr;
    if (o.kind == KT_KIND_CLUSTERTHROTTLE) {
      const int id = ns_dict.find(ns);
      if (id < 0 || !namespaces[(size_t)id].exists) return "";
      nso = &namespaces[(size_t)id];
    }
    for (auto& t : o.terms) {
      if (t.pod_sel.error.empty()) continue;
      if (o.kind == KT_KIND_THROTTLE) return t.pod_sel.error;
      if (!t.ns_sel.error.empty()) continue;
      if (ns_selector_matches(t.ns_sel, *nso)) return t.pod_sel.error;
    }
    return "";
  }

  void names_json(Writer& w, const char* key, const std::vector<int>& idx) const {
    w.key(key).begin_arr();
    for (int t : idx) w.str(throttles[(size_t)t].nn());
    w.end_arr();
  }
  std::string join_names(const std::vector<int>& idx) const {
    std::string s;
    for (size_t i = 0; i < idx.size(); ++i) s += (i ? "," : "") + throttles[(size_t)idx[i]].nn();
    return s;
  }
  // plugin.go:148-215
  void prefilter_json(Writer& w, const PodObj& pod, const PendingResult& r, size_t i) { prefilter_json(w, pod, r.row(i)); }
  void prefilter_json(Writer& w, const PodObj& pod, const RowView& r) {
    std::vector<int> bucket[2][4], aff[2];
    std::string err;
    for (int kind = 0; kind < 2 && err.empty(); ++kind) {  // throttleCtr first, then clusterThrottleCtr (plugin.go:153,165)
      err = controller_error(pod, r, kind);
      if (!err.empty()) break;
      aff[kind] = affected(r, kind);
      for (int t : aff[kind]) {
        const uint32_t code = (r.codes[(size_t)t >> 4] >> (2 * (t & 15))) & 3u;
        bucket[kind][code].push_back(t);
      }
    }
    w.begin_obj();
    if (!err.empty()) {
      w.key("code").str("Error").key("reasons").begin_arr().str(err).end_arr().end_obj();
      return;
    }
    const int T = KT_KIND_THROTTLE, C = KT_KIND_CLUSTERTHROTTLE;
    const auto& ex_c = bucket[C][KT_CHECK_POD_REQUESTS_EXCEEDS_THRESHOLD];
    const auto& ex_t = bucket[T][KT_CHECK_POD_REQUESTS_EXCEEDS_THRESHOLD];
    size_t total = 0;
    for (int kind = 0; kind < 2; ++kind)
      for (int c = 1; c < 4; ++c) total += bucket[kind][c].size();
    std::vector<std::string> reasons;
    auto reason = [&](const char* what, const char* status, const std::vector<int>& v) {
      if (!v.empty()) reasons.push_back(std::string(what) + "[" + status + "]=" + join_names(v));
    };
    if (total) {  // fixed order (Q10)
      reason("clusterthrottle", "pod-requests-exceeds-threshold", ex_c);
      reason("throttle", "pod-requests-exceeds-threshold", ex_t);
      reason("clusterthrottle", "active", bucket[C][KT_CHECK_ACTIVE]);
      reason("throttle", "active", bucket[T][KT_CHECK_ACTIVE]);
      reason("clusterthrottle", "insufficient", bucket[C][KT_CHECK_INSUFFICIENT]);
      reason("throttle", "insufficient", bucket[T][KT_CHECK_INSUFFICIENT]);
    }
    w.key("code").str(total ? "UnschedulableAndUnresolvable" : "Success");
    w.key("reasons").begin_arr();
    for (auto& s : reasons) w.str(s);
    w.end_arr();
    if (!ex_c.empty() || !ex_t.empty()) {
      std::vector<int> both = ex_c;
      both.insert(both.end(), ex_t.begin(), ex_t.end());
      w.key("event").begin_obj().key("type").str("Warning").key("reason").str("ResourceRequestsExceedsThrottleThreshold");
      w.key("message").str("It won't be scheduled unless decreasing resource requests or increasing ClusterThrottle/Throttle threshold because its resource "
                           "requests exceeds their thresholds: " + join_names(both));
      w.end_obj();
    }
    const char* ctl[2] = {"throttle", "clusterthrottle"};
    for (int kind = 0; kind < 2; ++kind) {
      w.key(ctl[kind]).begin_obj();
      names_json(w, "active", bucket[kind][KT_CHECK_ACTIVE]);
      names_json(w, "insufficient", bucket[kind][KT_CHECK_INSUFFICIENT]);
      names_json(w, "podRequestsExceedsThreshold", bucket[kind][KT_CHECK_POD_REQUESTS_EXCEEDS_THRESHOLD]);
      names_json(w, "affected", aff[kind]);
      w.end_obj();
    }
    w.end_obj();
  }

  // Reserve / UnReserve (throttle_controller.go:271-331): the pod's affected throttles come from the device
  std::string reserve_json(const Node& pod_node, bool reserve) {
    PodObj pod = pod_from(pod_node);
    PendingResult r = check_pending({pod}, 0);
    return reserve_result(pod, r.row(0), reserve);
  }
  std::string reserve_result(const PodObj& pod, const RowView& r, bool reserve) {
    std::vector<std::string> errs;
    const char* ctl[2] = {"ThrottleController", "ClusterThrottleController"};
    for (int kind = 0; kind < 2; ++kind) {
      const std::string e = controller_error(pod, r, kind);
      if (!e.empty()) {
        errs.push_back(std::string(reserve ? "Failed to reserve pod=" : "Failed to unreserve pod ") + pod.nn() + " in " + ctl[kind] + ": " + e);
        continue;
      }
      for (int t : affected(r, kind)) {
        if (reserve) cache[kind].add(throttles[(size_t)t].nn(), pod);
        else cache[kind].remove(throttles[(size_t)t].nn(), pod.nn());
        reservation_changed((size_t)t);
      }
    }
    Writer w;
    w.begin_obj();
    if (reserve && !errs.empty()) {  // Reserve aggregates into one Error status; Unreserve only logs (plugin.go:223-235,246-254)
      w.key("code").str("Error").key("reasons").begin_arr();
      for (auto& e : errs) w.str(e);
      w.end_arr();
    } else {
      w.key("code").str("Success");
    }
    w.end_obj();
    return w.out;
  }

  // ---- the same calls for pods of the resident queue, addressed by key ----------------------------------------
  const PodObj& informer_pod(const std::string& ns, const std::string& pname) const {
    auto it = pod_index.find(ns + "/" + pname);
    if (it == pod_index.end()) fail("pod " + ns + "/" + pname + " is not in the informer cache");
    return pods[(size_t)it->second];
  }
  std::string pre_filter_key(const std::string& ns, const std::string& pname) {
    const PodObj pod = informer_pod(ns, pname);  // (value copy: a pass may re-create the engine and re-pack)
    Writer w;
    if (pod.pend_row < 0) {  // known to the informer but not waiting to be scheduled: checked like a manifest
      PendingResult r = check_pending({pod}, 0);
      prefilter_json(w, pod, r.row(0));
    } else {
      PendingResult r = queue_result(pod.pend_row);
      prefilter_json(w, pod, r.row(0));
    }
    return w.out;
  }
  std::string reserve_key(const std::string& ns, const std::string& pname, bool reserve) {
    const PodObj pod = informer_pod(ns, pname);
    // which throttles the pod affects does not depend on statuses or reservations: the cached row serves as long as the pod's
    // own row and the tables are what they were
    PendingResult r = pod.pend_row >= 0 ? queue_result(pod.pend_row) : check_pending({pod}, 0);
    return reserve_result(pod, r.row(0), reserve);
  }
  // PreFilter of the WHOLE resident queue: one verdict byte per queue row (0 free row, 1 Success, 2 UnschedulableAndUnresolvable,
  // 3 Error); at most one device pass, none when every cached verdict is current.
  int64_t pre_filter_queue(uint8_t* verdicts, int64_t cap) {
    const int64_t n = (int64_t)pend_pod.size();
    bool current = queue.valid;
    for (int64_t row = 0; row < n && current; ++row)
      if (pend_pod[(size_t)row] >= 0 && !queue_row_current(row)) current = false;
    if (!current) refresh_queue();
    else ++queue.hits;
    if (!broken_valid) { PendingResult none; none.Wp = queue.Wp; none.bitmap.assign((size_t)queue.Wp, 0); none.codes.assign(2 * (size_t)queue.Wp, 0); controller_error(PodObj(), none.row(0), KT_KIND_THROTTLE); }
    const std::vector<uint32_t> no_codes(2 * (size_t)queue.Wp, 0);
    for (int64_t row = 0; row < n && row < cap; ++row) {
      const int64_t slot = pend_pod[(size_t)row];
      if (slot < 0) { verdicts[row] = 0; continue; }
      uint8_t v = queue.admit[(size_t)row] ? 1 : 2;
      const PodObj& pod = pods[(size_t)slot];
      const int nsid = ns_dict.find(pod.ns);
      if (!broken.empty() || nsid < 0 || !namespaces[(size_t)nsid].exists) {  // the error paths that never reach the device
        const RowView rv{&queue.bitmap[(size_t)row * (size_t)queue.Wp], no_codes.data(), queue.admit[(size_t)row], queue.Wp};
        if (!controller_error(pod, rv, KT_KIND_THROTTLE).empty() || !controller_error(pod, rv, KT_KIND_CLUSTERTHROTTLE).empty()) v = 3;
      }
      verdicts[row] = v;
    }
    return n;
  }

  // ---- queue-ordered admission on the device (kt_admit_queue, csrc/kt_admit.cuh) ------------------------------
  bool admit_queue_on_device_possible(const std::vector<PodObj>& queue) {
    if (throttles.empty() || queue.empty()) return false;
    if (!broken_valid) {
      broken.clear();
      for (size_t t = 0; t < throttles.size(); ++t)
        if (throttles[t].live && !throttles[t].selector_error().empty()) broken.push_back(t);
      creation_order(broken);
      broken_valid = true;
    }
    if (!broken.empty()) return false;  // some pod may run into a conversion error: framework.Error, no Reserve
    // Reserve is idempotent per pod (podResourceAmountMap.add overwrites, reserved_resource_amounts.go:131-136): a queue pod that
    // already holds a reservation -- reserved in an earlier cycle and neither bound-and-observed nor unreserved since -- or that
    // stands in the queue twice adds NOTHING when it is admitted again, whereas the device's prefix sums would count its requests
    // a second time for everybody behind it.  Such queues take the pod-by-pod passes of the host (found by the event-stream chaos
    // test, seed 171: a bound pod's old pending manifest back in the queue).
    {
      std::unordered_set<std::string> holders;
      for (int kind = 0; kind < 2; ++kind)
        for (auto& thr : cache[kind].by_thr)
          for (auto& pod : thr.second) holders.insert(pod.first);
      for (auto& p : queue)
        if (!holders.insert(p.nn()).second) return false;
    }
    for (auto& p : queue) {
      const int id = ns_dict.find(p.ns);
      if (id < 0 || !namespaces[(size_t)id].exists) return false;  // "namespace not found": Error as well
    }
    return true;
  }
  std::string admit_queue_on_device(const std::vector<PodObj>& queue) {
    const size_t n = queue.size();
    sync_all();
    sync_status();
    sync_reserved();
    sync_pending(queue);
    if (namespaces_dirty || throttles_dirty || status_dirty || reserved_dirty) { sync_all(); sync_status(); sync_reserved(); }
    int32_t rounds = 0;
    int64_t admitted_dev = 0;
    check(kt_admit_queue(ctx, pend_capacity, (int64_t)n, 0, &rounds, &admitted_dev), "kt_admit_queue");
    PendingResult r;
    r.Wp = kt_match_words(ctx);
    r.bitmap.assign(n * (size_t)r.Wp, 0);
    r.codes.assign(n * 2 * (size_t)r.Wp, 0);
    r.admit.assign(n, 1);
    std::vector<int64_t> rows(n);
    for (size_t i = 0; i < n; ++i) rows[i] = pend_capacity + (int64_t)i;
    check(kt_get_check_rows(ctx, (int64_t)n, rows.data(), r.codes.data(), r.admit.data()), "kt_get_check_rows");
    check(kt_get_match_rows(ctx, KT_PODS_PENDING, (int64_t)n, rows.data(), r.bitmap.data()), "kt_get_match_rows");
    Writer out;
    int admitted = 0;
    std::vector<std::string> results(n);
    for (size_t i = 0; i < n; ++i) {
      Writer w;
      prefilter_json(w, queue[i], r.row(i));
      results[i] = w.out;
      const bool success = w.out.compare(0, 17, "{\"code\":\"Success\"") == 0;
      if (success != (r.admit[i] != 0)) fail("kt_admit_queue: the admit bit of " + queue[i].nn() + " contradicts its check codes");
      if (!success) continue;
      // Reserve (throttle_controller.go:271-292): ResourceAmountOfPod joins the reservation of every affected throttle -- what
      // the device already counted for the pods behind this one
      ++admitted;
      for (int kind = 0; kind < 2; ++kind)
        for (int t : affected(r.row(i), kind)) { cache[kind].add(throttles[(size_t)t].nn(), queue[i]); reservation_changed((size_t)t); }
    }
    if ((int64_t)admitted != admitted_dev) fail("kt_admit_queue: admitted count mismatch");
    out.begin_obj().key("rounds").num(rounds).key("admitted").num(admitted).key("onDevice").raw("true").key("results").begin_arr();
    for (size_t i = 0; i < n; ++i) out.begin_obj().key("pod").str(queue[i].nn()).key("round").num(0).key("preFilter").raw(results[i]).end_obj();
    out.end_arr().end_obj();
    return out.out;
  }

  // ---- queue-ordered admission ----------------------------------------------------------------------------
  // The scheduler admits one pod per cycle: PreFilter, and on Success Reserve, so every admitted pod raises the reserved
  // amounts the NEXT pod is checked against (plugin.go:148-238).  For a sorted queue that sequence is reproduced exactly
  // with far fewer device passes than pods: one pass checks every undecided pod against the current reservations; going
  // through them in queue order, a pod's verdict is FINAL unless one of its affected throttles was reserved on by an
  // earlier pod of this very pass or is shared with an earlier pod that is itself still undecided -- those pods wait
  // for the next pass.  The first undecided pod is always final, so the loop terminates; pods that touch disjoint sets of
  // throttles are decided together.
  std::string admit_queue(const Node& arr) {
    if (!arr.is(Node::Arr)) fail("expected a JSON array of pods");
    std::vector<PodObj> queue;
    for (auto& e : arr.arr) queue.push_back(pod_from(*e));
    const size_t n = queue.size();
    if (admit_queue_on_device_possible(queue)) return admit_queue_on_device(queue);
    // (below: the same semantics with host-orchestrated passes -- kept for queues the device fixpoint does not take: a pod that
    // PreFilter answers with Error must not be reserved)
    std::vector<std::string> results(n);
    std::vector<int> round_of(n, 0);
    std::vector<size_t> undecided(n);
    for (size_t i = 0; i < n; ++i) undecided[i] = i;
    int rounds = 0, admitted = 0;
    while (!undecided.empty()) {
      ++rounds;
      std::vector<PodObj> batch;
      for (size_t i : undecided) batch.push_back(queue[i]);
      const PendingResult r = check_pending(batch, 0);
      const size_t W = (size_t)r.Wp;
      std::vector<uint32_t> dirty(W, 0);  // throttles whose reservation changed in this pass, or that an undecided earlier pod may still change
      std::vector<size_t> next;
      for (size_t k = 0; k < batch.size(); ++k) {
        const size_t i = undecided[k];
        const uint32_t* row = &r.bitmap[k * W];
        bool clean = true;
        for (size_t w = 0; w < W && clean; ++w) clean = (row[w] & dirty[w]) == 0;
        if (!clean) {  // depends on something not settled yet: decide it in a later pass, and shield what it may change
          for (size_t w = 0; w < W; ++w) dirty[w] |= row[w];
          next.push_back(i);
          continue;
        }
        Writer w;
        prefilter_json(w, batch[k], r, k);
        results[i] = w.out;
        round_of[i] = rounds;
        bool success = w.out.compare(0, 17, "{\"code\":\"Success\"") == 0;
        if (!success) continue;
        // Reserve (throttle_controller.go:271-292): ResourceAmountOfPod joins the reservation of every affected throttle
        bool reserve_error = false;
        for (int kind = 0; kind < 2; ++kind) reserve_error = reserve_error || !controller_error(batch[k], r, k, kind).empty();
        if (reserve_error) continue;
        ++admitted;
        for (int kind = 0; kind < 2; ++kind)
          for (int t : affected(r, k, kind)) { cache[kind].add(throttles[(size_t)t].nn(), batch[k]); reservation_changed((size_t)t); }
        for (size_t w2 = 0; w2 < W; ++w2) dirty[w2] |= row[w2];
      }
      undecided.swap(next);
    }
    Writer out;
    out.begin_obj().key("rounds").num(rounds).key("admitted").num(admitted).key("results").begin_arr();
    for (size_t i = 0; i < n; ++i) {
      out.begin_obj().key("pod").str(queue[i].nn()).key("round").num(round_of[i]).key("preFilter").raw(results[i]).end_obj();
    }
    out.end_arr().end_obj();
    return out.out;
  }

  // ---- informer events --------------------------------------------------------------------------------
  void apply_pod(const Node& v) {
    PodObj p = pod_from(v);
    auto it = pod_index.find(p.nn());
    if (it == pod_index.end()) {
      const int64_t row = alloc_row(p.ns);
      p.row = row;
      p.seq = next_pod_seq++;
      pod_index[p.nn()] = row;
      totals_add(p, +1);
      pods[(size_t)row] = std::move(p);
      dirty_rows.insert(row);
      queue_update(row);
      return;
    }
    // The informer's copy is replaced FIRST: the pass below only asks which throttles the old and the new pod match, which
    // does not depend on the running rows, and an update that repairs a snapshot the packer refuses (column overflow) must
    // not be refused for it.
    const int64_t row = it->second;
    const PodObj old = pods[(size_t)row];
    p.row = row;
    p.seq = old.seq;
    p.pend_row = old.pend_row;
    totals_add(old, -1);
    totals_add(p, +1);
    pods[(size_t)row] = std::move(p);
    dirty_rows.insert(row);
    queue_update(row);
    const PodObj& cur = pods[(size_t)row];
    // UpdateFunc (throttle_controller.go:459-507): the throttle assignment can only change with labels / namespace;
    // then the pod's reservation moves from (old \ new) to (new \ old) throttles
    const bool relevant = should_count_in(old) || should_count_in(cur);
    if (relevant && !throttles.empty() && old.labels != cur.labels) {
      const PodObj now = cur;  // check_pending may re-create the engine; keep value copies
      // From here on the update IS committed (pods[row] holds the new object, resource names it brought stay interned): the
      // reference's UpdateFunc cannot refuse an event either -- when it fails to work out the throttles it logs and returns
      // (utilruntime.HandleError, throttle_controller.go:470-483).  A pass that throws (refused snapshot, engine error) is
      // reported as a warning of a SUCCESSFUL apply, and nothing is rolled back.
      apply_committed = true;
      PendingResult r;
      try {
        r = check_pending({old, now}, 0);
      } catch (const std::exception& e) {
        apply_warning = std::string("pod updated; reservation move skipped: ") + e.what();
        return;
      }
      for (int kind = 0; kind < 2; ++kind) {
        if (!controller_error(old, r, 0, kind).empty() || !controller_error(now, r, 1, kind).empty()) continue;  // HandleError + return
        const std::vector<int> a = affected(r, 0, kind), b = affected(r, 1, kind);
        for (int t : a)
          if (std::find(b.begin(), b.end(), t) == b.end()) { cache[kind].remove(throttles[(size_t)t].nn(), now.nn()); reservation_changed((size_t)t); }
        for (int t : b)
          if (std::find(a.begin(), a.end(), t) == a.end()) { cache[kind].add(throttles[(size_t)t].nn(), now); reservation_changed((size_t)t); }
      }
    }
  }
  void delete_pod(const std::string& ns, const std::string& pname) {
    auto it = pod_index.find(ns + "/" + pname);
    if (it == pod_index.end()) return;
    const int64_t row = it->second;
    const PodObj old = pods[(size_t)row];
    // the row goes first (see apply_pod): a delete that repairs a refused snapshot must not be refused for it
    totals_add(old, -1);
    if (old.pend_row >= 0) queue_release(old.pend_row);
    pods[(size_t)row] = PodObj();  // tombstone row: flags == 0, no labels
    pods[(size_t)row].row = row;
    pod_index.erase(it);
    ns_free_rows[old.ns].push_back(row);  // the slot stays with its namespace's arena
    dirty_rows.insert(row);
    // DeleteFunc (:509-515): a scheduled pod that disappears is un-reserved from its affected throttles
    if (should_count_in(old) && !old.node_name.empty() && !throttles.empty()) {
      PendingResult r;
      try {
        r = check_pending({old}, 0);
      } catch (...) {
        // the pod is gone whatever happens to the pass: its reservations must not outlive it (reconcile only un-reserves pods
        // that are still in the index) -- without the device's answer it leaves every throttle's reservation, a superset
        for (int kind = 0; kind < 2; ++kind)
          if (cache[kind].remove_everywhere(old.nn())) { reserved_dirty = true; queue_void(); }
        throw;
      }
      for (int kind = 0; kind < 2; ++kind) {
        if (!controller_error(old, r, 0, kind).empty()) continue;
        for (int t : affected(r, 0, kind))
          if (cache[kind].remove(throttles[(size_t)t].nn(), old.nn())) reservation_changed((size_t)t);
      }
    }
  }
  void apply_namespace(const Node& v) {
    const std::string nm = v["metadata"]["name"].str();
    const Node& lab = v["metadata"]["labels"];
    // refuse before touching any state: the object is rejected, the plugin stays usable
    if ((int)lab.obj.size() > KT_MAX_LABEL_SLOTS - 1)  // one slot is the internal "exists" label
      fail("namespace " + nm + " has more than " + std::to_string(KT_MAX_LABEL_SLOTS - 1) + " labels");
    const int32_t id = ns_id(nm);
    NamespaceObj& n = namespaces[(size_t)id];
    n.exists = true;
    n.labels.clear();
    for (auto& kv : lab.obj) n.labels.emplace_back(kv.first, kv.second->str());
    if ((int)n.labels.size() > max_ns_labels) {
      max_ns_labels = (int)n.labels.size();
      if (ctx && max_ns_labels + 1 > lim.ns_label_slots) drop_engine();
    }
    namespaces_dirty = true;
  }
  void apply_throttle(const Node& v, int kind) {
    ThrottleObj o;
    o.kind = kind;
    const Node& md = v["metadata"];
    o.ns = kind == KT_KIND_THROTTLE ? md["namespace"].str() : "";
    o.name = md["name"].str();
    o.uid = md["uid"].str();
    const Node& spec = v["spec"];
    o.throttler_name = spec["throttlerName"].str();
    o.threshold = res_amount(spec["threshold"]);
    for (auto& ov : spec["temporaryThresholdOverrides"].arr) {
      Override x;
      x.begin = (*ov)["begin"].str();
      x.end = (*ov)["end"].str();
      x.threshold = res_amount((*ov)["threshold"]);
      o.overrides.push_back(std::move(x));
    }
    // the reference's JSON tag is "selectorTerms" (throttle_selector.go:26)
    for (auto& t : spec["selector"]["selectorTerms"].arr) {
      Term term;
      term.pod_sel = compile_selector((*t)["podSelector"]);
      if (kind == KT_KIND_CLUSTERTHROTTLE) term.ns_sel = compile_selector((*t)["namespaceSelector"]);
      o.terms.push_back(std::move(term));
    }
    o.live = true;
    // the status the manifest carries, parsed BEFORE anything is committed: a manifest that is refused leaves no trace
    const Node& st = v["status"];
    const bool has_status = st.is(Node::Obj);
    if (has_status) {
      const Node& ct = st["calculatedThreshold"];
      o.st_calc = res_amount(ct["threshold"]);
      o.st_calc_at_set = false;
      o.st_calc_at = 0;
      if (ct["calculatedAt"].is(Node::Str) && !ct["calculatedAt"].text.empty()) {
        GoTime at;
        const std::string e = parse_rfc3339(ct["calculatedAt"].text, &at);
        if (!e.empty()) fail(e);
        o.st_calc_at_set = !at.zero;
        o.st_calc_at = at.sec;
      }
      for (auto& mnode : ct["messages"].arr) o.st_messages.push_back(mnode->str());
      o.st_thr_pod = st["throttled"]["resourceCounts"]["pod"].boolean(false);
      o.st_thr_req_nil = !st["throttled"]["resourceRequests"].is(Node::Obj);
      for (auto& kv : st["throttled"]["resourceRequests"].obj) o.st_thr_req[column(kv.first)] = kv.second->boolean(false);
      o.st_used = res_amount(st["used"]);
    }
    const std::string key = std::string(kind == KT_KIND_THROTTLE ? "T:" : "C:") + o.nn();
    auto it = thr_index.find(key);
    if (it == thr_index.end()) {
      o.seq = ++thr_seq;
      if (!free_thr.empty()) {  // the column of a deleted throttle (everything per column is re-uploaded: throttles_dirty below)
        const int t = free_thr.back();
        free_thr.pop_back();
        thr_index[key] = t;
        throttles[(size_t)t] = std::move(o);
        thr_reused = true;
      } else {
        thr_index[key] = (int)throttles.size();
        throttles.push_back(std::move(o));
      }
    } else {  // spec update: the status subresource is kept unless the manifest carries one
      ThrottleObj& old = throttles[(size_t)it->second];
      o.seq = old.seq;
      if (old.metrics_pending) record_metrics(old);  // the gauges keep the values of the last reconcile, not of this update
      if (!has_status) {
        o.st_calc = old.st_calc; o.st_calc_at_set = old.st_calc_at_set; o.st_calc_at = old.st_calc_at; o.st_messages = old.st_messages;
        o.st_thr_pod = old.st_thr_pod; o.st_thr_req = old.st_thr_req; o.st_thr_req_nil = old.st_thr_req_nil; o.st_used = old.st_used;
      }
      old = std::move(o);
    }
    throttles_dirty = status_dirty = reserved_dirty = true;
    broken_valid = false;
  }
  void delete_throttle(int kind, const std::string& ns, const std::string& tname) {
    const std::string nn = (kind == KT_KIND_THROTTLE ? ns : std::string()) + "/" + tname;
    auto it = thr_index.find(std::string(kind == KT_KIND_THROTTLE ? "T:" : "C:") + nn);
    if (it == thr_index.end()) return;
    // the column can never match or be reconciled again; the next new throttle takes it over
    ThrottleObj& o = throttles[(size_t)it->second];
    free_thr.push_back(it->second);
    if (o.metrics_pending) { record_metrics(o); o.metrics_pending = false; }  // its series outlive it, as a GaugeVec's do
    o.live = false;
    o.terms.clear();
    // The reservation cache keeps the entry: reserved_resource_amounts.go has no way to drop a throttle, so what was reserved on
    // this name is still counted if a throttle of the same name comes back (until those pods are observed or deleted).
    thr_index.erase(it);
    throttles_dirty = status_dirty = reserved_dirty = true;
    broken_valid = false;
  }

  std::string status_json(const std::string& ns, const std::string& tname) {
    auto it = thr_index.find(ns.empty() ? "C:/" + tname : "T:" + ns + "/" + tname);
    if (it == thr_index.end()) fail("throttle " + ns + "/" + tname + " not found");
    const ThrottleObj& o = throttles[(size_t)it->second];
    Writer w;
    w.begin_obj().key("calculatedThreshold").begin_obj().key("threshold");
    amount_json(w, o.st_calc);
    w.key("calculatedAtSet").boolean(o.st_calc_at_set).key("calculatedAtUnix").num(o.st_calc_at);
    if (!o.st_messages.empty()) {
      w.key("messages").begin_arr();
      for (auto& s : o.st_messages) w.str(s);
      w.end_arr();
    }
    w.end_obj();
    w.key("throttled").begin_obj().key("resourceCounts").begin_obj().key("pod").boolean(o.st_thr_pod).end_obj();
    if (!o.st_thr_req_nil) {
      w.key("resourceRequests").begin_obj();
      for (auto& kv : o.st_thr_req) w.key(cols[(size_t)kv.first].name).boolean(kv.second);
      w.end_obj();
    }
    w.end_obj();
    w.key("used");
    amount_json(w, o.st_used);
    w.end_obj();
    return w.out;
  }
  // ---- the status subresource exactly as the reference's UpdateStatus would send it (encoding/json of v1alpha1.ThrottleStatus:
  // throttle_types.go:113-117, resource_amount.go:27-44, calculated_threshold.go:24-30): struct fields in declaration order,
  // map keys sorted, nil / empty maps and nil counts omitted, quantities in their canonical spelling (Quantity.String), the
  // zero time as null.
  void amount_manifest(Writer& w, const ResAmount& a, bool column_format) const {
    w.begin_obj();
    if (a.has_counts) w.key("resourceCounts").begin_obj().key("pod").num(a.pod).end_obj();
    if (!a.requests.empty()) {
      std::map<std::string, std::string> byname;
      for (auto& kv : a.requests) {
        const ResourceColumn& c = cols[(size_t)kv.first];
        // a parsed quantity keeps its own format; a sum takes the format its first addend had -- the column's, here
        byname[c.name] = kt::canonical_string(kv.second.mant, kv.second.exp, column_format ? c.format : kv.second.format);
      }
      w.key("resourceRequests").begin_obj();
      for (auto& kv : byname) w.key(kv.first).str(kv.second);
      w.end_obj();
    }
    w.end_obj();
  }
  std::string status_manifest_json(const std::string& ns, const std::string& tname) {
    auto it = thr_index.find(ns.empty() ? "C:/" + tname : "T:" + ns + "/" + tname);
    if (it == thr_index.end()) fail("throttle " + ns + "/" + tname + " not found");
    const ThrottleObj& o = throttles[(size_t)it->second];
    Writer w;
    w.begin_obj().key("calculatedThreshold").begin_obj().key("threshold");
    amount_manifest(w, o.st_calc, false);
    w.key("calculatedAt");
    if (o.st_calc_at_set) w.str(format_rfc3339_utc(o.st_calc_at));
    else w.raw("null");
    if (!o.st_messages.empty()) {
      w.key("messages").begin_arr();
      for (auto& m : o.st_messages) w.str(m);
      w.end_arr();
    }
    w.end_obj();
    w.key("throttled").begin_obj().key("resourceCounts").begin_obj().key("pod").boolean(o.st_thr_pod).end_obj();
    if (!o.st_thr_req.empty()) {
      std::map<std::string, bool> byname;
      for (auto& kv : o.st_thr_req) byname[cols[(size_t)kv.first].name] = kv.second;
      w.key("resourceRequests").begin_obj();
      for (auto& kv : byname) w.key(kv.first).boolean(kv.second);
      w.end_obj();
    }
    w.end_obj();
    w.key("used");
    amount_manifest(w, o.st_used, true);
    w.end_obj();
    return w.out;
  }
  std::string reserved_json(int kind, const std::string& nn) {
    Writer w;
    ResAmount total;
    std::vector<std::string> names;
    auto it = cache[kind ? 1 : 0].by_thr.find(nn);
    if (it != cache[kind ? 1 : 0].by_thr.end())
      for (auto& pod : it->second) {  // totalResoruceAmount (:148-156): result = result.Add(ResourceAmountOfPod)
        names.push_back(pod.first);
        total.has_counts = true;
        total.pod += 1;
        total.requests_nil = false;
        for (auto& kv : pod.second) {
          auto f = total.requests.find(kv.first);
          if (f == total.requests.end()) total.requests[kv.first] = kv.second;
          else f->second = kt::quantity_add(f->second, kv.second);
        }
      }
    w.begin_obj().key("amount");
    amount_json(w, total);
    w.key("pods").begin_arr();
    for (auto& n : names) w.str(n);
    w.end_arr().end_obj();
    return w.out;
  }
};

namespace {

template <class F>
const char* guarded(kth_plugin* p, F&& f) {
  if (!p) return ret(err_json("null plugin handle"));
  std::lock_guard<std::mutex> lk(p->mu);
  try {
    return ret(f());
  } catch (const std::exception& e) {
    return ret(err_json(e.what()));
  }
}

// kth_eval: host-only pieces, no device (a scratch plugin supplies the dictionaries)
std::string eval_request(const Node& req) {
  const std::string fn = req["fn"].str();
  kth_plugin scratch;
  Writer w;
  if (fn == "ParseQuantity" || fn == "CanonicalQuantity") {
    const Quantity q = kt::parse_quantity(req["value"].scalar());
    w.begin_obj().key("decimal").str(kt::decimal_string(q)).key("format").num((int)q.format);
    w.key("canonical").str(kt::canonical_string(q.mant, q.exp, q.format)).end_obj();
    return w.out;
  }
  if (fn == "PodRequestResourceList" || fn == "ResourceAmountOfPod") {
    const PodObj p = scratch.pod_from(req["pod"]);
    ResAmount a;
    a.requests_nil = false;
    a.requests = p.request;
    if (fn == "ResourceAmountOfPod") { a.has_counts = true; a.pod = 1; }
    if (fn == "PodRequestResourceList") {
      w.begin_obj();
      for (auto& kv : a.requests) w.key(scratch.cols[(size_t)kv.first].name).str(kt::decimal_string(kv.second));
      w.end_obj();
    } else {
      scratch.amount_json(w, a);
    }
    return w.out;
  }
  if (fn == "ParseRFC3339") {
    GoTime t;
    const std::string e = parse_rfc3339(req["value"].str(), &t);
    w.begin_obj();
    if (!e.empty()) w.key("error").str(e);
    w.key("unix").num(t.sec).key("nsec").num(t.nsec).end_obj();
    return w.out;
  }
  if (fn == "OverrideMessages") {
    scratch.apply_throttle(req["throttle"], req["throttle"]["kind"].str("Throttle") == "ClusterThrottle" ? KT_KIND_CLUSTERTHROTTLE : KT_KIND_THROTTLE);
    w.begin_arr();
    for (auto& s : kth_plugin::override_messages(scratch.throttles[0])) w.str(s);
    w.end_arr();
    return w.out;
  }
  if (fn == "NextOverrideHappensIn") {
    scratch.apply_throttle(req["throttle"], req["throttle"]["kind"].str("Throttle") == "ClusterThrottle" ? KT_KIND_CLUSTERTHROTTLE : KT_KIND_THROTTLE);
    GoTime now;
    const std::string e = parse_rfc3339(req["now"].str(), &now);
    if (!e.empty()) fail(e);
    __int128 d = 0;
    const bool have = kth_plugin::next_override_happens_in(scratch.throttles[0], now, &d);
    w.begin_obj().key("have").boolean(have).key("nanos").num((long long)d).end_obj();
    return w.out;
  }
  if (fn == "ThrottleMetrics") {  // recordThrottleMetrics / recordClusterThrottleMetrics of one manifest (spec + status)
    scratch.apply_throttle(req["throttle"], req["throttle"]["kind"].str("Throttle") == "ClusterThrottle" ? KT_KIND_CLUSTERTHROTTLE : KT_KIND_THROTTLE);
    scratch.record_metrics(scratch.throttles[0]);
    w.begin_obj().key("text").str(scratch.metrics_text()).end_obj();
    return w.out;
  }
  if (fn == "FormatFloat") {
    w.begin_obj().key("text").str(kth_plugin::go_float(std::strtod(req["value"].scalar().c_str(), nullptr))).end_obj();
    return w.out;
  }
  if (fn == "ScaledValue") {
    w.begin_obj().key("value").num((long long)kt::quantity_scaled_value(kt::parse_quantity(req["value"].scalar()), (int)req["scale"].integer(0))).end_obj();
    return w.out;
  }
  if (fn == "ValidateSelector") {
    const CompiledSelector c = compile_selector(req["selector"]);
    w.begin_obj().key("valid").boolean(c.error.empty());
    if (!c.error.empty()) w.key("error").str(c.error);
    w.key("requirements").num((long long)c.reqs.size()).end_obj();
    return w.out;
  }
  fail("unknown fn: " + fn);
}

}  // namespace

extern "C" {

int kth_new_plugin(kth_plugin** out, const char* args_json, int device) {
  if (!out) return KT_ERR_INVALID;
  *out = nullptr;
  try {
    ktjson::NodePtr args = ktjson::parse(args_json ? args_json : "{}");
    // DecodePluginArgs (plugin_args.go:42-60): name and targetSchedulerName are required
    const std::string nm = (*args)["name"].str(), target = (*args)["targetSchedulerName"].str();
    if (nm.empty()) { g_new_plugin_error = "Name must not be empty"; return KT_ERR_INVALID; }
    if (target.empty()) { g_new_plugin_error = "TargetSchedulerName must not be empty"; return KT_ERR_INVALID; }
    kth_plugin* p = new kth_plugin();
    p->name = nm;
    p->target_scheduler = target;
    p->device = device;
    try {
      p->ensure_engine();  // fail at construction, like NewPlugin does when its controllers cannot start
    } catch (const std::exception& e) {
      g_new_plugin_error = e.what();
      delete p;
      return KT_ERR_CUDA;
    }
    p->drop_engine();  // created again with the right limits once objects arrive
    *out = p;
    return KT_OK;
  } catch (const std::exception& e) {
    g_new_plugin_error = e.what();
    return KT_ERR_INVALID;
  }
}
const char* kth_new_plugin_error(void) { return g_new_plugin_error.c_str(); }
void kth_free(kth_plugin* p) {
  if (!p) return;
  if (p->ctx) kt_destroy(p->ctx);
  delete p;
}

const char* kth_apply(kth_plugin* p, const char* manifest_json) {
  return guarded(p, [&]() -> std::string {
    ktjson::NodePtr v = ktjson::parse(manifest_json);
    const std::string kind = (*v)["kind"].str();
    const size_t n_cols = p->cols.size();
    p->apply_committed = false;
    p->apply_warning.clear();
    try {
      if (kind == "Pod") p->apply_pod(*v);
      else if (kind == "Namespace") p->apply_namespace(*v);
      else if (kind == "Throttle") p->apply_throttle(*v, KT_KIND_THROTTLE);
      else if (kind == "ClusterThrottle") p->apply_throttle(*v, KT_KIND_CLUSTERTHROTTLE);
      else fail("unsupported kind: " + kind);
    } catch (...) {
      if (!p->apply_committed) p->rollback_columns(n_cols);  // the refused object's resource names go with it
      throw;
    }
    if (!p->apply_warning.empty()) {
      Writer w;
      w.begin_obj().key("ok").raw("true").key("warning").str(p->apply_warning).end_obj();
      return w.out;
    }
    return "{\"ok\":true}";
  });
}
const char* kth_delete(kth_plugin* p, const char* kind, const char* ns, const char* name) {
  return guarded(p, [&]() -> std::string {
    const std::string k = kind ? kind : "", n = ns ? ns : "", nm = name ? name : "";
    if (k == "Pod") p->delete_pod(n, nm);
    else if (k == "Throttle") p->delete_throttle(KT_KIND_THROTTLE, n, nm);
    else if (k == "ClusterThrottle") p->delete_throttle(KT_KIND_CLUSTERTHROTTLE, "", nm);
    else if (k == "Namespace") {
      const int id = p->ns_dict.find(nm);
      if (id >= 0) { p->namespaces[(size_t)id].exists = false; p->namespaces[(size_t)id].labels.clear(); p->namespaces_dirty = true; }
    } else fail("unsupported kind: " + k);
    return "{\"ok\":true}";
  });
}
const char* kth_reconcile_all(kth_plugin* p, const char* now_rfc3339) {
  return guarded(p, [&]() { return p->reconcile_all(now_rfc3339 ? now_rfc3339 : ""); });
}
const char* kth_get_status(kth_plugin* p, const char* ns, const char* name) {
  return guarded(p, [&]() { return p->status_json(ns ? ns : "", name ? name : ""); });
}
const char* kth_get_status_manifest(kth_plugin* p, const char* ns, const char* name) {
  return guarded(p, [&]() -> std::string { return p->status_manifest_json(ns ? ns : "", name ? name : ""); });
}
const char* kth_pre_filter(kth_plugin* p, const char* pod_json) {
  return guarded(p, [&]() {
    ktjson::NodePtr v = ktjson::parse(pod_json);
    p->check_only_names = true;
    std::vector<PodObj> batch;
    try { batch.push_back(p->pod_from(*v)); } catch (...) { p->check_only_names = false; throw; }
    p->check_only_names = false;
    kth_plugin::PendingResult r = p->check_pending(batch, 0);  // PreFilter passes isThrottledOnEqual = false
    Writer w;
    p->prefilter_json(w, batch[0], r, 0);
    return w.out;
  });
}
const char* kth_pre_filter_key(kth_plugin* p, const char* ns, const char* name) {
  return guarded(p, [&]() { return p->pre_filter_key(ns ? ns : "", name ? name : ""); });
}
const char* kth_reserve_key(kth_plugin* p, const char* ns, const char* name) {
  return guarded(p, [&]() { return p->reserve_key(ns ? ns : "", name ? name : "", true); });
}
const char* kth_unreserve_key(kth_plugin* p, const char* ns, const char* name) {
  return guarded(p, [&]() { return p->reserve_key(ns ? ns : "", name ? name : "", false); });
}
int64_t kth_pod_row(kth_plugin* p, const char* ns, const char* name) {
  if (!p) return -1;
  std::lock_guard<std::mutex> lk(p->mu);
  auto it = p->pod_index.find(std::string(ns ? ns : "") + "/" + (name ? name : ""));
  return it == p->pod_index.end() ? -1 : it->second;
}
int64_t kth_queue_row(kth_plugin* p, const char* ns, const char* name) {
  if (!p) return -1;
  std::lock_guard<std::mutex> lk(p->mu);
  auto it = p->pod_index.find(std::string(ns ? ns : "") + "/" + (name ? name : ""));
  return it == p->pod_index.end() ? -1 : p->pods[(size_t)it->second].pend_row;
}
int64_t kth_pre_filter_queue(kth_plugin* p, uint8_t* verdicts, int64_t cap) {
  if (!p || cap < 0 || (cap > 0 && !verdicts)) return -1;
  std::lock_guard<std::mutex> lk(p->mu);
  try {
    return p->pre_filter_queue(verdicts, cap);
  } catch (const std::exception& e) {
    ret(err_json(e.what()));  // kth_last_error
    return -1;
  }
}
const char* kth_last_error(void) { return g_ret.c_str(); }
const char* kth_queue_stats(kth_plugin* p) {
  return guarded(p, [&]() -> std::string {
    Writer w;
    w.begin_obj().key("queued").num((long long)(p->pend_pod.size() - p->pend_free.size())).key("rows").num((long long)p->pend_pod.size());
    w.key("passes").num((long long)p->queue.passes).key("hits").num((long long)p->queue.hits);
    // device columns the throttles occupy (deleted throttles' columns are handed out again) and how many of them are live
    w.key("throttleColumns").num((long long)p->throttles.size()).key("liveThrottles").num((long long)p->thr_index.size());
    // the label dictionaries: what the selectors mention (+ one "other value" entry per key), however many labels the pods carry
    w.key("labelKeys").num((long long)p->labels.keys.size()).key("labelValues").num((long long)p->labels.n_values());
    w.key("resourceColumns").num((long long)p->cols.size());
    if (p->words_stat < 0 || p->throttles_dirty || p->namespaces_dirty) {  // (cached per table version: M x namespaces selector evaluations)
      long long total = 0, n_ns = 0;
      for (size_t i = 0; i < p->namespaces.size(); ++i) {
        if (!p->namespaces[i].exists) continue;
        std::set<size_t> words;
        for (size_t t = 0; t < p->throttles.size(); ++t) {
          const ThrottleObj& o = p->throttles[t];
          if (!o.live) continue;
          bool applies = false;
          if (o.kind == KT_KIND_THROTTLE) applies = o.ns == p->namespaces[i].name;
          else
            for (auto& term : o.terms)
              if (term.ns_sel.error.empty() && kth_plugin::ns_selector_matches(term.ns_sel, p->namespaces[i])) { applies = true; break; }
          if (applies) words.insert(t >> 5);
        }
        total += (long long)words.size();
        ++n_ns;
      }
      p->words_stat = n_ns ? total * 100 / n_ns : 0;
    }
    // 32-throttle words a namespace's pods visit (x100, mean over the existing namespaces): what the column order is about
    w.key("wordsPerNamespaceX100").num(p->words_stat);
    if (p->throttles_dirty || p->namespaces_dirty) p->words_stat = -1;  // not laid out yet: do not keep it
    w.end_obj();
    return w.out;
  });
}
const char* kth_pre_filter_batch(kth_plugin* p, const char* pods_json) {
  return guarded(p, [&]() {
    ktjson::NodePtr v = ktjson::parse(pods_json);
    if (!v->is(Node::Arr)) fail("expected a JSON array of pods");
    std::vector<PodObj> batch;
    p->check_only_names = true;
    try { for (auto& e : v->arr) batch.push_back(p->pod_from(*e)); } catch (...) { p->check_only_names = false; throw; }
    p->check_only_names = false;
    kth_plugin::PendingResult r = p->check_pending(batch, 0);
    Writer w;
    w.begin_arr();
    for (size_t i = 0; i < batch.size(); ++i) p->prefilter_json(w, batch[i], r, i);
    w.end_arr();
    return w.out;
  });
}
const char* kth_admit_queue(kth_plugin* p, const char* pods_json) {
  return guarded(p, [&]() { return p->admit_queue(*ktjson::parse(pods_json)); });
}
const char* kth_reserve(kth_plugin* p, const char* pod_json) {
  return guarded(p, [&]() { return p->reserve_json(*ktjson::parse(pod_json), true); });
}
const char* kth_unreserve(kth_plugin* p, const char* pod_json) {
  return guarded(p, [&]() { return p->reserve_json(*ktjson::parse(pod_json), false); });
}
const char* kth_reserved(kth_plugin* p, int kind, const char* throttle_nn) {
  return guarded(p, [&]() { return p->reserved_json(kind, throttle_nn ? throttle_nn : ""); });
}
const char* kth_metrics(kth_plugin* p) {
  return guarded(p, [&]() -> std::string {
    p->flush_metrics();
    return p->metrics_text();
  });
}
const char* kth_eval(const char* request_json) {
  try {
    return ret(eval_request(*ktjson::parse(request_json)));
  } catch (const std::exception& e) {
    return ret(err_json(e.what()));
  }
}

}  // extern "C"
