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

// The host layer is also linked, for CPU tests, against engine test doubles (tests/host_stub) that implement only the calls
// the rest of this file makes: weak references let such a build load, and kth_affected_pods / kth_reconcile / kth_pre_filter_keys
// / kth_apply_events / kth_queue_report fail in it.  The product library defines these calls in kt_engine.cu, so the references
// are always bound there.
#pragma weak kt_get_match_columns
#pragma weak kt_reconcile_throttles
#pragma weak kt_check_pending_rows
#pragma weak kt_match_pods
#pragma weak kt_check_pods            // without it (older engine doubles) check_pending runs a pass over queue + scratch rows
#pragma weak kt_get_check_summary
#pragma weak kt_update_status_rows    // without them (older engine doubles) sync_status / sync_reserved upload whole tables
#pragma weak kt_update_reserved_rows
#pragma weak kt_update_namespace_rows  // without it (older engine doubles) every Namespace event uploads all namespace rows
#pragma weak kt_update_threshold_rows  // without it (older engine doubles) every threshold or override edit recompiles the tables
#pragma weak kt_update_selector_rows   // without it (older engine doubles) every deletion and selector edit recompiles the tables
#pragma weak kt_append_throttle_rows   // without it (older engine doubles) every creation recompiles the tables, hole fills included
#pragma weak kt_move_throttle_columns  // without it (older engine doubles) placement rule 4 and hole compaction recompile the tables

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
// The key of a throttle in kth_plugin::thr_index: "T:namespace/name" for a Throttle, "C:/name" for a ClusterThrottle.
std::string thr_key(int kind, const std::string& ns, const std::string& name) {
  return (kind == KT_KIND_THROTTLE ? "T:" + ns : std::string("C:")) + "/" + name;
}

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
  std::unordered_map<std::string, int> thr_index;  // thr_key -> column, live throttles only
  // the column of the throttle a (namespace, name) argument names -- a ClusterThrottle when the namespace is empty --, -1 if none
  int find_throttle(const std::string& ns, const std::string& tname) const {
    auto it = thr_index.find(thr_key(ns.empty() ? KT_KIND_CLUSTERTHROTTLE : KT_KIND_THROTTLE, ns, tname));
    return it == thr_index.end() ? -1 : it->second;
  }
  // Device columns of deleted throttles are handed out again (a scheduler that lives for months sees throttles come and go: M,
  // the table compile and every pass would only ever grow otherwise).  Whatever lists throttles for the caller -- affected
  // throttles of a pod (the order of the names inside a PreFilter reason), the broken-selector walk (WHICH error a pod gets),
  // reconcile's changed list -- is in creation order, as the reference's lister-backed slices are, not in column order.
  std::vector<int> free_thr;
  long long words_stat = -1;  // kth_queue_stats: words per namespace of the current layout (-1: not computed)
  uint64_t thr_seq = 0;
  bool thr_reused = false;  // some column holds a younger throttle than a higher one: column order is not creation order any more
  size_t m_dev = 0;  // throttle columns the engine holds: [m_dev, throttles.size()) are creations appended by the next sync
  template <class V>
  void creation_order(V& cols_list) const {  // sort a list of throttle columns by creation
    if (thr_reused) std::stable_sort(cols_list.begin(), cols_list.end(), [&](size_t a, size_t b) { return throttles[a].seq < throttles[b].seq; });
  }
  // status_dirty / reserved_dirty: the next sync uploads every column (the engine holds none, or the columns' layout or scale
  // changed).  Otherwise the columns listed in status_cols / reserved_cols go alone (kt_update_status_rows / _reserved_rows).
  // spec_cols: the columns whose threshold or overrides changed and nothing else of the spec (kt_update_threshold_rows, unless
  // the throttles are uploaded whole anyway).  sel_cols: the columns deleted, or whose terms or throttlerName changed, in place
  // (kt_update_selector_rows, likewise).
  bool throttles_dirty = true, namespaces_dirty = true, status_dirty = true, reserved_dirty = true;
  // namespaces_dirty: the next sync sends namespace rows -- all of them with namespaces_full (the engine holds none, the label
  // encoding changed, or the tables are compiled again anyway), else only the rows in ns_dirty (kt_update_namespace_rows).
  bool namespaces_full = true;
  std::set<int32_t> ns_dirty;
  struct ColumnSet {  // throttle columns, each listed once
    std::vector<size_t> list;
    std::vector<char> in;
    void add(size_t t) {
      if (in.size() <= t) in.resize(t + 1, 0);
      if (!in[t]) { in[t] = 1; list.push_back(t); }
    }
    void clear() {
      for (size_t t : list) in[t] = 0;
      list.clear();
    }
  } status_cols, reserved_cols, spec_cols, sel_cols;
  uint64_t col_epoch = 0;  // bumped whenever a resource column is added or changes its scale: every packed column may change
  std::vector<size_t> broken;  // columns of the throttles with a podSelector that does not convert (controller_error)
  bool broken_valid = false;
  const std::vector<size_t>& broken_throttles() {  // usually none, so not a walk over all throttles per pod: built on first need
    if (!broken_valid) {
      broken.clear();
      for (size_t t = 0; t < throttles.size(); ++t)
        if (throttles[t].live && !throttles[t].selector_error().empty()) broken.push_back(t);
      creation_order(broken);
      broken_valid = true;
    }
    return broken;
  }

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
    // The cache is indexed by the columns of the pass that filled it (m of them).  A column move renumbers the columns without
    // voiding it: pass_col[t] is the pass column of current column t (-1: a column the pass did not have), composed across
    // moves; empty means current = pass column.  Rows are translated when read, dirty marks when set.
    size_t m = 0;
    std::vector<int32_t> pass_col;
  } queue;
  void queue_void() { queue.valid = false; }
  static int match_words(size_t m) {  // words per match row of m throttle columns (kt_match_words after they are synced)
    const int w = (int)((m + 31) / 32);
    return std::max(4, (w + 3) / 4 * 4);
  }
  long pass_column(size_t t) const {
    if (!queue.pass_col.empty()) return t < queue.pass_col.size() ? queue.pass_col[t] : -1;
    return t < queue.m ? (long)t : -1;
  }
  void throttle_state_changed(size_t t) {  // status or reservations of throttle column t
    const long p = queue.valid ? pass_column(t) : -1;
    if (p >= 0 && ((size_t)p >> 5) < queue.dirty.size()) queue.dirty[(size_t)p >> 5] |= 1u << (p & 31);
  }
  // Queue row `row`'s cached match row and check codes in the current columns, Wp words (and 2 x Wp code words) wide.
  void cached_row(int64_t row, int Wp, uint32_t* bm, uint32_t* codes) const {
    const uint32_t* src = &queue.bitmap[(size_t)row * (size_t)queue.Wp];
    std::vector<uint32_t> pc(2 * (size_t)queue.Wp, 0);
    auto it = queue.codes.find(row);
    if (it != queue.codes.end())
      for (auto& e : it->second) pc[e.first] = e.second;
    if (queue.pass_col.empty() && Wp == queue.Wp) {
      std::copy_n(src, Wp, bm);
      if (codes) std::copy(pc.begin(), pc.end(), codes);
      return;
    }
    std::fill_n(bm, Wp, 0u);
    if (codes) std::fill_n(codes, 2 * (size_t)Wp, 0u);
    for (size_t t = 0; t < throttles.size() && t < 32 * (size_t)Wp; ++t) {
      const long p = pass_column(t);
      if (p < 0) continue;
      if ((src[(size_t)p >> 5] >> (p & 31)) & 1u) bm[t >> 5] |= 1u << (t & 31);
      if (codes) codes[t >> 4] |= ((pc[(size_t)p >> 4] >> (2 * (p & 15))) & 3u) << (2 * (t & 15));
    }
  }
  void reservation_changed(size_t t) { reserved_cols.add(t); throttle_state_changed(t); }
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
    ++col_epoch;
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
      ++col_epoch;
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

  // A namespace first met through a Namespace event is one more row (the caller marks it: namespace_changed); one first met
  // through a pod or a throttle compiles the tables again, as everything else about the throttle set does.
  int32_t ns_id(const std::string& ns_name, bool namespace_event = false) {
    const uint32_t id = ns_dict.id(ns_name);
    if (namespaces.size() <= id) {
      namespaces.resize(id + 1);
      namespaces[id].name = ns_name;
      if (!namespace_event) namespaces_dirty = namespaces_full = throttles_dirty = true;  // Throttle namespace equality is part of the compiled tables
    }
    return (int32_t)id;
  }

  // Namespace `id` was created, relabelled or deleted: its row goes to the device with the next sync, and the cached verdicts
  // of the queued pods in it are void -- no other pod's verdict reads that row.
  void namespace_changed(int32_t id) {
    namespaces_dirty = true;
    ns_dirty.insert(id);
    if (!queue.valid) return;
    const std::string& nm = namespaces[(size_t)id].name;
    for (size_t row = 0; row < pend_pod.size() && row < queue.row_ok.size(); ++row)
      if (pend_pod[row] >= 0 && pods[(size_t)pend_pod[row]].ns == nm) queue.row_ok[row] = 0;
  }

  // ---- engine --------------------------------------------------------------------------------------
  void drop_engine() {
    if (ctx) kt_destroy(ctx);
    ctx = nullptr;
    sparse_cap = 0;
    queue.valid = false;
    pods_full_upload = pend_full_upload = throttles_dirty = namespaces_dirty = namespaces_full = status_dirty = reserved_dirty = true;
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

  // Namespace i's row into column `col` of lab [LN][stride].
  void pack_namespace(size_t i, int64_t* lab, size_t stride, size_t col) {
    int s = 0;
    for (auto& kv : namespaces[i].labels) {
      const int64_t code = labels.encode(kv.first, kv.second);
      if (code != KT_LABEL_EMPTY) lab[(size_t)(s++) * stride + col] = code;
    }
    // A namespace the lister does not hold (never seen, or deleted) is not in the list affectedPods walks
    // (clusterthrottle_controller.go:227) -- no ClusterThrottle term may match it, not even one whose namespaceSelector is
    // empty.  Existing namespaces carry one internal label (a key no real label can have) that every term requires.
    if (namespaces[i].exists && labels.encode(kNsExistsKey, "1") != KT_LABEL_EMPTY) lab[(size_t)(s++) * stride + col] = labels.encode(kNsExistsKey, "1");
  }
  // A Namespace event changes one row, and only the namespace masks of the tables depend on it: the dirty rows go alone, and
  // only their queued pods lost their cached verdicts (namespace_changed).  Everything is sent again -- and every cached verdict
  // voided -- for the first upload, a new engine, a change of the label encoding, or when the throttles are uploaded anyway.
  void sync_namespaces() {
    ensure_engine();
    if (!namespaces_dirty) return;
    words_stat = -1;
    const int LN = lim.ns_label_slots;
    const size_t n = namespaces.size();
    if (namespaces_full || throttles_dirty || !kt_update_namespace_rows) {
      queue_void();  // (see sync_throttles)
      std::vector<int64_t> lab((size_t)LN * std::max<size_t>(n, 1), KT_LABEL_EMPTY);
      for (size_t i = 0; i < n; ++i) pack_namespace(i, lab.data(), n, i);
      check(kt_upload_namespaces(ctx, (int32_t)n, lab.data()), "kt_upload_namespaces");
    } else {
      const std::vector<int32_t> idx(ns_dirty.begin(), ns_dirty.end());
      const size_t k = idx.size();
      std::vector<int64_t> lab((size_t)LN * std::max<size_t>(k, 1), KT_LABEL_EMPTY);
      for (size_t i = 0; i < k; ++i) pack_namespace((size_t)idx[i], lab.data(), k, i);
      check(kt_update_namespace_rows(ctx, (int32_t)n, (int64_t)k, idx.data(), lab.data()), "kt_update_namespace_rows");
    }
    namespaces_dirty = namespaces_full = false;
    ns_dirty.clear();
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
  // The column order of the full path: live throttles only (the holes compacted), ClusterThrottles after Throttles, each
  // group -- a Throttle's namespace, a ClusterThrottle's namespace set -- together, by creation within it.  Both the whole
  // upload (reorder_columns) and a column move (move_columns) lay the columns out by it.
  std::vector<size_t> column_order() const {
    struct Key {
      int kind;
      std::string set;
      uint64_t seq;
      size_t idx;
    };
    std::vector<Key> keys;
    std::map<std::string, std::string> set_of;  // distinct ClusterThrottle signatures: evaluated once
    for (size_t t = 0; t < throttles.size(); ++t) {
      const ThrottleObj& o = throttles[t];
      if (!o.live) continue;
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
    std::vector<size_t> order;
    order.reserve(keys.size());
    for (auto& k : keys) order.push_back(k.idx);
    return order;
  }
  void reorder_columns() {
    const std::vector<size_t> order = column_order();
    bool same = order.size() == throttles.size();
    for (size_t i = 0; same && i < order.size(); ++i) same = order[i] == i;
    if (same) return;
    lay_out(order);
    queue_void();
    status_dirty = reserved_dirty = true;
  }
  // The throttles in the given column order (the ones not listed are dropped), with the index rebuilt.
  void lay_out(const std::vector<size_t>& order) {
    std::vector<ThrottleObj> laid_out;
    laid_out.reserve(order.size());
    for (size_t t : order) laid_out.push_back(std::move(throttles[t]));
    throttles = std::move(laid_out);
    thr_index.clear();
    free_thr.clear();
    thr_reused = false;
    for (size_t t = 0; t < throttles.size(); ++t) {
      thr_index[thr_key(throttles[t].kind, throttles[t].ns, throttles[t].name)] = (int)t;
      if (t && throttles[t].seq < throttles[t - 1].seq) thr_reused = true;  // column order is not creation order
    }
    broken_valid = false;
  }
  // A new layout without a whole upload (relayout_pending: placement rule 4, hole compaction): at the next sync, like the whole
  // upload it replaces, the columns are laid out as the full path would (column_order), and the device follows through one
  // kt_move_throttle_columns (sync_move), before every other column delta.  src[j] is the device column current column j comes
  // from, -1 for a live throttle the device does not hold yet (a creation, an append not sent): those become empty columns there
  // and are filled through the selector, threshold, status and reserved deltas.  The pending column deltas are re-indexed; the
  // cached verdicts are kept, their columns mapped (QueueCache::pass_col).
  bool relayout_pending = false;
  bool status_held = false;  // the engine holds an observed status (kt_upload_status since the last kt_upload_throttles)
  std::vector<int32_t> move_columns() {
    const std::vector<size_t> order = column_order();
    const size_t m0 = throttles.size();
    std::vector<long> new_of(m0, -1);
    std::vector<int32_t> src(order.size()), pass(order.size());
    for (size_t j = 0; j < order.size(); ++j) {
      const size_t t = order[j];
      new_of[t] = (long)j;
      src[j] = t >= m_dev ? -1 : (int32_t)t;
      pass[j] = (int32_t)pass_column(t);
    }
    lay_out(order);
    for (ColumnSet* cs : {&status_cols, &reserved_cols, &spec_cols, &sel_cols}) {
      const std::vector<size_t> old = cs->list;
      cs->clear();
      for (size_t t : old)
        if (t < m0 && new_of[t] >= 0) cs->add((size_t)new_of[t]);
    }
    for (size_t j = 0; j < src.size(); ++j)
      if (src[j] < 0) {  // filled through the column deltas
        sel_cols.add(j);
        spec_cols.add(j);
        status_cols.add(j);
        reserved_cols.add(j);
      }
    if (queue.valid) queue.pass_col.swap(pass);
    words_stat = -1;
    return src;
  }
  void sync_move() {
    if (!relayout_pending) return;
    relayout_pending = false;
    const std::vector<int32_t> src = move_columns();
    check(kt_move_throttle_columns(ctx, (int32_t)src.size(), src.data()), "kt_move_throttle_columns");
    m_dev = throttles.size();
    if (!status_held) status_dirty = true;  // a status column delta replaces columns of a status the engine holds
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
    const size_t m = throttles.size();
    SelectorColumns scols = selector_columns(AllColumns{m});
    const ThresholdColumns tcols = threshold_columns(AllColumns{m});
    kt_throttle_cols tc = tcols.cols();
    scols.put(&tc);
    const kt_selector_table st = scols.table();
    sync_namespaces();  // Throttle rows may have introduced namespace ids
    check(kt_upload_throttles(ctx, (int32_t)m, &tc, &st), "kt_upload_throttles");
    m_dev = m;
    relayout_pending = false;  // (the whole upload lays the columns out)
    status_held = false;
    throttles_dirty = false;
    status_dirty = reserved_dirty = true;  // kt_upload_throttles forgets both
    spec_cols.clear();
    sel_cols.clear();
  }
  // What compile_tables reads of the listed throttles: kind, ns_id, flags ([k]) and the selector CSR over them, in list order
  // (requirement pool: all podSelector requirements in term order, then all namespaceSelector ones).  A deleted throttle's column
  // has no terms and flags 0.
  struct SelectorColumns {
    std::vector<uint8_t> kind, flags;
    std::vector<int32_t> nsid;
    std::vector<int32_t> term_off{0}, pod_req_off{0}, ns_req_off, req_val_off{0};
    std::vector<uint8_t> term_flags, req_op;
    std::vector<uint32_t> req_key, req_vals;
    void put(kt_throttle_cols* tc) const { tc->kind = kind.data(); tc->ns_id = nsid.data(); tc->flags = flags.data(); }
    kt_selector_table table() const {
      kt_selector_table st{};
      st.n_terms = (int32_t)term_flags.size(); st.n_reqs = (int32_t)req_key.size(); st.n_vals = (int32_t)req_vals.size();
      st.term_off = term_off.data(); st.term_flags = term_flags.data(); st.pod_req_off = pod_req_off.data(); st.ns_req_off = ns_req_off.data();
      st.req_key = req_key.data(); st.req_op = req_op.data(); st.req_val_off = req_val_off.data(); st.req_vals = req_vals.data();
      return st;
    }
  };
  template <class List>
  SelectorColumns selector_columns(const List& list) {
    const size_t k = list.size();
    SelectorColumns sc;
    sc.kind.resize(k); sc.flags.resize(k); sc.nsid.resize(k);
    std::vector<std::vector<Requirement>> ns_reqs_of_term;
    auto push_reqs = [&](const std::vector<Requirement>& reqs) {
      for (auto& r : reqs) {
        const uint32_t kid = labels.key_id(r.key);  // (all of it interned by sync_vocabulary already)
        sc.req_key.push_back(kid);
        sc.req_op.push_back(r.op);
        for (auto& v : r.values) sc.req_vals.push_back(labels.value_id(kid, v));
        sc.req_val_off.push_back((int32_t)sc.req_vals.size());
      }
    };
    for (size_t i = 0; i < k; ++i) {
      const ThrottleObj& o = throttles[list[i]];
      sc.kind[i] = (uint8_t)o.kind;
      sc.nsid[i] = o.kind == KT_KIND_THROTTLE ? ns_id(o.ns) : -1;
      sc.flags[i] = 0;
      if (o.live && o.throttler_name == name) sc.flags[i] |= KT_THR_RESPONSIBLE;  // isResponsibleFor, throttle_controller.go:213-215
      for (auto& term : o.terms) {
        // a podSelector that does not convert: the term matches nobody and shadows the LATER terms for exactly the pods that
        // reach it (KT_TERM_POD_INVALID; the table compiler scopes that by namespace / namespaceSelector)
        sc.term_flags.push_back((term.ns_sel.error.empty() ? 0 : KT_TERM_NS_INVALID) |  // Q9: swallowed, the term is false
                                (term.pod_sel.error.empty() ? 0 : KT_TERM_POD_INVALID));
        push_reqs(term.pod_sel.reqs);  // (none when the selector is broken)
        sc.pod_req_off.push_back((int32_t)sc.req_key.size());
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
      sc.term_off.push_back((int32_t)sc.term_flags.size());
    }
    sc.ns_req_off.push_back((int32_t)sc.req_key.size());
    for (auto& reqs : ns_reqs_of_term) {
      push_reqs(reqs);
      sc.ns_req_off.push_back((int32_t)sc.req_key.size());
    }
    return sc;
  }
  // Creations placed at the end (apply_throttle, place_creation): the columns [m_dev, m) in one kt_append_throttle_rows, before
  // any column delta that may list them.  Their status and reservations, when not zero, follow as column deltas (status_cols /
  // reserved_cols, set by apply_throttle).
  void sync_appends() {
    const size_t m = throttles.size();
    if (m_dev >= m) return;
    std::vector<size_t> list;
    for (size_t t = m_dev; t < m; ++t) list.push_back(t);
    const SelectorColumns scols = selector_columns(list);
    const ThresholdColumns tcols = threshold_columns(list);
    kt_throttle_cols tc = tcols.cols();
    scols.put(&tc);
    const kt_selector_table st = scols.table();
    check(kt_append_throttle_rows(ctx, (int64_t)list.size(), &tc, &st, nullptr), "kt_append_throttle_rows");
    m_dev = m;
  }
  // Deletions and in-place selector / throttlerName edits (delete_throttle, apply_throttle): one kt_update_selector_rows for the
  // listed columns, with the column layout kept.  The engine patches its tables when the new terms fit them and compiles them
  // again otherwise; either way the statuses and reservations it holds stay.
  void sync_selectors() {
    if (sel_cols.list.empty()) return;
    const SelectorColumns scols = selector_columns(sel_cols.list);
    kt_throttle_cols tc{};
    scols.put(&tc);
    const kt_selector_table st = scols.table();
    const std::vector<int32_t> idx(sel_cols.list.begin(), sel_cols.list.end());
    check(kt_update_selector_rows(ctx, (int64_t)idx.size(), idx.data(), &tc, &st, nullptr), "kt_update_selector_rows");
    sel_cols.clear();
  }
  // The spec columns of the listed throttles that no compiled table reads: spec.threshold ([R][k] / [k]) and the
  // temporaryThresholdOverrides in spec order (ovr_off[k+1], ovr_thr[R][n_ovr]).  kind, ns_id and flags stay null.
  struct ThresholdColumns {
    std::vector<int32_t> ovr_off;
    std::vector<int64_t> thr, thr_cnt, ovr_begin, ovr_end, ovr_thr, ovr_cnt;
    std::vector<uint32_t> thr_present, ovr_present;
    std::vector<uint8_t> ovr_flags;
    kt_throttle_cols cols() const {
      kt_throttle_cols tc{};
      tc.thr = thr.data(); tc.thr_present = thr_present.data(); tc.thr_cnt = thr_cnt.data(); tc.ovr_off = ovr_off.data();
      tc.n_ovr = ovr_off.back(); tc.ovr_begin = ovr_begin.data(); tc.ovr_end = ovr_end.data(); tc.ovr_flags = ovr_flags.data();
      tc.ovr_thr = ovr_thr.data(); tc.ovr_present = ovr_present.data(); tc.ovr_cnt = ovr_cnt.data();
      return tc;
    }
  };
  template <class List>
  ThresholdColumns threshold_columns(const List& list) const {
    const int R = lim.n_resources;
    const size_t k = list.size();
    ThresholdColumns tc;
    tc.ovr_off.assign(k + 1, 0);
    tc.thr.assign((size_t)R * std::max<size_t>(k, 1), 0); tc.thr_cnt.assign(k, 0); tc.thr_present.assign(k, 0);
    std::vector<std::vector<int64_t>> ovr_vals;  // per override: R values
    auto amount_cols = [&](const ResAmount& a, int64_t* vals, size_t stride, uint32_t* present, int64_t* cnt) {
      *present = 0;
      *cnt = 0;
      if (a.has_counts) { *present |= KT_COUNT_BIT; *cnt = a.pod; }
      for (auto& kv : a.requests) {
        vals[(size_t)kv.first * stride] = at_scale(kv.first, kv.second);
        *present |= 1u << kv.first;
      }
    };
    for (size_t i = 0; i < k; ++i) {
      const ThrottleObj& o = throttles[list[i]];
      amount_cols(o.threshold, &tc.thr[i], k, &tc.thr_present[i], &tc.thr_cnt[i]);
      for (const Override& ov : o.overrides) {
        GoTime b, e;
        uint8_t f = 0;
        if (!ov.begin.empty() && !parse_rfc3339(ov.begin, &b).empty()) f = KT_OVR_PARSE_ERROR;
        if (!ov.end.empty() && !parse_rfc3339(ov.end, &e).empty()) f = KT_OVR_PARSE_ERROR;
        tc.ovr_begin.push_back(b.zero ? KT_TIME_OPEN_BEGIN : clamp_ns(b.ns()));
        tc.ovr_end.push_back(e.zero ? KT_TIME_OPEN_END : clamp_ns(e.ns()));
        tc.ovr_flags.push_back(f);
        std::vector<int64_t> vals((size_t)R, 0);
        uint32_t pr;
        int64_t cnt;
        amount_cols(ov.threshold, vals.data(), 1, &pr, &cnt);
        ovr_vals.push_back(std::move(vals));
        tc.ovr_present.push_back(pr);
        tc.ovr_cnt.push_back(cnt);
      }
      tc.ovr_off[i + 1] = (int32_t)tc.ovr_begin.size();
    }
    const size_t n_ovr = tc.ovr_begin.size();
    tc.ovr_thr.assign((size_t)R * std::max<size_t>(n_ovr, 1), 0);
    for (size_t i = 0; i < n_ovr; ++i)
      for (int r = 0; r < R; ++r) tc.ovr_thr[(size_t)r * n_ovr + i] = ovr_vals[i][(size_t)r];
    return tc;
  }
  // Threshold and override edits that left the tables alone: one kt_update_threshold_rows for the listed columns.  No "more than
  // half dirty" rule here: the alternative is a table recompile, never cheaper.
  void sync_thresholds() {
    if (spec_cols.list.empty()) return;
    const ThresholdColumns tcols = threshold_columns(spec_cols.list);
    const kt_throttle_cols tc = tcols.cols();
    const std::vector<int32_t> idx(spec_cols.list.begin(), spec_cols.list.end());
    check(kt_update_threshold_rows(ctx, (int64_t)idx.size(), idx.data(), &tc), "kt_update_threshold_rows");
    spec_cols.clear();
  }

  // Whether the dirty columns go as a delta (the callers check first that no full upload is pending): the engine has the call and
  // at most half the columns changed.  Past half a delta carries about as many bytes as the whole table; the half itself is a
  // guess, not a measured break-even point.
  bool column_delta(const ColumnSet& dirty, bool have_call) const { return have_call && 2 * dirty.list.size() <= throttles.size(); }
  // The observed status of the listed throttle columns, shaped [R][k] / [k] (k = list.size()).
  struct StatusColumns {
    std::vector<uint8_t> calculated;
    std::vector<int64_t> calc_thr, calc_cnt, used, used_cnt;
    std::vector<uint32_t> calc_present, used_present, throttled;
    kt_status_cols cols() const {
      return kt_status_cols{calculated.data(), calc_thr.data(), calc_present.data(), calc_cnt.data(), used.data(), used_present.data(), used_cnt.data(), throttled.data()};
    }
  };
  template <class List>
  StatusColumns status_columns(const List& list) const {
    const int R = lim.n_resources;
    const size_t k = list.size();
    StatusColumns sc;
    sc.calculated.assign(k, 0);
    sc.calc_thr.assign((size_t)R * k, 0); sc.calc_cnt.assign(k, 0); sc.used.assign((size_t)R * k, 0); sc.used_cnt.assign(k, 0);
    sc.calc_present.assign(k, 0); sc.used_present.assign(k, 0); sc.throttled.assign(k, 0);
    for (size_t i = 0; i < k; ++i) {
      const ThrottleObj& o = throttles[list[i]];
      sc.calculated[i] = o.st_calc_at_set;  // !CalculatedAt.Time.IsZero() (throttle_types.go:129-132)
      if (o.st_calc.has_counts) { sc.calc_present[i] |= KT_COUNT_BIT; sc.calc_cnt[i] = o.st_calc.pod; }
      for (auto& kv : o.st_calc.requests) { sc.calc_thr[(size_t)kv.first * k + i] = at_scale(kv.first, kv.second); sc.calc_present[i] |= 1u << kv.first; }
      if (o.st_used.has_counts) { sc.used_present[i] |= KT_COUNT_BIT; sc.used_cnt[i] = o.st_used.pod; }
      for (auto& kv : o.st_used.requests) { sc.used[(size_t)kv.first * k + i] = at_scale(kv.first, kv.second); sc.used_present[i] |= 1u << kv.first; }
      if (o.st_thr_pod) sc.throttled[i] |= KT_COUNT_BIT;
      for (auto& kv : o.st_thr_req)
        if (kv.second) sc.throttled[i] |= 1u << kv.first;
    }
    return sc;
  }
  struct AllColumns {  // 0 .. m-1 as a list
    size_t m;
    size_t size() const { return m; }
    size_t operator[](size_t i) const { return i; }
  };
  void sync_status() {
    const size_t m = throttles.size();
    if (m > 0 && (status_dirty || (!status_cols.list.empty() && !column_delta(status_cols, kt_update_status_rows != nullptr)))) {
      const StatusColumns sc = status_columns(AllColumns{m});
      const kt_status_cols c = sc.cols();
      check(kt_upload_status(ctx, &c), "kt_upload_status");
      status_held = true;
    } else if (m > 0 && !status_cols.list.empty()) {
      const StatusColumns sc = status_columns(status_cols.list);
      const kt_status_cols c = sc.cols();
      const std::vector<int32_t> idx(status_cols.list.begin(), status_cols.list.end());
      check(kt_update_status_rows(ctx, (int64_t)idx.size(), idx.data(), &c), "kt_update_status_rows");
    }
    status_dirty = false;
    status_cols.clear();
  }

  // reservedResourceAmounts.reservedResourceAmount(nn) of the listed throttle columns, re-summed from the reservation cache,
  // shaped [R][k] / [k]; returns whether any of them holds a reservation.
  template <class List>
  bool reserved_columns(const List& list, std::vector<int64_t>& reserved, std::vector<uint32_t>& present, std::vector<int64_t>& cnt) const {
    const int R = lim.n_resources;
    const size_t k = list.size();
    reserved.assign((size_t)R * k, 0);
    present.assign(k, 0);
    cnt.assign(k, 0);
    bool any = false;
    for (size_t i = 0; i < k; ++i) {
      const ThrottleObj& o = throttles[list[i]];
      auto it = cache[o.kind].by_thr.find(o.nn());
      if (it == cache[o.kind].by_thr.end() || it->second.empty()) continue;
      any = true;
      present[i] |= KT_COUNT_BIT;  // every reserved ResourceAmountOfPod carries Counts{Pod: 1}
      cnt[i] = (int64_t)it->second.size();
      for (auto& pod : it->second)
        for (auto& kv : pod.second) {
          reserved[(size_t)kv.first * k + i] += at_scale(kv.first, kv.second);
          present[i] |= 1u << kv.first;
        }
    }
    return any;
  }
  void sync_reserved() {
    const size_t m = throttles.size();
    std::vector<int64_t> reserved, cnt;
    std::vector<uint32_t> present;
    if (m > 0 && (reserved_dirty || (!reserved_cols.list.empty() && !column_delta(reserved_cols, kt_update_reserved_rows != nullptr)))) {
      if (reserved_columns(AllColumns{m}, reserved, present, cnt)) check(kt_set_reserved(ctx, reserved.data(), present.data(), cnt.data()), "kt_set_reserved");
      else check(kt_set_reserved(ctx, nullptr, nullptr, nullptr), "kt_set_reserved");
    } else if (m > 0 && !reserved_cols.list.empty()) {  // only the columns whose reservations changed are summed again
      reserved_columns(reserved_cols.list, reserved, present, cnt);
      const std::vector<int32_t> idx(reserved_cols.list.begin(), reserved_cols.list.end());
      check(kt_update_reserved_rows(ctx, (int64_t)idx.size(), idx.data(), reserved.data(), present.data(), cnt.data()), "kt_update_reserved_rows");
    }
    reserved_dirty = false;
    reserved_cols.clear();
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
    namespaces_dirty = namespaces_full = true;  // (a handful of rows: packed whole)
  }
  void sync_all() {
    sync_vocabulary();
    sync_pods();
    sync_namespaces();
    sync_throttles();
    sync_move();        // (after sync_throttles, which carries the new layout when it uploads the throttles; before every delta)
    sync_appends();     // (after sync_throttles, which sends these columns too when it uploads the throttles)
    sync_selectors();   // (after both: a hole fill or an edit may list an appended column)
    sync_thresholds();
  }
  // Everything a PreFilter view reads: the tables, the informer copy of the statuses and the reservations.  A table change voids
  // the cached queue verdicts on the way (sync_namespaces / sync_throttles); afterwards no dirty flag is set.
  void sync_state() {
    sync_all();
    sync_status();
    sync_reserved();
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

  // The kt_reconcile_out columns of k throttles, as kt_get_reconcile_rows and kt_reconcile_throttles fill them.
  struct ReconcileCols {
    size_t k;
    std::vector<int64_t> used, used_cnt, calc_thr, calc_cnt;
    std::vector<uint32_t> used_present, throttled, calc_present;
    std::vector<uint8_t> ovr_active;
    kt_reconcile_out out;
    ReconcileCols(size_t k, int R)
        : k(k), used((size_t)R * std::max<size_t>(k, 1)), used_cnt(k), calc_thr((size_t)R * std::max<size_t>(k, 1)), calc_cnt(k),
          used_present(k), throttled(k), calc_present(k), ovr_active(k),
          out{used.data(), used_present.data(), used_cnt.data(), throttled.data(), calc_thr.data(), calc_present.data(), calc_cnt.data(), ovr_active.data()} {}
    ReconcileCols(const ReconcileCols&) = delete;  // `out` points into this object's columns
    ReconcileCols& operator=(const ReconcileCols&) = delete;
  };
  // What reconcile writes for throttle t from its device status (entry q of st): status.used, calculatedThreshold (Q6),
  // throttled, compared under Semantic.DeepEqual; records the gauges.  Returns whether the status changed.
  bool update_status(size_t t, const ReconcileCols& st, size_t q, const GoTime& now) {
    const kt_reconcile_out& ro = st.out;
    const size_t k = st.k;
    ThrottleObj& o = throttles[t];
    o.host_dirty = false;
    ResAmount nu;  // used := ResourceAmount{}; used = used.Add(ResourceAmountOfPod(p)) ...
    if (ro.used_present[q] & KT_COUNT_BIT) {
      nu.has_counts = true;
      nu.pod = ro.used_cnt[q];
      nu.requests_nil = false;
      for (int r = 0; r < (int)cols.size(); ++r)
        if ((ro.used_present[q] >> r) & 1) nu.requests[r] = from_scale(r, ro.used[(size_t)r * k + q]);
    }
    ResAmount nc;  // CalculateThreshold(now).Threshold
    nc.has_counts = ro.calc_present[q] & KT_COUNT_BIT;
    nc.pod = nc.has_counts ? ro.calc_cnt[q] : 0;
    nc.requests_nil = false;
    for (int r = 0; r < (int)cols.size(); ++r)
      if ((ro.calc_present[q] >> r) & 1) nc.requests[r] = from_scale(r, ro.calc_thr[(size_t)r * k + q]);
    if (!ro.override_active[q]) nc = o.threshold;  // no active override: spec.threshold itself (keeps nil-ness and spelling)
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
    const bool thr_pod = ro.throttled[q] & KT_COUNT_BIT;
    std::map<int, bool> thr_req;
    for (auto& kv : o.st_calc.requests) thr_req[kv.first] = (ro.throttled[q] >> kv.first) & 1;
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
      throttle_state_changed(t);  // PreFilter reads this status: cached verdicts of the pods it affects are void
      status_cols.add(t);
    }
    return status_changed;
  }

  // What a reconcile of several throttles returns: kth_reconcile_all's object; kth_reconcile's adds errors and notFound.
  struct ReconcileReport {
    int reconciled = 0;
    std::vector<std::string> changed;
    std::vector<std::pair<std::string, long long>> requeue;  // enqueueAfter(thr, *nextOverrideHappensIn)
    std::vector<std::pair<std::string, std::string>> errors;
    std::vector<std::string> not_found;
    std::string json(bool keyed) const {
      Writer w;
      w.begin_obj().key("reconciled").num(reconciled).key("changed").begin_arr();
      for (auto& c : changed) w.str(c);
      w.end_arr().key("requeueAfterNanos").begin_obj();
      for (auto& r : requeue) w.key(r.first).num(r.second);
      w.end_obj();
      if (keyed) {
        w.key("errors").begin_obj();
        for (auto& er : errors) w.key(er.first).str(er.second);
        w.end_obj().key("notFound").begin_arr();
        for (auto& nf : not_found) w.str(nf);
        w.end_arr();
      }
      w.end_obj();
      return w.out;
    }
  };

  // reconcile(key) of the responsible throttle t once the device has answered for it.  Both callers give the answer in one form:
  // matched(row) says whether t matches running row `row` -- the RUNNING relation, affectedPods: counted pods, finished ones
  // included --, and [fin0, fin1) holds every finished row t matches (rows t does not match may be among them).  err_rows are
  // selector_error_rows(t); q is t's entry in st, < 0 when the device says its status does not change.  Returns the error that
  // fails the reconcile, "" when it ran.
  template <class Matched>
  std::string reconcile_throttle(size_t t, const Matched& matched, const std::vector<int64_t>& err_rows, const int64_t* fin0, const int64_t* fin1,
                                 const ReconcileCols& st, int64_t q, const GoTime& now, ReconcileReport& rep) {
    ThrottleObj& o = throttles[t];
    // A Throttle with a podSelector term that does not convert: affectedPods (throttle_controller.go:221-246) only fails -- and
    // the reconcile with it: status untouched, nothing un-reserved (:233-236) -- when some counted pod of the namespace actually
    // REACHES that term, i.e. matches none of the valid terms before it (those are what the device column holds,
    // sync_throttles).  The first such pod in informer order names the error.  ClusterThrottles: see DESIGN.md "Known
    // deviations" (their terms carry their own namespace scope).
    const PodObj* first = nullptr;
    for (int64_t r : err_rows)
      if (!matched(r) && (!first || pods[(size_t)r].seq < first->seq)) first = &pods[(size_t)r];
    if (first) return reachable_selector_error(o, first->ns);
    ++rep.reconciled;
    if (q >= 0 && update_status(t, st, (size_t)q, now)) rep.changed.push_back(o.nn());
    __int128 after = 0;
    if (next_override_happens_in(o, now, &after)) rep.requeue.emplace_back(o.nn(), (long long)(after > INT64_MAX ? INT64_MAX : after));
    // unreserveAffectedPods: every affected pod the informer has observed leaves the reservation cache -- except, for a
    // Throttle, the finished ones the reference's list loses.  Q8 (throttle_controller.go:241, `terminatedPods =
    // append(nonterminatedPods, pod)`): the THROTTLE controller's list of terminated affected pods ends up holding only the
    // LAST terminated match of the namespace (a Throttle matches the pods of its own namespace only), so of the finished pods
    // that still hold a reservation only that one is un-reserved; the others keep it until the pod is deleted.  (Which pod is
    // "last" is the informer's map order in the reference; the oracle and this code take the order of first appearance.)
    auto it = cache[o.kind].by_thr.find(o.nn());
    if (it == cache[o.kind].by_thr.end()) return "";
    int64_t last_fin = -2;  // computed on first need
    std::vector<std::string> gone;
    for (auto& pod : it->second) {
      auto pi = pod_index.find(pod.first);
      if (pi == pod_index.end() || !matched(pi->second)) continue;
      if (o.kind == KT_KIND_THROTTLE && !(pod_flags(pods[(size_t)pi->second]) & KT_POD_NOT_FINISHED)) {
        if (last_fin == -2) {
          last_fin = -1;
          for (const int64_t* r = fin0; r < fin1; ++r) {
            const PodObj& p = pods[(size_t)*r];
            if (matched(*r) && !(pod_flags(p) & KT_POD_NOT_FINISHED) && (last_fin < 0 || p.seq > pods[(size_t)last_fin].seq)) last_fin = *r;
          }
        }
        if (pi->second != last_fin) continue;
      }
      gone.push_back(pod.first);
    }
    for (auto& g : gone)
      if (it->second.erase(g)) reservation_changed(t);
    return "";
  }

  std::string reconcile_all(const std::string& now_s) {
    GoTime now;
    std::string e = parse_rfc3339(now_s, &now);
    if (!e.empty()) fail(e);
    sync_all();
    const size_t m = throttles.size();
    ReconcileReport rep;
    if (m == 0) return rep.json(false);
    // The informer copy of every status is on the device (sync_status: a no-op unless some status changed since the last
    // upload), so the pass itself diffs what it computes against it (throttle_controller.go:157 DeepEqual): only the throttles it
    // lists -- plus those applied since their last reconcile, whose host-only status parts may differ -- are looked at and
    // downloaded below (SURVEY 8f.3: the download and the host's work are proportional to what changed, not to M).
    sync_status();
    check(kt_evaluate(ctx, clamp_ns(now.ns()), KT_EVAL_FRESH_STATUS | KT_EVAL_SKIP_CHECK), "kt_evaluate");
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
    ReconcileCols st(k, lim.n_resources);
    if (k) check(kt_get_reconcile_rows(ctx, (int64_t)k, todo_idx.data(), &st.out), "kt_get_reconcile_rows");
    // The match words of the running rows the throttles' steps ask about (a row's words hold every throttle's bit).  First the
    // pods that are reserved somewhere: their match rows decide what reconcile un-reserves (:135-155).
    std::vector<int64_t> rows;
    {
      std::set<std::string> seen;
      for (int k = 0; k < 2; ++k)
        for (auto& thr : cache[k].by_thr)
          for (auto& pod : thr.second) {
            auto it = pod_index.find(pod.first);
            if (it != pod_index.end() && seen.insert(pod.first).second) rows.push_back(it->second);
          }
    }
    const int Wp = kt_match_words(ctx);
    std::vector<std::vector<uint32_t>> words;
    std::unordered_map<int64_t, const uint32_t*> words_of;
    auto fetch = [&](const std::vector<int64_t>& rs) {
      if (rs.empty()) return;
      words.emplace_back(rs.size() * (size_t)Wp);
      check(kt_get_match_rows(ctx, KT_PODS_RUNNING, (int64_t)rs.size(), rs.data(), words.back().data()), "kt_get_match_rows");
      for (size_t i = 0; i < rs.size(); ++i) words_of[rs[i]] = words.back().data() + i * (size_t)Wp;
    };
    fetch(rows);
    // Q8 asks which finished pod is the last match of a Throttle only when a finished pod holds a reservation: then the rows of
    // the finished counted pods
    bool any_finished_reserved = false;
    for (int64_t r : rows) any_finished_reserved |= !(pod_flags(pods[(size_t)r]) & KT_POD_NOT_FINISHED);
    std::vector<int64_t> fin_rows;
    if (any_finished_reserved) {
      for (auto& p : pods)
        if (p.live && should_count_in(p) && !(pod_flags(p) & KT_POD_NOT_FINISHED)) fin_rows.push_back(p.row);
      fetch(fin_rows);
    }
    // the counted pods a broken podSelector term may be in the way of
    std::vector<std::vector<int64_t>> err_rows(m);
    for (size_t t = 0; t < m; ++t)
      if (throttles[t].live && throttles[t].throttler_name == name) {
        err_rows[t] = selector_error_rows(throttles[t]);
        fetch(err_rows[t]);
      }

    std::vector<size_t> thr_order(m);
    for (size_t t = 0; t < m; ++t) thr_order[t] = t;
    creation_order(thr_order);
    for (size_t t : thr_order) {
      const ThrottleObj& o = throttles[t];
      if (!o.live || o.throttler_name != name) continue;  // only responsible throttles are ever enqueued (:403-425)
      auto matched = [&](int64_t r) { return ((words_of.at(r)[t >> 5] >> (t & 31)) & 1) != 0; };
      // (a selector error leaves t as it is: kth_reconcile_all does not report it)
      reconcile_throttle(t, matched, err_rows[t], fin_rows.data(), fin_rows.data() + fin_rows.size(), st, pos[t], now, rep);
    }
    return rep.json(false);
  }

  // The counted pods a broken podSelector term of o is in the way of: the Throttle's namespace, or -- per term -- the
  // namespaces a ClusterThrottle term's namespaceSelector matches (clusterthrottle_controller.go:224-270 walks exactly those
  // pods).  affectedPods fails when one of them matches none of the valid terms before it (its bit is clear).  Empty when o
  // has no broken term.
  std::vector<int64_t> selector_error_rows(const ThrottleObj& o) const {
    std::vector<int64_t> ns_rows;
    if (o.selector_error().empty()) return ns_rows;
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
    return ns_rows;
  }

  // ---- affectedPods of one throttle (kth_affected_pods) -----------------------------------------------------------
  // Both relations come from one GIVEN_STATUS pass that reconciles too: the running rows it matches are what a reconcile
  // would sum, the pending codes are what PreFilter by key would answer.  Its results stay good until some other entry
  // point runs (every one of them may change the state or run a pass of its own: `epoch`).
  uint64_t epoch = 1, columns_epoch = 0;
  void column_of(int kind, int32_t t, std::vector<int64_t>& rows, std::vector<uint8_t>* codes) {
    if (!kt_get_match_columns) fail("kth_affected_pods: the engine this plugin is linked against has no kt_get_match_columns");
    int64_t off[2] = {0, 0}, cap = 256;
    while (true) {
      rows.resize((size_t)cap);
      if (codes) codes->resize((size_t)cap);
      check(kt_get_match_columns(ctx, kind, 1, &t, off, rows.data(), codes ? codes->data() : nullptr, cap), "kt_get_match_columns");
      if (off[1] <= cap) break;
      cap = off[1];
    }
    rows.resize((size_t)off[1]);
    if (codes) codes->resize((size_t)off[1]);
  }
  std::string affected_pods(const std::string& ns, const std::string& tname) {
    const int found_at = find_throttle(ns, tname);
    if (found_at < 0) fail((ns.empty() ? "clusterthrottle " : "throttle ") + ns + "/" + tname + " not found");
    const ThrottleObj& found = throttles[(size_t)found_at];
    if (found.throttler_name != name) fail(found.nn() + " belongs to throttler \"" + found.throttler_name + "\", not to \"" + name + "\"");
    if (columns_epoch != epoch) {
      run_pending_pass({}, 0, 0);
      columns_epoch = codes_epoch = epoch;
    }
    const size_t t = (size_t)find_throttle(ns, tname);  // (the pass may have laid the columns out anew)
    std::vector<int64_t> run_rows, pend_rows;
    std::vector<uint8_t> codes;
    column_of(KT_PODS_RUNNING, (int32_t)t, run_rows, nullptr);
    column_of(KT_PODS_PENDING, (int32_t)t, pend_rows, &codes);
    const ThrottleObj& o = throttles[t];
    // a counted pod that reaches a broken term: affectedPods returns that error (throttle_controller.go:233-236); the first such
    // pod in informer order names it
    const std::vector<int64_t> err_rows = selector_error_rows(o);
    if (!err_rows.empty()) {
      const PodObj* first = nullptr;
      for (int64_t r : err_rows)
        if (!std::binary_search(run_rows.begin(), run_rows.end(), r) && (!first || pods[(size_t)r].seq < first->seq)) first = &pods[(size_t)r];
      if (first) fail(reachable_selector_error(o, first->ns));
    }
    auto by_key = [](const PodObj* a, const PodObj* b) { return a->ns != b->ns ? a->ns < b->ns : a->name < b->name; };
    std::vector<const PodObj*> running, finished;
    for (int64_t r : run_rows) {
      const PodObj& p = pods[(size_t)r];
      ((pod_flags(p) & KT_POD_NOT_FINISHED) ? running : finished).push_back(&p);
    }
    std::vector<std::pair<const PodObj*, uint8_t>> queued;
    for (size_t i = 0; i < pend_rows.size(); ++i) {
      const int64_t r = pend_rows[i];
      // (free queue rows are tombstones, which a selector without requirements still matches on the pending side; scratch
      // rows hold manifests, not queued pods)
      if (r < (int64_t)pend_pod.size() && pend_pod[(size_t)r] >= 0) queued.emplace_back(&pods[(size_t)pend_pod[(size_t)r]], codes[i]);
    }
    std::sort(running.begin(), running.end(), by_key);
    std::sort(finished.begin(), finished.end(), by_key);
    std::sort(queued.begin(), queued.end(), [&](const auto& a, const auto& b) { return by_key(a.first, b.first); });
    static const char* const kStatus[4] = {"not-throttled", "active", "insufficient", "pod-requests-exceeds-threshold"};
    Writer w;
    w.begin_obj().key("pods").begin_arr();
    for (const PodObj* p : running) w.str(p->nn());
    w.end_arr().key("terminatedPods").begin_arr();
    for (const PodObj* p : finished) w.str(p->nn());
    w.end_arr().key("queued").begin_arr();
    for (auto& q : queued) w.begin_obj().key("pod").str(q.first->nn()).key("status").str(kStatus[q.second & 3u]).end_obj();
    w.end_arr().end_obj();
    return w.out;
  }

  // ---- the scheduling queue per throttle (kth_queue_report) ----------------------------------------------------------
  // The verdicts are kth_pre_filter_queue's: the cached ones when they are current, else those of the one pass that refreshes
  // them.  The per-throttle numbers come from one kt_get_check_summary over the device codes, which must be those of a pass at
  // this state: the refresh just run, or the last pass of kth_affected_pods or of this call at the same `epoch` (the cached
  // verdicts being current says nothing about what the device holds: other calls run passes of their own); else one runs here.
  uint64_t codes_epoch = 0;
  std::string queue_report() {
    if (!kt_get_check_summary) fail("kth_queue_report: the engine this plugin is linked against has no kt_get_check_summary");
    const int64_t n = (int64_t)pend_pod.size();
    std::vector<uint8_t> verdicts((size_t)n);
    const uint64_t passes = queue.passes;
    pre_filter_queue(verdicts.data(), n);
    if (queue.passes != passes) codes_epoch = epoch;
    if (codes_epoch != epoch) {
      run_pending_pass({}, 0);
      codes_epoch = epoch;
    }
    int64_t count[4] = {0, 0, 0, 0};
    for (uint8_t v : verdicts) ++count[v & 3u];
    std::vector<size_t> ours;  // (the pass may have laid the columns out anew)
    for (size_t t = 0; t < throttles.size(); ++t)
      if (throttles[t].live && throttles[t].throttler_name == name) ours.push_back(t);
    creation_order(ours);
    const size_t m = throttles.size(), R = (size_t)lim.n_resources;
    std::vector<int64_t> status_cnt(3 * m), sole_cnt(m), held(R * m);
    std::vector<uint32_t> held_present(m);
    if (!ours.empty()) {
      // class 0: free queue rows (tombstones, which a selector without requirements still matches); 2: PreFilter is Error
      std::vector<uint8_t> cls((size_t)pend_capacity, 0);
      for (int64_t r = 0; r < n; ++r) cls[(size_t)r] = verdicts[(size_t)r] == 3 ? 2 : verdicts[(size_t)r] != 0 ? 1 : 0;
      const kt_check_summary out{status_cnt.data(), sole_cnt.data(), held.data(), held_present.data()};
      check(kt_get_check_summary(ctx, 0, pend_capacity, cls.data(), &out), "kt_get_check_summary");
    }
    Writer w;
    w.begin_obj().key("queued").num((long long)(count[1] + count[2] + count[3])).key("success").num((long long)count[1]);
    w.key("unschedulable").num((long long)count[2]).key("error").num((long long)count[3]).key("throttles").begin_arr();
    for (size_t t : ours) {
      const ThrottleObj& o = throttles[t];
      w.begin_obj().key("key").str(o.nn()).key("kind").str(o.kind == KT_KIND_THROTTLE ? "Throttle" : "ClusterThrottle");
      w.key("active").num((long long)status_cnt[t]).key("insufficient").num((long long)status_cnt[m + t]);
      w.key("podRequestsExceedsThreshold").num((long long)status_cnt[2 * m + t]).key("onlyBlocker").num((long long)sole_cnt[t]);
      ResAmount a;  // ResourceAmount{} .Add(ResourceAmountOfPod(p)) over the held-back pods, as reconcile sums status.used
      if (held_present[t] & KT_COUNT_BIT) {
        a.has_counts = true;
        a.pod = (long long)(status_cnt[t] + status_cnt[m + t] + status_cnt[2 * m + t]);
        a.requests_nil = false;
        for (size_t r = 0; r < cols.size() && r < R; ++r)
          if ((held_present[t] >> r) & 1) a.requests[(int)r] = from_scale((int)r, held[r * m + t]);
      }
      w.key("heldBack");
      amount_json(w, a);
      w.end_obj();
    }
    w.end_arr().end_obj();
    return w.out;
  }

  // ---- reconcile(key) for listed throttles (kth_reconcile) -----------------------------------------------------------
  // Each distinct key gets what reconcile_all does for its throttle (reconcile_throttle) from one kt_reconcile_throttles call
  // over the listed columns only.  Throttles that are not listed are not touched.
  std::string reconcile_keys(const std::string& keys_json, const std::string& now_s) {
    GoTime now;
    std::string e = parse_rfc3339(now_s, &now);
    if (!e.empty()) fail(e);
    ktjson::NodePtr keys = ktjson::parse(keys_json.c_str());
    if (!keys->is(Node::Arr)) fail("reconcile: keys must be a JSON array of \"namespace/name\" (Throttle) or \"/name\" (ClusterThrottle)");
    if (!kt_reconcile_throttles) fail("kth_reconcile: the engine this plugin is linked against has no kt_reconcile_throttles");
    sync_all();  // (may lay the throttle columns out anew: keys are resolved after it)
    ReconcileReport rep;
    std::vector<std::pair<std::string, int32_t>> todo;  // key, throttle column
    std::set<std::string> seen;
    for (auto& kp : keys->arr) {
      if (!kp->is(Node::Str)) fail("reconcile: every key must be a string");
      const std::string key = kp->text;
      if (!seen.insert(key).second) continue;
      // cache.SplitMetaNamespaceKey, with "/name" for a ClusterThrottle (controller.go:95-101)
      const size_t slash = key.find('/');
      const std::string ns = slash == std::string::npos ? "" : key.substr(0, slash), tname = slash == std::string::npos ? "" : key.substr(slash + 1);
      if (slash == std::string::npos || tname.empty() || tname.find('/') != std::string::npos) {
        rep.errors.emplace_back(key, "unexpected key format: \"" + key + "\"");
        continue;
      }
      const int t = find_throttle(ns, tname);
      if (t < 0 || !throttles[(size_t)t].live) { rep.not_found.push_back(key); continue; }  // the lister's NotFound: nil
      if (throttles[(size_t)t].throttler_name != name) continue;  // only responsible throttles are ever enqueued (:403-425)
      todo.emplace_back(key, (int32_t)t);
    }
    const size_t k = todo.size();
    std::vector<int32_t> idx(k);
    for (size_t q = 0; q < k; ++q) idx[q] = todo[q].second;
    ReconcileCols st(k, lim.n_resources);
    std::vector<int64_t> off(k + 1, 0), rows;
    int64_t cap = 1024;
    while (k) {  // the matched rows of every listed throttle, ascending
      rows.resize((size_t)cap);
      check(kt_reconcile_throttles(ctx, clamp_ns(now.ns()), (int64_t)k, idx.data(), &st.out, off.data(), rows.data(), cap), "kt_reconcile_throttles");
      if (off[k] <= cap) break;
      cap = off[k];
    }
    for (size_t q = 0; q < k; ++q) {
      const size_t t = (size_t)idx[q];
      const int64_t* r0 = rows.data() + off[q];
      const int64_t* r1 = rows.data() + off[q + 1];
      auto matched = [&](int64_t r) { return std::binary_search(r0, r1, r); };
      const std::string err = reconcile_throttle(t, matched, selector_error_rows(throttles[t]), r0, r1, st, (int64_t)q, now, rep);
      if (!err.empty()) rep.errors.emplace_back(todo[q].first, err);
    }
    return rep.json(true);
  }

  // ---- pending pods: one device pass for a batch ----------------------------------------------------------
  struct RowView {  // one pending pod's share of a pass: affectedThrottles row, 2-bit check codes, admit bit
    const uint32_t* bitmap;
    const uint32_t* codes;
    uint8_t admit;
    int Wp;
  };
  struct PendingResult {  // k pending rows: Wp match words, 2 * Wp check-code words and the admit byte each
    std::vector<uint32_t> bitmap, codes;
    std::vector<uint8_t> admit;
    int Wp = 0;
    PendingResult() = default;
    PendingResult(size_t k, int Wp) : bitmap(k * (size_t)Wp, 0), codes(k * 2 * (size_t)Wp, 0), admit(k, 1), Wp(Wp) {}
    RowView row(size_t i) const { return RowView{bitmap.data() + i * (size_t)Wp, codes.data() + i * 2 * (size_t)Wp, admit[i], Wp}; }
  };
  // The PENDING table's capacities for the queue and k scratch rows.  A capacity that grows means a full upload, which re-packs
  // every row and so voids the cached verdicts -- at once, also on the paths that check a batch without uploading it
  // (check_pending), so that the queue cache keeps one rule whichever path checked the batch.
  void size_pending(int64_t k) {
    int64_t want_q = std::max<int64_t>(64, pend_capacity), want_s = std::max<int64_t>(16, scratch_capacity);
    while (want_q < (int64_t)pend_pod.size()) want_q *= 2;
    while (want_s < k) want_s *= 2;
    if (want_q != pend_capacity || want_s != scratch_capacity) {
      pend_capacity = want_q;
      scratch_capacity = want_s;
      pend_full_upload = true;
    }
    if (pend_full_upload) queue.valid = false;
  }
  // The device's PENDING table = the resident queue rows + `k` scratch rows holding `batch` (pods that are not in the informer
  // cache), brought up to date together with the state a PreFilter view reads (sync_state).  Row deltas; a full upload only
  // when a capacity grows or the packing changed.
  void sync_pending(const std::vector<PodObj>& batch) {
    sync_state();
    const int L = lim.label_slots, R = lim.n_resources;
    const int64_t k = (int64_t)batch.size();
    size_pending(k);
    const bool full = pend_full_upload;
    const int64_t first_scratch = pend_capacity;
    std::vector<int64_t> rows;  // the rows a delta packs (a full upload packs every row)
    if (!full) {
      rows.assign(pend_dirty.begin(), pend_dirty.end());
      const int64_t n_scratch = std::max(k, scratch_used);  // this batch, and what the last one left behind
      for (int64_t i = 0; i < n_scratch; ++i) rows.push_back(pend_capacity + i);
    }
    const size_t n = full ? (size_t)(pend_capacity + scratch_capacity) : rows.size();
    if (n) {
      PodObj tomb;
      auto pod_at = [&](int64_t row) -> const PodObj& {
        if (row >= first_scratch) return row - first_scratch < k ? batch[(size_t)(row - first_scratch)] : tomb;
        const int64_t slot = row < (int64_t)pend_pod.size() ? pend_pod[(size_t)row] : -1;
        return slot >= 0 ? pods[(size_t)slot] : tomb;
      };
      std::vector<int64_t> lab((size_t)L * n), req((size_t)R * n);
      std::vector<uint32_t> present(n), flags(n);
      std::vector<int32_t> nsid(n);
      for (size_t i = 0; i < n; ++i) pack_pod(pod_at(full ? (int64_t)i : rows[i]), lab, req, present, flags, nsid, n, i);
      if (namespaces_dirty || throttles_dirty) sync_state();  // packing introduced new namespace ids
      if (full)
        check(kt_upload_pods(ctx, KT_PODS_PENDING, (int64_t)n, lab.data(), req.data(), present.data(), flags.data(), nsid.data()), "kt_upload_pods(pending)");
      else
        check(kt_update_pod_rows(ctx, KT_PODS_PENDING, (int64_t)n, rows.data(), lab.data(), req.data(), present.data(), flags.data(), nsid.data()),
              "kt_update_pod_rows(pending)");
    }
    if (full) pend_full_upload = false;
    pend_dirty.clear();
    scratch_used = k;
  }
  // One pass over the PENDING table (queue + scratch rows): PreFilter reads the informer copy of .status; reconcile is a
  // separate event (KT_EVAL_GIVEN_STATUS).  Afterwards the device holds the verdicts of every queue row at this state.
  // (kth_affected_pods asks for skip = 0: the running relation of the same state as well)
  void run_pending_pass(const std::vector<PodObj>& batch, uint32_t extra_flags, uint32_t skip = KT_EVAL_SKIP_RECONCILE) {
    sync_pending(batch);
    if (throttles.empty()) return;
    check(kt_evaluate(ctx, 0, KT_EVAL_GIVEN_STATUS | skip | extra_flags), "kt_evaluate");
  }
  // The first k scratch rows as the pass (or kt_admit_queue) that just ran left them.
  PendingResult scratch_rows(size_t k) {
    PendingResult out(k, kt_match_words(ctx));
    if (throttles.empty() || k == 0) return out;
    std::vector<int64_t> rows(k);
    for (size_t i = 0; i < k; ++i) rows[i] = pend_capacity + (int64_t)i;
    check(kt_get_check_rows(ctx, (int64_t)k, rows.data(), out.codes.data(), out.admit.data()), "kt_get_check_rows");
    check(kt_get_match_rows(ctx, KT_PODS_PENDING, (int64_t)k, rows.data(), out.bitmap.data()), "kt_get_match_rows");
    return out;
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
    queue.m = throttles.size();
    queue.pass_col.clear();
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
    if (!queue.valid || throttles_dirty || (namespaces_dirty && namespaces_full) || pend_full_upload) return false;
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

  // PreFilter of pods given by value (manifests, and informer pods checked like one).  With kt_check_pods the batch is packed and
  // checked in one call that costs the words of each pod's namespace: no row is uploaded and no pass runs, so the device keeps
  // the codes of the last pass, which kth_affected_pods and kth_queue_report only reuse at an unchanged `epoch` (every
  // non-reading entry point moves it).  Without it (older engine doubles) the batch takes scratch rows behind the queue and one
  // pass over both.  Either way the state is synced first and the capacities are sized for the batch (size_pending), so that the
  // statuses, reservations, cached verdicts and errors come out the same.
  PendingResult check_pending(const std::vector<PodObj>& batch, uint32_t extra_flags) {
    if (!kt_check_pods) {
      run_pending_pass(batch, extra_flags);
      return scratch_rows(batch.size());
    }
    sync_state();
    size_pending((int64_t)batch.size());
    const size_t k = batch.size();
    const int L = lim.label_slots, R = lim.n_resources;
    std::vector<int64_t> lab((size_t)L * k), req((size_t)R * k);
    std::vector<uint32_t> present(k), flags(k);
    std::vector<int32_t> nsid(k);
    for (size_t i = 0; i < k; ++i) pack_pod(batch[i], lab, req, present, flags, nsid, k, i);
    if (namespaces_dirty || throttles_dirty) sync_state();  // packing introduced new namespace ids
    PendingResult out(k, kt_match_words(ctx));
    if (throttles.empty() || k == 0) return out;
    check(kt_check_pods(ctx, extra_flags, (int64_t)k, lab.data(), req.data(), present.data(), nsid.data(), out.bitmap.data(), out.codes.data(),
                        out.admit.data()),
          "kt_check_pods");
    return out;
  }
  // PreFilter of a pod of the resident queue: from the cached verdicts when they are current, else after ONE pass that
  // refreshes the whole queue's.
  PendingResult queue_result(int64_t row) {
    if (!queue_row_current(row)) refresh_queue();
    else ++queue.hits;
    const int Wp = std::max(queue.Wp, match_words(throttles.size()));
    PendingResult out(1, Wp);
    cached_row(row, Wp, out.bitmap.data(), out.codes.data());
    out.admit[0] = queue.admit[(size_t)row];
    return out;
  }
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
  std::string controller_error(const PodObj& pod, const RowView& r, int kind) {
    if (kind == KT_KIND_CLUSTERTHROTTLE) {
      const int id = ns_dict.find(pod.ns);
      if (id < 0 || !namespaces[(size_t)id].exists) return "namespace \"" + pod.ns + "\" not found";  // namespaceInformer.Lister().Get (clusterthrottle_controller.go:273-276)
    }
    for (size_t t : broken_throttles()) {
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
  // PreFilter for a list of keys in ONE kt_check_pending_rows call over the listed rows only: each entry is what pre_filter_key
  // would return at this moment, but nothing is read from or written to the cached queue verdicts (no pass, no hit).  Pods the
  // informer holds that are not queued take scratch rows of the same call.
  std::string pre_filter_keys(const std::string& keys_json) {
    ktjson::NodePtr keys = ktjson::parse(keys_json.c_str());
    if (!keys->is(Node::Arr)) fail("pre_filter_keys: keys must be a JSON array of \"namespace/name\" strings");
    if (!kt_check_pending_rows) fail("kth_pre_filter_keys: the engine this plugin is linked against has no kt_check_pending_rows");
    const size_t n = keys->arr.size();
    std::vector<std::string> err(n), key(n);
    std::vector<int64_t> scratch_of(n, -1);  // index into `batch` of a pod that is not queued
    std::vector<PodObj> batch;
    for (size_t i = 0; i < n; ++i) {
      const Node& kp = *keys->arr[i];
      if (!kp.is(Node::Str)) { err[i] = "pre_filter_keys: every key must be a string"; continue; }
      key[i] = kp.text;
      const size_t slash = key[i].find('/');
      if (slash == std::string::npos || slash + 1 == key[i].size() || key[i].find('/', slash + 1) != std::string::npos) {
        err[i] = "unexpected key format: \"" + key[i] + "\"";
        continue;
      }
      auto it = pod_index.find(key[i]);
      if (it == pod_index.end()) { err[i] = "pod " + key[i] + " is not in the informer cache"; continue; }
      const PodObj& pod = pods[(size_t)it->second];
      if (pod.pend_row < 0) { scratch_of[i] = (int64_t)batch.size(); batch.push_back(pod); }  // (value copy: the sync may re-pack)
    }
    // the state sync every entry point does (it may void cached verdicts, as anywhere else), then the rows as they are now
    sync_pending(batch);
    std::vector<int64_t> rows, at(n, -1);
    std::vector<PodObj> who;
    for (size_t i = 0; i < n; ++i) {
      if (!err[i].empty()) continue;
      at[i] = (int64_t)rows.size();
      if (scratch_of[i] >= 0) {
        rows.push_back(pend_capacity + scratch_of[i]);
        who.push_back(batch[(size_t)scratch_of[i]]);
      } else {
        const PodObj& pod = pods[(size_t)pod_index.at(key[i])];
        rows.push_back(pod.pend_row);
        who.push_back(pod);
      }
    }
    const size_t k = rows.size();
    PendingResult r(k, kt_match_words(ctx));
    if (!throttles.empty() && k)  // PreFilter passes isThrottledOnEqual = false
      check(kt_check_pending_rows(ctx, 0, (int64_t)k, rows.data(), r.bitmap.data(), r.codes.data(), r.admit.data()), "kt_check_pending_rows");
    Writer w;
    w.begin_arr();
    for (size_t i = 0; i < n; ++i) {
      if (at[i] < 0) w.begin_obj().key("error").str(err[i]).end_obj();
      else prefilter_json(w, who[(size_t)at[i]], r.row((size_t)at[i]));
    }
    w.end_arr();
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
    const bool any_broken = !broken_throttles().empty();
    const int Wp = std::max(queue.Wp, match_words(throttles.size()));
    const std::vector<uint32_t> no_codes(2 * (size_t)Wp, 0);
    std::vector<uint32_t> bm((size_t)Wp);
    for (int64_t row = 0; row < n && row < cap; ++row) {
      const int64_t slot = pend_pod[(size_t)row];
      if (slot < 0) { verdicts[row] = 0; continue; }
      uint8_t v = queue.admit[(size_t)row] ? 1 : 2;
      const PodObj& pod = pods[(size_t)slot];
      const int nsid = ns_dict.find(pod.ns);
      if (any_broken || nsid < 0 || !namespaces[(size_t)nsid].exists) {  // the error paths that never reach the device
        cached_row(row, Wp, bm.data(), nullptr);
        const RowView rv{bm.data(), no_codes.data(), queue.admit[(size_t)row], Wp};
        if (!controller_error(pod, rv, KT_KIND_THROTTLE).empty() || !controller_error(pod, rv, KT_KIND_CLUSTERTHROTTLE).empty()) v = 3;
      }
      verdicts[row] = v;
    }
    return n;
  }

  // ---- queue-ordered admission on the device (kt_admit_queue, csrc/kt_admit.cuh) ------------------------------
  bool admit_queue_on_device_possible(const std::vector<PodObj>& queue) {
    if (throttles.empty() || queue.empty()) return false;
    if (!broken_throttles().empty()) return false;  // some pod may run into a conversion error: framework.Error, no Reserve
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
    sync_pending(queue);
    int32_t rounds = 0;
    int64_t admitted_dev = 0;
    check(kt_admit_queue(ctx, pend_capacity, (int64_t)n, 0, &rounds, &admitted_dev), "kt_admit_queue");
    const PendingResult r = scratch_rows(n);
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
        prefilter_json(w, batch[k], r.row(k));
        results[i] = w.out;
        round_of[i] = rounds;
        bool success = w.out.compare(0, 17, "{\"code\":\"Success\"") == 0;
        if (!success) continue;
        // Reserve (throttle_controller.go:271-292): ResourceAmountOfPod joins the reservation of every affected throttle
        bool reserve_error = false;
        for (int kind = 0; kind < 2; ++kind) reserve_error = reserve_error || !controller_error(batch[k], r.row(k), kind).empty();
        if (reserve_error) continue;
        ++admitted;
        for (int kind = 0; kind < 2; ++kind)
          for (int t : affected(r.row(k), kind)) { cache[kind].add(throttles[(size_t)t].nn(), batch[k]); reservation_changed((size_t)t); }
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
  // The informer's copy of a pod is replaced (or added): returns whether the plugin held the pod before, with that copy in *old.
  bool store_pod(PodObj p, PodObj* old) {
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
      return false;
    }
    const int64_t row = it->second;
    *old = pods[(size_t)row];
    p.row = row;
    p.seq = old->seq;
    p.pend_row = old->pend_row;
    totals_add(*old, -1);
    totals_add(p, +1);
    pods[(size_t)row] = std::move(p);
    dirty_rows.insert(row);
    queue_update(row);
    return true;
  }
  // UpdateFunc (throttle_controller.go:459-507): the throttle assignment can only change with labels / namespace;
  // then the pod's reservation moves from (old \ new) to (new \ old) throttles
  bool moves_reservation(const PodObj& old, const PodObj& cur) const {
    return (should_count_in(old) || should_count_in(cur)) && !throttles.empty() && old.labels != cur.labels;
  }
  void move_reservation(const PodObj& old, const PodObj& now, const RowView& ro, const RowView& rn) {
    for (int kind = 0; kind < 2; ++kind) {
      if (!controller_error(old, ro, kind).empty() || !controller_error(now, rn, kind).empty()) continue;  // HandleError + return
      const std::vector<int> a = affected(ro, kind), b = affected(rn, kind);
      for (int t : a)
        if (std::find(b.begin(), b.end(), t) == b.end()) { cache[kind].remove(throttles[(size_t)t].nn(), now.nn()); reservation_changed((size_t)t); }
      for (int t : b)
        if (std::find(a.begin(), a.end(), t) == a.end()) { cache[kind].add(throttles[(size_t)t].nn(), now); reservation_changed((size_t)t); }
    }
  }
  void apply_pod(const Node& v) {
    // The informer's copy is replaced FIRST: the pass below only asks which throttles the old and the new pod match, which
    // does not depend on the running rows, and an update that repairs a snapshot the packer refuses (column overflow) must
    // not be refused for it.
    PodObj old;
    PodObj p = pod_from(v);
    const int64_t slot = pod_index.count(p.nn()) ? pod_index.at(p.nn()) : -1;
    if (!store_pod(std::move(p), &old)) return;
    const PodObj& cur = pods[(size_t)slot];
    if (moves_reservation(old, cur)) {
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
      move_reservation(old, now, r.row(0), r.row(1));
    }
  }
  // The pod leaves the informer cache: returns whether the plugin held it, with its last copy in *old.
  bool drop_pod(const std::string& ns, const std::string& pname, PodObj* old) {
    auto it = pod_index.find(ns + "/" + pname);
    if (it == pod_index.end()) return false;
    const int64_t row = it->second;
    *old = pods[(size_t)row];
    // the row goes first (see apply_pod): a delete that repairs a refused snapshot must not be refused for it
    totals_add(*old, -1);
    if (old->pend_row >= 0) queue_release(old->pend_row);
    pods[(size_t)row] = PodObj();  // tombstone row: flags == 0, no labels
    pods[(size_t)row].row = row;
    pod_index.erase(it);
    ns_free_rows[old->ns].push_back(row);  // the slot stays with its namespace's arena
    dirty_rows.insert(row);
    return true;
  }
  // DeleteFunc (:509-515): a scheduled pod that disappears is un-reserved from its affected throttles
  bool unreserves(const PodObj& old) const { return should_count_in(old) && !old.node_name.empty() && !throttles.empty(); }
  void unreserve_deleted(const PodObj& old, const RowView& r) {
    for (int kind = 0; kind < 2; ++kind) {
      if (!controller_error(old, r, kind).empty()) continue;
      for (int t : affected(r, kind))
        if (cache[kind].remove(throttles[(size_t)t].nn(), old.nn())) reservation_changed((size_t)t);
    }
  }
  // the pod is gone whatever happens to the pass: its reservations must not outlive it (reconcile only un-reserves pods that are
  // still in the index) -- without the device's answer it leaves every throttle's reservation, a superset
  void unreserve_everywhere(const PodObj& old) {
    for (int kind = 0; kind < 2; ++kind)
      if (cache[kind].remove_everywhere(old.nn())) { reserved_dirty = true; queue_void(); }
  }
  void delete_pod(const std::string& ns, const std::string& pname) {
    PodObj old;
    if (!drop_pod(ns, pname, &old)) return;
    if (unreserves(old)) {
      PendingResult r;
      try {
        r = check_pending({old}, 0);
      } catch (...) {
        unreserve_everywhere(old);
        throw;
      }
      unreserve_deleted(old, r.row(0));
    }
  }
  void delete_namespace(const std::string& nm) {
    const int id = ns_dict.find(nm);
    if (id >= 0) { namespaces[(size_t)id].exists = false; namespaces[(size_t)id].labels.clear(); namespace_changed(id); }
  }

  // ---- informer events in batches (kth_apply_events) ----------------------------------------------------------------
  // The reference's controllers reconcile what their informer handlers enqueue (throttle_controller.go:401-531,
  // clusterthrottle_controller.go:433-563).  A batch of watch events is applied in order; the pod events between two table
  // events (Throttle, ClusterThrottle, Namespace) form a run whose pod versions take ONE kt_match_pods call, after the events of
  // the run are stored.  The tables cannot change inside a run, and no affected set depends on reservations, so the run's
  // reservation edits -- the same ones apply_pod / delete_pod make -- are applied afterwards, in event order, with the same
  // result as event by event.
  struct PodEvent {
    size_t ev = 0;
    bool keys = false;         // the handler enqueues the affected throttles (shouldCountIn of a version it looks at)
    bool move = false;         // UpdateFunc moves the reservation (moves_reservation)
    bool unreserve = false;    // DeleteFunc un-reserves a counted, scheduled pod (unreserves)
    std::vector<PodObj> ver;   // the versions the handler looks at: {new} AddFunc, {old, new} UpdateFunc, {old} DeleteFunc
    std::vector<size_t> at;    // each version's row in the run's match result
  };
  struct EventOut {
    std::string error, warning;
    bool keys = false;                 // the entry carries "enqueue"
    std::vector<std::string> enqueue;  // reconcile keys, creation order
  };
  // affectedThrottles of each version (one device call for the distinct (namespace, label set) pairs), as a PendingResult
  PendingResult match_versions(const std::vector<PodObj>& vers) {
    sync_state();
    const int L = lim.label_slots;
    const size_t k = vers.size();
    std::vector<int64_t> lab((size_t)L * k, KT_LABEL_EMPTY);
    std::vector<int32_t> nsid(k);
    for (size_t i = 0; i < k; ++i) {  // the label slots pack_pod gives a pending row
      int s = 0;
      for (auto& kv : vers[i].labels) {
        const int64_t code = labels.encode(kv.first, kv.second);
        if (code != KT_LABEL_EMPTY) lab[(size_t)(s++) * k + i] = code;
      }
      nsid[i] = ns_id(vers[i].ns);
    }
    if (namespaces_dirty || throttles_dirty) sync_state();  // packing introduced new namespace ids
    PendingResult r(k, kt_match_words(ctx));
    check(kt_match_pods(ctx, (int64_t)k, lab.data(), nsid.data(), r.bitmap.data()), "kt_match_pods");
    return r;
  }
  // The keys a pod event enqueues: per controller, the affected throttles of every version the handler looks at, or none when
  // affectedThrottles fails for one of them (HandleError + return; the other controller has its own handler).
  std::vector<std::string> enqueued(const PodEvent& pe, const PendingResult& r) {
    std::vector<int> cols_hit;
    for (int kind = 0; kind < 2; ++kind) {
      std::vector<int> mine;
      bool failed = false;
      for (size_t j = 0; j < pe.ver.size() && !failed; ++j) {
        const RowView row = r.row(pe.at[j]);
        if (!controller_error(pe.ver[j], row, kind).empty()) failed = true;
        else for (int t : affected(row, kind)) mine.push_back(t);
      }
      if (!failed) cols_hit.insert(cols_hit.end(), mine.begin(), mine.end());
    }
    std::sort(cols_hit.begin(), cols_hit.end());
    cols_hit.erase(std::unique(cols_hit.begin(), cols_hit.end()), cols_hit.end());
    creation_order(cols_hit);
    std::vector<std::string> keys;
    for (int t : cols_hit) keys.push_back(throttles[(size_t)t].nn());
    return keys;
  }
  // One device call for a run of pod events, then their reservation edits in event order and their keys.  When the call fails,
  // each event reports what kth_apply / kth_delete report when their pass fails (the move is skipped with a warning; a deleted
  // pod leaves every reservation and the event is an error), and none carries keys.
  void match_run(std::vector<PodEvent>& run, std::vector<EventOut>& out) {
    if (run.empty()) return;
    std::vector<PodObj> uniq;
    std::map<std::pair<std::string, std::vector<std::pair<std::string, std::string>>>, size_t> seen;
    for (auto& pe : run) {
      pe.at.clear();
      for (auto& v : pe.ver) {
        auto labs = v.labels;
        std::sort(labs.begin(), labs.end());
        auto ins = seen.emplace(std::make_pair(v.ns, std::move(labs)), uniq.size());
        if (ins.second) uniq.push_back(v);
        pe.at.push_back(ins.first->second);
      }
    }
    PendingResult r;
    std::string err;
    try {
      r = match_versions(uniq);
    } catch (const std::exception& e) {
      err = e.what();
    }
    for (auto& pe : run) {
      EventOut& o = out[pe.ev];
      if (!err.empty()) {
        o.keys = false;
        if (pe.move) o.warning = "pod updated; reservation move skipped: " + err;
        else if (pe.unreserve) { unreserve_everywhere(pe.ver[0]); o.error = err; }
        else o.warning = "affected throttles not computed: " + err;
        continue;
      }
      if (pe.move) move_reservation(pe.ver[0], pe.ver[1], r.row(pe.at[0]), r.row(pe.at[1]));
      if (pe.unreserve) unreserve_deleted(pe.ver[0], r.row(pe.at[0]));
      if (pe.keys) o.enqueue = enqueued(pe, r);
    }
    run.clear();
  }
  // One watch event: the state change kth_apply / kth_delete makes, with the pod pass left to the run.
  void apply_event(const std::string& type, const std::string& kind, const Node& obj, size_t i, EventOut& o, std::vector<PodEvent>& run) {
    const bool is_thr = kind == "Throttle" || kind == "ClusterThrottle";
    const int tkind = kind == "Throttle" ? KT_KIND_THROTTLE : KT_KIND_CLUSTERTHROTTLE;
    if (type == "DELETED") {
      const std::string ns = obj["metadata"]["namespace"].str(), nm = obj["metadata"]["name"].str();
      if (kind == "Pod") {
        PodObj old;
        if (drop_pod(ns, nm, &old) && should_count_in(old) && !throttles.empty()) {
          PodEvent pe;
          pe.ev = i;
          pe.keys = true;
          pe.unreserve = unreserves(old);
          pe.ver = {old};
          run.push_back(std::move(pe));
        }
      } else if (is_thr) {  // DeleteFunc: isResponsibleFor the object the plugin held
        auto it = thr_index.find(thr_key(tkind, ns, nm));
        if (it != thr_index.end() && throttles[(size_t)it->second].throttler_name == name) o.enqueue.push_back(throttles[(size_t)it->second].nn());
        delete_throttle(tkind, ns, nm);
      } else if (kind == "Namespace") {
        delete_namespace(nm);
      } else {
        fail("unsupported kind: " + kind);
      }
    } else if (kind == "Pod") {
      PodObj p = pod_from(obj);
      const std::string nn = p.nn();
      PodObj old;
      const bool held = store_pod(std::move(p), &old);
      const PodObj& cur = pods[(size_t)pod_index.at(nn)];
      PodEvent pe;
      pe.ev = i;
      if (held) {  // UpdateFunc: the plugin's own store decides, as in kth_apply
        pe.keys = should_count_in(old) || should_count_in(cur);
        pe.move = moves_reservation(old, cur);
        pe.ver = {old, cur};
      } else {     // AddFunc
        pe.keys = should_count_in(cur);
        pe.ver = {cur};
      }
      if ((pe.keys && !throttles.empty()) || pe.move) run.push_back(std::move(pe));
    } else if (kind == "Namespace") {
      apply_namespace(obj);
    } else if (is_thr) {  // AddFunc / UpdateFunc: isResponsibleFor the new object
      apply_throttle(obj, tkind);
      const ThrottleObj& t = throttles[(size_t)thr_index.at(thr_key(tkind, obj["metadata"]["namespace"].str(), obj["metadata"]["name"].str()))];
      if (t.throttler_name == name) o.enqueue.push_back(t.nn());
    } else {
      fail("unsupported kind: " + kind);
    }
    o.keys = true;
  }
  std::string apply_events(const std::string& events_json) {
    ktjson::NodePtr evs = ktjson::parse(events_json.c_str());
    if (!evs->is(Node::Arr)) fail("apply_events: events must be a JSON array of watch events");
    if (!kt_match_pods) fail("kth_apply_events: the engine this plugin is linked against has no kt_match_pods");
    const size_t n = evs->arr.size();
    std::vector<EventOut> out(n);
    std::vector<PodEvent> run;
    for (size_t i = 0; i < n; ++i) {
      const Node& e = *evs->arr[i];
      EventOut& o = out[i];
      const std::string at = "event " + std::to_string(i) + ": ";
      if (!e.is(Node::Obj)) { o.error = at + "a watch event must be an object"; continue; }
      const std::string type = e["type"].str();
      if (type != "ADDED" && type != "MODIFIED" && type != "DELETED") { o.error = at + "unknown type \"" + type + "\""; continue; }
      const Node& obj = e["object"];
      if (!obj.is(Node::Obj)) { o.error = at + "missing object"; continue; }
      const std::string kind = obj["kind"].str();
      if (kind == "Throttle" || kind == "ClusterThrottle" || kind == "Namespace") match_run(run, out);  // the tables change here
      const size_t n_cols = cols.size();
      apply_committed = false;
      apply_warning.clear();
      try {
        apply_event(type, kind, obj, i, o, run);
      } catch (const std::exception& ex) {
        if (type != "DELETED" && !apply_committed) rollback_columns(n_cols);  // as kth_apply: the refused object's resource names go with it
        o.error = ex.what();
        o.keys = false;
        o.enqueue.clear();
      }
    }
    match_run(run, out);
    Writer w;
    std::vector<std::string> all;
    std::unordered_set<std::string> in_all;
    w.begin_obj().key("results").begin_arr();
    for (auto& o : out) {
      w.begin_obj();
      if (!o.error.empty()) {
        w.key("error").str(o.error).end_obj();
        continue;
      }
      w.key("ok").raw("true");
      if (!o.warning.empty()) w.key("warning").str(o.warning);
      if (o.keys) {
        w.key("enqueue").begin_arr();
        for (auto& k : o.enqueue) {
          w.str(k);
          if (in_all.insert(k).second) all.push_back(k);
        }
        w.end_arr();
      }
      w.end_obj();
    }
    w.end_arr().key("enqueue").begin_arr();
    for (auto& k : all) w.str(k);
    w.end_arr().end_obj();
    return w.out;
  }

  void apply_namespace(const Node& v) {
    const std::string nm = v["metadata"]["name"].str();
    const Node& lab = v["metadata"]["labels"];
    // refuse before touching any state: the object is rejected, the plugin stays usable
    if ((int)lab.obj.size() > KT_MAX_LABEL_SLOTS - 1)  // one slot is the internal "exists" label
      fail("namespace " + nm + " has more than " + std::to_string(KT_MAX_LABEL_SLOTS - 1) + " labels");
    const int32_t id = ns_id(nm, true);
    NamespaceObj& n = namespaces[(size_t)id];
    n.exists = true;
    n.labels.clear();
    for (auto& kv : lab.obj) n.labels.emplace_back(kv.first, kv.second->str());
    if ((int)n.labels.size() > max_ns_labels) {
      max_ns_labels = (int)n.labels.size();
      if (ctx && max_ns_labels + 1 > lim.ns_label_slots) drop_engine();
    }
    namespace_changed(id);
  }
  // Everything of two throttles of one key that the compiled tables and the per-column spec on the device are made of.
  static bool same_selector(const CompiledSelector& a, const CompiledSelector& b) {
    if (a.error != b.error || a.reqs.size() != b.reqs.size()) return false;
    for (size_t i = 0; i < a.reqs.size(); ++i)
      if (a.reqs[i].key != b.reqs[i].key || a.reqs[i].op != b.reqs[i].op || a.reqs[i].values != b.reqs[i].values) return false;
    return true;
  }
  // What compile_tables and the column layout read: kind, namespace, throttlerName (the responsibility flag) and the terms.
  static bool same_tables(const ThrottleObj& a, const ThrottleObj& b) {
    if (a.kind != b.kind || a.ns != b.ns || a.throttler_name != b.throttler_name || a.terms.size() != b.terms.size()) return false;
    for (size_t i = 0; i < a.terms.size(); ++i)
      if (!same_selector(a.terms[i].pod_sel, b.terms[i].pod_sel) || !same_selector(a.terms[i].ns_sel, b.terms[i].ns_sel)) return false;
    return true;
  }
  // What threshold_columns reads: spec.threshold and the temporaryThresholdOverrides.
  static bool same_threshold_columns(const ThrottleObj& a, const ThrottleObj& b) {
    if (!amount_equal(a.threshold, b.threshold) || a.overrides.size() != b.overrides.size()) return false;
    for (size_t i = 0; i < a.overrides.size(); ++i)
      if (a.overrides[i].begin != b.overrides[i].begin || a.overrides[i].end != b.overrides[i].end || !amount_equal(a.overrides[i].threshold, b.overrides[i].threshold))
        return false;
    return true;
  }
  // apiequality.Semantic.DeepEqual on two ThrottleStatus values (empty maps are nil maps)
  static bool same_status(const ThrottleObj& a, const ThrottleObj& b) {
    return amount_equal(a.st_calc, b.st_calc) && a.st_calc_at_set == b.st_calc_at_set && a.st_calc_at == b.st_calc_at && a.st_messages == b.st_messages &&
           a.st_thr_pod == b.st_thr_pod && a.st_thr_req == b.st_thr_req && amount_equal(a.st_used, b.st_used);
  }
  void apply_throttle(const Node& v, int kind) {
    const uint64_t epoch = col_epoch;  // a new resource name or a finer scale re-packs every column
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
    const std::string key = thr_key(kind, o.ns, o.name);
    auto it = thr_index.find(key);
    if (it == thr_index.end()) {
      o.seq = ++thr_seq;
      const bool delta = creation_delta(o, epoch);
      const long at = delta ? place_creation(o) : -1;
      if (delta && at < 0 && kt_move_throttle_columns) {  // rule 4: the columns laid out again by a move, the new one filled
        const size_t t = throttles.size();
        thr_index[key] = (int)t;
        throttles.push_back(std::move(o));
        relayout_pending = true;
        selector_changed(t, true);
        return;
      }
      if (at >= 0) {  // a column delta: a hole filled in place, or a column appended by the next sync
        const size_t t = (size_t)at;
        const bool reserved_any = [&] {
          auto r = cache[o.kind].by_thr.find(o.nn());
          return r != cache[o.kind].by_thr.end() && !r->second.empty();
        }();
        thr_index[key] = (int)t;
        if (t < throttles.size()) {
          free_thr.erase(std::find(free_thr.begin(), free_thr.end(), (int)t));
          throttles[t] = std::move(o);
          thr_reused = true;
          sel_cols.add(t);
          spec_cols.add(t);
          status_cols.add(t);
          reserved_cols.add(t);  // the reservation cache keeps a deleted name's entries: a re-created name gets its totals back
        } else {
          throttles.push_back(std::move(o));
          if (has_status) status_cols.add(t);
          if (reserved_any) reserved_cols.add(t);
        }
        selector_changed(t, true);
        return;
      }
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
      // The same tables (a status echoed back by the informer after reconcile's UpdateStatus, or written by another replica; an
      // edit of the threshold or the overrides): the tables stay; only this column's status and threshold columns are sent
      // again, when they changed, and only the cached verdicts of the pods this throttle affects are void.
      const size_t t = (size_t)it->second;
      const bool tables_kept = epoch == col_epoch && same_tables(old, o), thresholds_kept = same_threshold_columns(old, o),
                 status_kept = same_status(old, o);
      // Other terms or another throttlerName in the same column (same kind and namespace, no label key or value the dictionaries
      // lack): the column is recompiled in place, without a new layout (kt_update_selector_rows).
      const bool selector_in_place = !tables_kept && epoch == col_epoch && old.ns == o.ns && selector_delta() && in_vocabulary(o) &&
                                     (thresholds_kept || kt_update_threshold_rows);
      old = std::move(o);
      if (selector_in_place) {
        sel_cols.add(t);
        selector_changed(t, true);
      }
      if (selector_in_place || (tables_kept && (thresholds_kept || (kt_update_threshold_rows && !throttles_dirty)))) {
        if (!thresholds_kept) {
          spec_cols.add(t);
          throttle_state_changed(t);
        }
        if (!status_kept) {
          status_cols.add(t);
          throttle_state_changed(t);
        }
        return;
      }
    }
    throttles_dirty = status_dirty = reserved_dirty = true;
    broken_valid = false;
  }
  void delete_throttle(int kind, const std::string& ns, const std::string& tname) {
    auto it = thr_index.find(thr_key(kind, ns, tname));
    if (it == thr_index.end()) return;
    // the column can never match or be reconciled again; the next new throttle takes it over
    const size_t t = (size_t)it->second;
    ThrottleObj& o = throttles[t];
    free_thr.push_back(it->second);
    if (o.metrics_pending) { record_metrics(o); o.metrics_pending = false; }  // its series outlive it, as a GaugeVec's do
    o.live = false;
    o.terms.clear();
    // The reservation cache keeps the entry: reserved_resource_amounts.go has no way to drop a throttle, so what was reserved on
    // this name is still counted if a throttle of the same name comes back (until those pods are observed or deleted).
    thr_index.erase(it);
    // The column becomes a hole that matches nothing (no terms, flags 0) until the next whole upload compacts it -- as long as at
    // most half the columns are holes.  That bound is a guess, not a measured break-even: past it every pass walks mostly dead
    // words, and a whole upload lays the columns out again.
    if (selector_delta() && 2 * free_thr.size() <= throttles.size()) {
      sel_cols.add(t);
      selector_changed(t, false);
      return;
    }
    if (selector_delta() && kt_move_throttle_columns && !thr_index.empty()) {  // past half holes: compacted by a move, not a whole upload
      throttle_state_changed(t);
      relayout_pending = true;
      return;
    }
    throttles_dirty = status_dirty = reserved_dirty = true;
    broken_valid = false;
  }
  // Whether a deletion or a selector edit can go as a column delta: the engine has the call and no whole upload is pending.
  bool selector_delta() const { return kt_update_selector_rows && !throttles_dirty; }
  // Whether a creation can go as a column delta: the engine has every call it needs, no whole upload is pending, no resource
  // column or scale changed (epoch), the selectors mention only known label keys and values, and a Throttle's namespace has an
  // id already (one first met here changes the namespace rows and keeps the full path).
  bool creation_delta(const ThrottleObj& o, uint64_t epoch) const {
    return kt_append_throttle_rows && selector_delta() && kt_update_threshold_rows && kt_update_status_rows && kt_update_reserved_rows &&
           epoch == col_epoch && in_vocabulary(o) && (o.kind != KT_KIND_THROTTLE || ns_dict.find(o.ns) >= 0);
  }
  // The column of a creation that goes as a column delta, or -1 (the full path, which lays the columns out again).  A pass costs
  // the words on each namespace's list (reorder_columns), so the new column goes where it adds no word to any list beyond what
  // the creation itself must add.  Its group is its namespace (a Throttle) or its namespace set (a ClusterThrottle,
  // namespace_set_of), as in reorder_columns:
  //   1. a hole in a 32-throttle word that holds a live column of the group;
  //   2. else, when the last word holds a live column of the group and has room, a new column at the end;
  //   3. else, when the group has no live column (every word it gets is one it must add): any hole, else a new column;
  //   4. else -1.
  long place_creation(const ThrottleObj& o) const {
    std::map<std::string, std::string> set_of;  // ClusterThrottle signature -> namespace set, evaluated once each
    auto group = [&](const ThrottleObj& x) -> const std::string& {
      if (x.kind == KT_KIND_THROTTLE) return x.ns;
      const std::string sig = ns_selector_signature(x);
      auto it = set_of.find(sig);
      if (it == set_of.end()) it = set_of.emplace(sig, namespace_set_of(x)).first;
      return it->second;
    };
    const std::string g = group(o);
    const size_t m = throttles.size();
    std::vector<char> holds((m + 31) / 32 + 1, 0);
    bool any = false;
    for (size_t t = 0; t < m; ++t)
      if (throttles[t].live && throttles[t].kind == o.kind && group(throttles[t]) == g) holds[t >> 5] = any = true;
    for (int t : free_thr)
      if (holds[(size_t)t >> 5]) return t;
    if (m % 32 && holds[m >> 5]) return (long)m;
    if (!any) return free_thr.empty() ? (long)m : free_thr.back();
    return -1;
  }
  // Every label key and value the throttle's selectors mention is in the dictionaries already: sync_vocabulary would intern
  // nothing, so no pod or namespace row has to be packed again.
  bool in_vocabulary(const ThrottleObj& o) const {
    auto known = [&](const std::vector<Requirement>& reqs) {
      for (auto& r : reqs) {
        const int kid = labels.keys.find(r.key);
        if (kid < 0) return false;
        for (auto& v : r.values)
          if (labels.vals[(size_t)kid].find(v) < 0) return false;
      }
      return true;
    };
    for (auto& term : o.terms) {
      if (!known(term.pod_sel.reqs)) return false;
      if (o.kind == KT_KIND_CLUSTERTHROTTLE && (!known(term.ns_sel.reqs) || labels.keys.find(kNsExistsKey) < 0)) return false;
    }
    return true;
  }
  // Column t's terms or flags changed in place: the cached verdicts of the pods it affected are void (the cached match rows say
  // which), and after an edit also those of the queued pods in the namespaces the new version can reach.
  void selector_changed(size_t t, bool edit) {
    throttle_state_changed(t);
    broken_valid = false;
    if (!edit || !queue.valid) return;
    const ThrottleObj& o = throttles[t];
    const std::string reach = o.kind == KT_KIND_THROTTLE ? std::string() : namespace_set_of(o);
    for (size_t row = 0; row < pend_pod.size() && row < queue.row_ok.size(); ++row) {
      if (pend_pod[row] < 0) continue;
      const std::string& ns = pods[(size_t)pend_pod[row]].ns;
      bool reached = ns == o.ns;
      if (o.kind != KT_KIND_THROTTLE) {
        const int id = ns_dict.find(ns);
        reached = id >= 0 && (size_t)id < reach.size() && reach[(size_t)id] == '1';
      }
      if (reached) queue.row_ok[row] = 0;
    }
  }

  std::string status_json(const std::string& ns, const std::string& tname) {
    const int t = find_throttle(ns, tname);
    if (t < 0) fail("throttle " + ns + "/" + tname + " not found");
    const ThrottleObj& o = throttles[(size_t)t];
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
    const int t = find_throttle(ns, tname);
    if (t < 0) fail("throttle " + ns + "/" + tname + " not found");
    const ThrottleObj& o = throttles[(size_t)t];
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

template <bool kReadsOnly = false, class F>
const char* guarded(kth_plugin* p, F&& f) {
  if (!p) return ret(err_json("null plugin handle"));
  std::lock_guard<std::mutex> lk(p->mu);
  if (!kReadsOnly) ++p->epoch;  // may change the state or run a pass: kth_affected_pods' last pass no longer answers
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
    else if (k == "Namespace") p->delete_namespace(nm);
    else fail("unsupported kind: " + k);
    return "{\"ok\":true}";
  });
}
const char* kth_apply_events(kth_plugin* p, const char* events_json) {
  return guarded(p, [&]() { return p->apply_events(events_json ? events_json : ""); });
}
const char* kth_reconcile_all(kth_plugin* p, const char* now_rfc3339) {
  return guarded(p, [&]() { return p->reconcile_all(now_rfc3339 ? now_rfc3339 : ""); });
}
const char* kth_reconcile(kth_plugin* p, const char* keys_json, const char* now_rfc3339) {
  return guarded(p, [&]() { return p->reconcile_keys(keys_json ? keys_json : "", now_rfc3339 ? now_rfc3339 : ""); });
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
    p->prefilter_json(w, batch[0], r.row(0));
    return w.out;
  });
}
const char* kth_pre_filter_key(kth_plugin* p, const char* ns, const char* name) {
  return guarded(p, [&]() { return p->pre_filter_key(ns ? ns : "", name ? name : ""); });
}
const char* kth_pre_filter_keys(kth_plugin* p, const char* keys_json) {
  return guarded(p, [&]() { return p->pre_filter_keys(keys_json ? keys_json : ""); });
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
  ++p->epoch;
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
    for (size_t i = 0; i < batch.size(); ++i) p->prefilter_json(w, batch[i], r.row(i));
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
const char* kth_affected_pods(kth_plugin* p, const char* ns, const char* name) {
  return guarded<true>(p, [&]() { return p->affected_pods(ns ? ns : "", name ? name : ""); });
}
const char* kth_queue_report(kth_plugin* p) {
  return guarded<true>(p, [&]() { return p->queue_report(); });
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
