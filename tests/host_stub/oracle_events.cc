// The object-level oracle's C API (oracle/ko_capi.cc, compiled in unchanged, with ko_world_reconcile_key of
// oracle_reconcile_key.cc) plus ko_world_event: one informer watch event ({"type": "ADDED" | "MODIFIED" | "DELETED", "object":
// manifest}) applied to the oracle World, returning the reconcile keys the reference's handlers enqueue at that moment
// (throttle_controller.go:401-531, clusterthrottle_controller.go:429-563), from World::affectedThrottles /
// affectedClusterThrottles with their error returns.  Built by tests/test_apply_events.py so that kth_apply_events can be
// compared event by event with it.  Returns {"keys": [...]} (unordered, without duplicates).
#include <set>

#include "oracle_reconcile_key.cc"

namespace {

// the affected throttles of the versions one handler looks at, per controller: none from a controller that fails on one of them
void affected_keys(const World& w, const std::vector<const Pod*>& vers, std::set<std::string>* keys) {
  for (int kind = 0; kind < 2; ++kind) {
    std::set<std::string> mine;
    bool failed = false;
    for (const Pod* p : vers) {
      std::vector<Throttle*> thrs;
      const std::string e = kind == 0 ? w.affectedThrottles(*p, &thrs) : w.affectedClusterThrottles(*p, &thrs);
      if (!e.empty()) { failed = true; break; }
      for (Throttle* t : thrs) mine.insert(t->NN());
    }
    if (!failed) keys->insert(mine.begin(), mine.end());
  }
}

}  // namespace

extern "C" const char* ko_world_event(void* h, const char* event_json) {
  try {
    World& w = ((KoWorld*)h)->w;
    Value ev = kojson::parse(event_json);
    const std::string type = ev.get("type").str_or("");
    const Value& obj = ev.get("object");
    const std::string kind = obj.get("kind").str_or("");
    const std::string ns = obj.get("metadata").get("namespace").str_or(""), name = obj.get("metadata").get("name").str_or("");
    std::set<std::string> keys;
    if (kind == "Pod") {
      auto it = w.podIndex.find(ns + "/" + name);
      const bool held = it != w.podIndex.end();
      const Pod old = held ? *w.pods[it->second] : Pod();
      if (type == "DELETED") {
        if (held && w.shouldCountIn(old)) affected_keys(w, {&old}, &keys);  // DeleteFunc
        w.deletePod(ns, name);
      } else {
        Pod p = pod_from(obj);
        if (!held) {
          if (w.shouldCountIn(p)) affected_keys(w, {&p}, &keys);  // AddFunc
        } else if (w.shouldCountIn(old) || w.shouldCountIn(p)) {
          affected_keys(w, {&old, &p}, &keys);  // UpdateFunc
        }
        w.applyPod(std::move(p));
      }
    } else if (kind == "Throttle" || kind == "ClusterThrottle") {
      const bool cluster = kind == "ClusterThrottle";
      if (type == "DELETED") {
        const Throttle* t = nullptr;
        if (cluster) {
          auto it = w.clthrIndex.find(name);
          if (it != w.clthrIndex.end()) t = w.clusterThrottles[it->second].get();
        } else {
          auto it = w.thrIndex.find(ns + "/" + name);
          if (it != w.thrIndex.end()) t = w.throttles[it->second].get();
        }
        if (t && w.isResponsibleFor(*t)) keys.insert(t->NN());
        w.deleteThrottle(cluster, ns, name);
      } else {
        Throttle t = throttle_from(obj);
        if (w.isResponsibleFor(t)) keys.insert(t.NN());
        w.upsertThrottle(std::move(t), !obj.get("status").is_obj());
      }
    } else if (kind == "Namespace") {
      if (type == "DELETED") w.deleteNamespace(name);
      else w.upsertNamespace(ns_from(obj));
    } else {
      return ret(err_obj("unknown kind: " + kind));
    }
    Value out = Value::object();
    Value arr = Value::array();
    for (auto& k : keys) arr.push(Value::str(k));
    out.set("keys", arr);
    return ret(out);
  } catch (const std::exception& e) {
    return ret(err_obj(e.what()));
  }
}
