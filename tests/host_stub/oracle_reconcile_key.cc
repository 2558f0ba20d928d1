// The object-level oracle's C API (oracle/ko_capi.cc, compiled in unchanged) plus ko_world_reconcile_key: the oracle World's own
// per-throttle World::reconcile(thr, now) -- the reference's reconcile(key) -- for one Throttle (kind 0) or ClusterThrottle
// (kind 1).  Built by tests/test_reconcile_keys.py into its own library so that kth_reconcile can be compared key by key with
// it.  Returns {"found": bool, "responsible": bool, "err": reconcile's error text or "", "statusChanged": bool}.
#include "../../oracle/ko_capi.cc"

extern "C" const char* ko_world_reconcile_key(void* h, int kind, const char* ns, const char* name, const char* now_rfc3339) {
  try {
    KoWorld* k = (KoWorld*)h;
    Time now;
    const std::string e = ParseRFC3339(now_rfc3339, &now);
    if (!e.empty()) return ret(err_obj(e));
    Throttle* t = nullptr;
    if (kind == 1) {
      auto it = k->w.clthrIndex.find(name);
      if (it != k->w.clthrIndex.end()) t = k->w.clusterThrottles[it->second].get();
    } else {
      auto it = k->w.thrIndex.find(std::string(ns) + "/" + name);
      if (it != k->w.thrIndex.end()) t = k->w.throttles[it->second].get();
    }
    Value o = Value::object();
    o.set("found", Value::boolean(t != nullptr));
    o.set("responsible", Value::boolean(t && k->w.isResponsibleFor(*t)));
    bool changed = false;
    std::string err;
    if (t && k->w.isResponsibleFor(*t)) err = k->w.reconcile(*t, now, &changed);
    o.set("err", Value::str(err));
    o.set("statusChanged", Value::boolean(changed));
    return ret(o);
  } catch (const std::exception& ex) {
    return ret(err_obj(ex.what()));
  }
}
