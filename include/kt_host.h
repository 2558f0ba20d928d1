/*
 * kt_host.h -- host side of the drop-in boundary: the kube-scheduler plugin surface of
 * everpeace/kube-throttler (pkg/scheduler_plugin/plugin.go) restated above the device engine of
 * kt_b200.h, plus the packer that turns Kubernetes objects into the engine's int64 columns.
 *
 * The reference plugin is Go; no Go toolchain exists in this image (DESIGN.md "Host language"), so the
 * host layer is C++ behind this C ABI.  A Go build keeps pkg/scheduler_plugin/plugin.go's exported
 * surface (NewPlugin / PreFilter / Reserve / Unreserve) and forwards each call to the kth_* function
 * named beside it below (cgo stub in INTEGRATION.md); informer events become kth_apply / kth_delete.
 *
 * Objects cross the boundary as Kubernetes JSON manifests (the wire format the informers already hold);
 * results come back as JSON.  Returned strings are owned by the plugin handle and stay valid until the
 * next call on the same handle FROM THE SAME THREAD (thread-local buffer).  All functions are
 * re-entrant; a handle serialises its calls with one mutex (PreFilter/Reserve run on the scheduling
 * goroutine, Unreserve and the informer handlers on others: plugin.go:217-257, throttle_controller.go:400-536).
 *
 * What runs where:
 *   host (this layer)  PodRequestResourceList / ResourceAmountOfPod once per pod event (resourcelist.go:27-46,
 *                      resource_amount.go:71-76), resource.Quantity parsing and per-column scaling, label /
 *                      namespace / resource dictionaries, LabelSelectorAsSelector validation, RFC3339 override
 *                      windows, the reservation cache (reserved_resource_amounts.go), status bookkeeping
 *                      (throttle_controller.go:120-133, Q6), PreFilter reason strings (plugin.go:177-214)
 *   device (kt_b200.h) every pod x throttle selector match, the per-throttle used sums, CalculateThreshold
 *                      at `now`, IsThrottled, the 4-step CheckThrottledFor and the admit bit
 * There is no CPU evaluation path here either: without a GPU kth_new_plugin fails.
 */
#ifndef KT_HOST_H_
#define KT_HOST_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct kth_plugin kth_plugin;

/* NewPlugin(configuration, handle) -- plugin.go:63-146.  args_json is the pluginConfig args object
 * (plugin_args.go:33-40): {"name": "...", "targetSchedulerName": "...", "kubeconfig": "...",
 * "reconcileTemporaryThresholdInterval": "15s", "controllerThrediness": N, "numKeyMutex": N}
 * -- the misspelt JSON tags are the reference's.  name and targetSchedulerName are required
 * (DecodePluginArgs, plugin_args.go:42-60).  Returns 0 or a negative kt_status; *out is NULL on failure
 * and kth_new_plugin_error() describes it. */
int kth_new_plugin(kth_plugin** out, const char* args_json, int device);
const char* kth_new_plugin_error(void);
void kth_free(kth_plugin* p);

/* Informer events (pod / namespace / throttle / clusterthrottle informers, plugin.go:77-112):
 * Add and Update are kth_apply(manifest), Delete is kth_delete.  kind is "Pod", "Namespace", "Throttle"
 * or "ClusterThrottle".  Pod updates move reservations between throttles when the pod's labels changed
 * (throttle_controller.go:469-500), pod deletes un-reserve (:509-515).  Returns {"ok":true} or {"error":...}. */
const char* kth_apply(kth_plugin* p, const char* manifest_json);
const char* kth_delete(kth_plugin* p, const char* kind, const char* ns, const char* name);

/* A batch of informer watch events, applied in order, with the reconcile keys the reference's handlers enqueue for each
 * (throttle_controller.go:401-531, clusterthrottle_controller.go:429-563).  events_json is a JSON array of
 * {"type": "ADDED" | "MODIFIED" | "DELETED", "object": manifest}: ADDED and MODIFIED are kth_apply(object), DELETED is
 * kth_delete(object.kind, object.metadata.namespace, object.metadata.name).  Returns
 *   {"results": [one entry per event, in order], "enqueue": [the union of the entries' keys, first appearance first]}
 * where an entry is what kth_apply / kth_delete return for the event plus "enqueue": [keys] on success.  Keys are spelled as
 * kth_reconcile takes them ("namespace/name" a Throttle, "/name" a ClusterThrottle), each entry's in creation order:
 *   Throttle / ClusterThrottle applied   its own key when the NEW object's throttlerName is this plugin's
 *   Throttle / ClusterThrottle deleted   its own key when the plugin held it and it was this plugin's
 *   Pod applied, not held before         if shouldCountIn(new): the throttles the new version affects
 *   Pod applied, held before             if shouldCountIn(old) || shouldCountIn(new): those of the held copy and of the new one
 *   Pod deleted                          if shouldCountIn(old): those of the held copy
 *   Namespace applied / deleted          nothing
 * per controller: a controller whose affectedThrottles fails for one of those versions (a reachable broken podSelector; for
 * ClusterThrottles also an unknown namespace) adds no key for the event, the other one's keys stand.
 * The pod events between two Throttle / ClusterThrottle / Namespace events form a run: the distinct (namespace, label set)
 * versions of a run take ONE kt_match_pods call and no pass over the scheduling queue; runs of pods that are not counted take
 * no device call at all.  Afterwards the plugin is in the state kth_apply / kth_delete event by event would leave (statuses,
 * reservations, PreFilter verdicts, affected pods, metrics, what a following reconcile returns); kth_queue_stats' passes and
 * hits may differ.  An event those calls refuse -- and a malformed event (not an object, unknown type, no object) -- is an
 * {"error": ...} entry, and the batch goes on.  When a run's device call fails, its events report what the single calls
 * report when their pass fails ({"ok":true,"warning":"pod updated; reservation move skipped: ..."}; a deleted pod leaves every
 * reservation and is an {"error": ...}; an event that only needed its keys is {"ok":true,"warning":...}), without "enqueue". */
const char* kth_apply_events(kth_plugin* p, const char* events_json);

/* reconcile(key) for EVERY responsible Throttle and ClusterThrottle in one device pass
 * (throttle_controller.go:84-211, clusterthrottle_controller.go:87-214): status.used,
 * status.calculatedThreshold (replaced only when threshold or messages changed, Q6), status.throttled
 * (onEqual = true), observed pods un-reserved.  now_rfc3339 is the controller clock.
 * Returns {"reconciled":N,"changed":[...names of throttles whose status changed...],
 *          "requeueAfterNanos":{name: ns until the next temporaryThresholdOverride boundary}} -- the latter is
 * NextOverrideHappensIn (throttle_types.go:37-63), what the reference passes to enqueueAfter (:201-208). */
const char* kth_reconcile_all(kth_plugin* p, const char* now_rfc3339);

/* reconcile(key) for the listed keys only (throttle_controller.go:84-211, clusterthrottle_controller.go:87-214): the reference's
 * controllers reconcile one workqueue key at a time, at the cost of the pods of the namespaces the throttle reaches.  keys_json
 * is a JSON array of names as kth_reconcile_all spells them under "changed": "namespace/name" for a Throttle, "/name" for a
 * ClusterThrottle.  Each distinct key, in the order given, gets exactly what kth_reconcile_all does for that throttle (status
 * under Q6 and Semantic.DeepEqual, cached verdicts, gauges, NextOverrideHappensIn, unreserveAffectedPods with Q8, or the
 * reachable broken-podSelector error that leaves the status and the reservations alone), from ONE device call over the listed
 * throttles' columns and the rows of the namespaces they reach (kt_reconcile_throttles).  Throttles that are not listed keep
 * their status, reservations and gauges.  Returns
 *   {"reconciled":n,"changed":[...],"requeueAfterNanos":{...},"errors":{key: text},"notFound":[...]}
 * an unknown or deleted key is in "notFound" (the lister's NotFound makes reconcile return nil, :95-101), a key of another
 * throttler is skipped, a malformed key is an entry of "errors". */
const char* kth_reconcile(kth_plugin* p, const char* keys_json, const char* now_rfc3339);

/* status of one Throttle (ns != "") or ClusterThrottle (ns == ""):
 * {"calculatedThreshold":{"threshold":{...},"calculatedAtSet":bool,"calculatedAtUnix":sec,"messages":[..]},
 *  "throttled":{"resourceCounts":{"pod":bool},"resourceRequests":{name:bool}},
 *  "used":{"resourceCounts":{"pod":n},"resourceRequests":{name:"decimal"}}} */
const char* kth_get_status(kth_plugin* p, const char* ns, const char* name);

/* The same status as the `status` subresource the reference's UpdateStatus sends (throttle_controller.go:157-173):
 * encoding/json of v1alpha1.ThrottleStatus -- fields in declaration order, map keys sorted, nil / empty members omitted,
 * quantities in their canonical spelling (resource.Quantity.String: "500m", "1", "512Mi"; util_throttle_test.go:169-177 asserts
 * them), calculatedAt as RFC3339 UTC or null.  What the Go build hands to
 * ScheduleV1alpha1().Throttles(ns).UpdateStatus for every name kth_reconcile_all lists under "changed". */
const char* kth_get_status_manifest(kth_plugin* p, const char* ns, const char* name);

/* PreFilter(ctx, state, pod) -- plugin.go:148-215.
 * {"code":"Success"|"UnschedulableAndUnresolvable"|"Error","reasons":[...],"event":{...}?,
 *  "throttle":{"active":[..],"insufficient":[..],"podRequestsExceedsThreshold":[..],"affected":[..]},
 *  "clusterthrottle":{...}}                       reasons are in the reference's fixed order (Q10).
 * Cost: after the state sync every entry point does, ONE device call (kt_check_pods) that evaluates the words of the pod's own
 * namespace -- it grows with the throttles that namespace can reach, not with the length of the resident scheduling queue; no
 * pod row is uploaded and no pass runs.  (Linked against an engine without kt_check_pods, the pod takes a scratch row behind
 * the queue and one pass over both.) */
const char* kth_pre_filter(kth_plugin* p, const char* pod_json);
/* The same for a whole scheduling queue in ONE device call: pods_json is a JSON array of pods, the
 * result a JSON array of PreFilter results (each pod checked against the same snapshot, independently). */
const char* kth_pre_filter_batch(kth_plugin* p, const char* pods_json);

/* ---- the scheduling queue, resident on the device -------------------------------------------------------------------
 * Pods the pod informer delivered (kth_apply) that are this scheduler's to place -- spec.schedulerName == targetSchedulerName,
 * no spec.nodeName yet, not finished -- are kept packed in the device's pending table as well, row by row, like the running
 * pods.  PreFilter / Reserve / Unreserve for such a pod can then be addressed BY KEY: no manifest crosses the boundary, nothing
 * is parsed, packed or uploaded per call.  ONE device pass answers for the whole queue; its verdicts are cached on the host and
 * stay good per pod until something that pod's verdict depends on changes (its own row, any throttle / namespace object, the
 * status or the reservations of a throttle IT is affected by).  In the scheduler's PreFilter -> Reserve -> next pod cycle a
 * PreFilter therefore only costs a device pass when the pod shares a throttle with what was just reserved.
 * Results have the shape of kth_pre_filter / kth_reserve.  A pod the informer holds that is not queued (already bound, other
 * scheduler) is checked like a manifest; an unknown key is an {"error": ...}. */
const char* kth_pre_filter_key(kth_plugin* p, const char* ns, const char* name);
const char* kth_reserve_key(kth_plugin* p, const char* ns, const char* name);
const char* kth_unreserve_key(kth_plugin* p, const char* ns, const char* name);
/* PreFilter by key for a list of pods, checked on the device row by row (kt_check_pending_rows): the cost follows the listed
 * pods' own namespaces, not the length of the queue.  keys_json is a JSON array of "namespace/name" strings; the result is a
 * JSON array with one entry per key, in the order given:
 *   a queued pod                      exactly what kth_pre_filter_key returns at this moment (reasons in Q10 order, event,
 *                                     affected lists, controller errors);
 *   a pod the informer holds, not queued   the same, checked in a scratch row of the same call;
 *   an unknown pod / a malformed key  {"error": ...}.
 * All listed pods take one device call after the state sync every entry point does.  The cached queue verdicts are neither
 * consulted nor refreshed (kth_queue_stats' passes and hits stay as they are); nothing is reserved and no status written. */
const char* kth_pre_filter_keys(kth_plugin* p, const char* keys_json);
/* PreFilter of EVERY queued pod in (at most) one device pass, no JSON: verdicts[row] = 0 free row, 1 Success,
 * 2 UnschedulableAndUnresolvable, 3 Error, for rows [0, min(cap, rows)); returns the number of queue rows (or -1, see
 * kth_last_error).  kth_queue_row gives the row of a queued pod (-1: not queued); rows are stable while the pod stays queued. */
int64_t kth_pre_filter_queue(kth_plugin* p, uint8_t* verdicts, int64_t cap);
int64_t kth_queue_row(kth_plugin* p, const char* ns, const char* name);
/* Row of a pod in the device's running-pod table (-1: unknown pod).  Diagnostic: rows are handed out from per-namespace arenas
 * of 32 consecutive rows, so that the 32 rows a warp walks share a namespace under any churn. */
int64_t kth_pod_row(kth_plugin* p, const char* ns, const char* name);
const char* kth_last_error(void);
/* {"queued":n,"rows":r,"passes":device passes over the queue so far,"hits":by-key calls answered from cached verdicts,
 *  "throttleColumns":device columns the throttles occupy (deleted throttles' columns are reused),"liveThrottles":m,
 *  "labelKeys":k,"labelValues":v (the label dictionaries: what the selectors mention),"resourceColumns":c,
 *  "wordsPerNamespaceX100":32-throttle words a namespace's pods visit, x100}.  A deletion or selector edit applied as a column
 * delta keeps its column until the next whole upload: passes, hits, throttleColumns and wordsPerNamespaceX100 may differ from a
 * plugin that uploads every change whole (they reflect the last whole upload, holes included); every other result is the same. */
const char* kth_queue_stats(kth_plugin* p);

/* Queue-ordered admission: PreFilter and, on Success, Reserve for every pod of a SORTED scheduling queue, with exactly
 * the results the scheduler gets admitting them one per cycle (each admitted pod raises the reservations the next one is
 * checked against, plugin.go:148-238) -- but in as few device passes as the conflicts between the pods allow: a pass
 * decides every undecided pod none of whose affected throttles was reserved on earlier in the same pass.
 * {"rounds":k,"admitted":n,"results":[{"pod":"ns/name","round":i,"preFilter":{...as kth_pre_filter...}}...]} in queue order;
 * the admitted pods stay reserved (kth_unreserve / a reconcile that observes them bound releases them).  Each round of the
 * host-orchestrated form is one kt_check_pods call over the round's undecided pods. */
const char* kth_admit_queue(kth_plugin* p, const char* pods_json);

/* Reserve / Unreserve -- plugin.go:217-257: {"code":"Success"} or {"code":"Error","reasons":[...]}.  The pod's affected
 * throttles come from one kt_check_pods call, as for kth_pre_filter: the cost follows the pod's namespace, not the queue. */
const char* kth_reserve(kth_plugin* p, const char* pod_json);
const char* kth_unreserve(kth_plugin* p, const char* pod_json);
/* reservedResourceAmount(nn) of one controller's cache (kind 0 = Throttle, 1 = ClusterThrottle):
 * {"amount":{...},"pods":["ns/name",...]} -- reserved_resource_amounts.go:113-126. */
const char* kth_reserved(kth_plugin* p, int kind, const char* throttle_nn);

/* affectedPods(thr) of one Throttle (ns != "") or ClusterThrottle (ns == ""), read from the device's match relations
 * (throttle_controller.go:221-246, clusterthrottle_controller.go:224-270), plus the queued pods the throttle holds back:
 * {"pods":["ns/name",...],"terminatedPods":[...],"queued":[{"pod":"ns/name","status":"active"},...]}
 *   pods            affectedNonTerminatedPods: counted (shouldCountIn), matching, not finished -- exactly what the next
 *                   reconcile sums into status.used
 *   terminatedPods  EVERY matching counted pod that has finished.  A listing, not reconcile's slice: the reference's Throttle
 *                   controller keeps only the last of them (Q8, DESIGN.md section 5), which stays reproduced in reconcile's
 *                   un-reservation and is not copied here
 *   queued          the pods of the resident scheduling queue whose affected throttles include this one, with the
 *                   CheckThrottleStatus that PreFilter by key would give now (informer status + reservations,
 *                   isThrottledOnEqual = false): "not-throttled", "active", "insufficient", "pod-requests-exceeds-threshold"
 * Every list is sorted by namespace, then name (the reference's lister order is unspecified).  Pods of namespaces the lister
 * does not hold never appear for a ClusterThrottle.  {"error": ...} for an unknown throttle, a throttle whose throttlerName is
 * not this plugin's, and a podSelector conversion error that some counted pod reaches (the text affectedPods returns; the first
 * such pod in informer order names it).  No side effects: no status is written, no gauge recorded, nothing un-reserved, and
 * every other call answers as it would have; a device pass runs only when the state changed since the last one this call ran. */
const char* kth_affected_pods(kth_plugin* p, const char* ns, const char* name);

/* The scheduling queue per throttle -- which throttles hold the queue back, how many pods and how much they ask for -- in one
 * call instead of one kth_affected_pods per throttle:
 * {"queued":n,"success":n,"unschedulable":n,"error":n,
 *  "throttles":[{"key":"ns/name" | "/name","kind":"Throttle" | "ClusterThrottle","active":n,"insufficient":n,
 *                "podRequestsExceedsThreshold":n,"onlyBlocker":n,"heldBack":{...}},...]}
 *   queued, success, unschedulable, error   the counts of kth_pre_filter_queue's verdicts 1-3 (queued is their sum)
 *   throttles       every live throttle whose throttlerName is this plugin's, in creation order, keyed as kth_reconcile takes them
 *   active, insufficient, podRequestsExceedsThreshold   the counts of kth_affected_pods(t).queued by status
 *   heldBack        the ResourceAmountOfPod sum of the queued pods whose status there is not "not-throttled", spelled as
 *                   kth_get_status's "used"; {} with no such pod
 *   onlyBlocker     the queued pods whose kth_pre_filter_key is UnschedulableAndUnresolvable with one reason naming t alone
 * No side effects: nothing is reserved, no status written, no gauge recorded (kth_queue_stats' passes and hits may change).  At
 * most one device pass over the pending table -- none when the cached queue verdicts are current and the device still holds
 * the codes of a pass at this state -- then one kt_get_check_summary. */
const char* kth_queue_report(kth_plugin* p);

/* The controllers' Prometheus gauges in text exposition format (throttle_metrics.go:27-131,
 * clusterthrottle_metrics.go:27-131, metrics_recorder.go:25-67): throttle_* families labelled {name,namespace,resource,uid},
 * clusterthrottle_* families labelled {name,resource,uid}; spec threshold / status.throttled / status.used /
 * status.calculatedThreshold, counts as the pod count (0 when nil), cpu as MilliValue, other resources as Value.  Series are
 * recorded when kth_reconcile_all handles a throttle and, like a GaugeVec's, are never dropped.  What the Go build would
 * feed legacyregistry with (or serve next to it). */
const char* kth_metrics(kth_plugin* p);

/* Host-only helpers of the packer, exposed so that they can be pinned against the reference's unit
 * tests without a GPU: {"fn":"ParseQuantity","value":..} | {"fn":"PodRequestResourceList","pod":{..}} |
 * {"fn":"ResourceAmountOfPod","pod":{..}} | {"fn":"ParseRFC3339","value":..} |
 * {"fn":"OverrideMessages","throttle":{..}} | {"fn":"NextOverrideHappensIn","throttle":{..},"now":..} | {"fn":"ValidateSelector","selector":{..}} |
 * {"fn":"CanonicalQuantity","value":..} | {"fn":"ThrottleMetrics","throttle":{..spec+status..}} | {"fn":"ScaledValue","value":..,"scale":n} |
 * {"fn":"FormatFloat","value":..}.  Never touches a device. */
const char* kth_eval(const char* request_json);

#ifdef __cplusplus
}
#endif
#endif /* KT_HOST_H_ */
