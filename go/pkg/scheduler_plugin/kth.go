// NOT COMPILED IN THIS REPOSITORY'S ENVIRONMENT (no Go toolchain in the image; see go/README.md).
//
// cgo shim over include/kt_host.h: one Go method per kth_* entry point, nothing else.  Strings returned by the library
// live in a thread-local buffer that the next call FROM THE SAME OS THREAD overwrites; a goroutine can migrate between
// the C call and C.GoString only if it is descheduled in between, so every call pins its OS thread for that window.

package scheduler_plugin

/*
#cgo CFLAGS: -I${SRCDIR}/../../../include
#cgo LDFLAGS: -L${SRCDIR}/../../../kube_throttler_b200 -lkt_b200 -Wl,-rpath,${SRCDIR}/../../../kube_throttler_b200
#include <stdlib.h>
#include "kt_host.h"
*/
import "C"

import (
	"encoding/json"
	"fmt"
	"runtime"
	"unsafe"
)

// engine is the handle behind NewPlugin: packer, reservation cache, status bookkeeping and the device pass.
type engine struct{ h *C.kth_plugin }

type kthError struct {
	Error string `json:"error"`
}

func newEngine(args *KubeThrottlerPluginArgs, device int) (*engine, error) {
	js, err := json.Marshal(args) // the library reads the same (misspelt) tags
	if err != nil {
		return nil, err
	}
	cs := C.CString(string(js))
	defer C.free(unsafe.Pointer(cs))
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	var h *C.kth_plugin
	if rc := C.kth_new_plugin(&h, cs, C.int(device)); rc != 0 {
		return nil, fmt.Errorf("kth_new_plugin: %s (kt_status %d; there is no CPU fallback)", C.GoString(C.kth_new_plugin_error()), int(rc))
	}
	return &engine{h}, nil
}

func (e *engine) close() { C.kth_free(e.h) }

// call runs one kth_* function that takes a JSON document and returns one; out may be nil.
func (e *engine) call(fn func(*C.char) *C.char, in interface{}, out interface{}) error {
	js, err := json.Marshal(in)
	if err != nil {
		return err
	}
	cs := C.CString(string(js))
	defer C.free(unsafe.Pointer(cs))
	runtime.LockOSThread()
	raw := C.GoString(fn(cs))
	runtime.UnlockOSThread()
	return decode(raw, out)
}

func decode(raw string, out interface{}) error {
	var ke kthError
	if len(raw) > 9 && raw[:9] == `{"error":` && json.Unmarshal([]byte(raw), &ke) == nil && ke.Error != "" {
		return fmt.Errorf("%s", ke.Error)
	}
	if out == nil {
		return nil
	}
	return json.Unmarshal([]byte(raw), out)
}

// informer events
func (e *engine) apply(obj interface{}) error {
	return e.call(func(p *C.char) *C.char { return C.kth_apply(e.h, p) }, obj, nil)
}

func (e *engine) delete(kind, ns, name string) error {
	ck, cn, cm := C.CString(kind), C.CString(ns), C.CString(name)
	defer C.free(unsafe.Pointer(ck))
	defer C.free(unsafe.Pointer(cn))
	defer C.free(unsafe.Pointer(cm))
	runtime.LockOSThread()
	raw := C.GoString(C.kth_delete(e.h, ck, cn, cm))
	runtime.UnlockOSThread()
	return decode(raw, nil)
}

// reconcileResult is what kth_reconcile_all reports: which statuses changed and when to come back for an override boundary.
type reconcileResult struct {
	Reconciled        int              `json:"reconciled"`
	Changed           []string         `json:"changed"`           // "ns/name" (Throttle) or "/name" (ClusterThrottle)
	RequeueAfterNanos map[string]int64 `json:"requeueAfterNanos"` // NextOverrideHappensIn, throttle_types.go:37-63
}

func (e *engine) reconcileAll(nowRFC3339 string) (*reconcileResult, error) {
	cs := C.CString(nowRFC3339)
	defer C.free(unsafe.Pointer(cs))
	runtime.LockOSThread()
	raw := C.GoString(C.kth_reconcile_all(e.h, cs))
	runtime.UnlockOSThread()
	var r reconcileResult
	if err := decode(raw, &r); err != nil {
		return nil, err
	}
	return &r, nil
}

// reconcileKeysResult is what kth_reconcile reports for the listed keys; keys of other throttlers are skipped.
type reconcileKeysResult struct {
	reconcileResult
	Errors   map[string]string `json:"errors"`   // key -> reconcile's error (malformed key, reachable broken podSelector)
	NotFound []string          `json:"notFound"` // unknown or deleted: the lister's NotFound, reconcile returns nil
}

// reconcileKeys is reconcile(key) for the listed keys only ("ns/name" for a Throttle, "/name" for a ClusterThrottle), in one
// device call over the listed throttles and the namespaces they reach.
func (e *engine) reconcileKeys(keys []string, nowRFC3339 string) (*reconcileKeysResult, error) {
	js, err := json.Marshal(keys)
	if err != nil {
		return nil, err
	}
	ck, cs := C.CString(string(js)), C.CString(nowRFC3339)
	defer C.free(unsafe.Pointer(ck))
	defer C.free(unsafe.Pointer(cs))
	runtime.LockOSThread()
	raw := C.GoString(C.kth_reconcile(e.h, ck, cs))
	runtime.UnlockOSThread()
	var r reconcileKeysResult
	if err := decode(raw, &r); err != nil {
		return nil, err
	}
	return &r, nil
}

// watchEvent is one informer event as kth_apply_events takes it: Type is "ADDED", "MODIFIED" or "DELETED".
type watchEvent struct {
	Type   string      `json:"type"`
	Object interface{} `json:"object"`
}

// applyEventsEntry is what kth_apply / kth_delete report for one event, plus the keys its handlers enqueue.
type applyEventsEntry struct {
	OK      bool     `json:"ok"`
	Warning string   `json:"warning"`
	Error   string   `json:"error"`
	Enqueue []string `json:"enqueue"`
}

type applyEventsResult struct {
	Results []applyEventsEntry `json:"results"`
	Enqueue []string           `json:"enqueue"` // the union of the entries' keys, first appearance first
}

// applyEvents applies a batch of informer events in order and returns, per event, the reconcile keys the reference's handlers
// enqueue ("ns/name" for a Throttle, "/name" for a ClusterThrottle), for reconcileKeys.  The pod events between two table events
// take one device call.
func (e *engine) applyEvents(events []watchEvent) (*applyEventsResult, error) {
	var r applyEventsResult
	if err := e.call(func(p *C.char) *C.char { return C.kth_apply_events(e.h, p) }, events, &r); err != nil {
		return nil, err
	}
	return &r, nil
}

// statusManifest is the `status` subresource as encoding/json would render v1alpha1.ThrottleStatus.
func (e *engine) statusManifest(ns, name string) ([]byte, error) {
	cn, cm := C.CString(ns), C.CString(name)
	defer C.free(unsafe.Pointer(cn))
	defer C.free(unsafe.Pointer(cm))
	runtime.LockOSThread()
	raw := C.GoString(C.kth_get_status_manifest(e.h, cn, cm))
	runtime.UnlockOSThread()
	if err := decode(raw, nil); err != nil {
		return nil, err
	}
	return []byte(raw), nil
}

// preFilterResult mirrors kth_pre_filter's answer: the framework code, the reasons in the reference's fixed order and,
// when some throttle's threshold is below the pod's own requests, the Warning event to record.
type preFilterResult struct {
	Code    string   `json:"code"` // Success | UnschedulableAndUnresolvable | Error
	Reasons []string `json:"reasons"`
	Event   *struct {
		Type    string `json:"type"`
		Reason  string `json:"reason"`
		Message string `json:"message"`
	} `json:"event"`
}

func (e *engine) preFilter(pod interface{}) (*preFilterResult, error) {
	var r preFilterResult
	err := e.call(func(p *C.char) *C.char { return C.kth_pre_filter(e.h, p) }, pod, &r)
	return &r, err
}

// preFilterKeysEntry is one entry of kth_pre_filter_keys: a PreFilter result, or Error for an unknown pod or a malformed key.
type preFilterKeysEntry struct {
	preFilterResult
	Error string `json:"error"`
}

// preFilterKeys is PreFilter by key for pods the informer already delivered ("namespace/name"), one entry per key in order, in
// one device call over the listed rows only.
func (e *engine) preFilterKeys(keys []string) ([]preFilterKeysEntry, error) {
	var r []preFilterKeysEntry
	err := e.call(func(p *C.char) *C.char { return C.kth_pre_filter_keys(e.h, p) }, keys, &r)
	return r, err
}

// queueReportThrottle is one throttle's entry of kth_queue_report.
type queueReportThrottle struct {
	Key                         string          `json:"key"`
	Kind                        string          `json:"kind"`
	Active                      int64           `json:"active"`
	Insufficient                int64           `json:"insufficient"`
	PodRequestsExceedsThreshold int64           `json:"podRequestsExceedsThreshold"`
	OnlyBlocker                 int64           `json:"onlyBlocker"`
	HeldBack                    json.RawMessage `json:"heldBack"`
}

// queueReport is kth_queue_report: the verdict counts of the scheduling queue and, for every throttle of this plugin, the queued
// pods it holds back by status, the ones it alone blocks and their ResourceAmount sum -- one device call, not one affectedPods
// call per throttle.
type queueReport struct {
	Queued        int64                 `json:"queued"`
	Success       int64                 `json:"success"`
	Unschedulable int64                 `json:"unschedulable"`
	Error         int64                 `json:"error"`
	Throttles     []queueReportThrottle `json:"throttles"`
}

func (e *engine) queueReport() (*queueReport, error) {
	var r queueReport
	runtime.LockOSThread()
	raw := C.GoString(C.kth_queue_report(e.h))
	runtime.UnlockOSThread()
	return &r, decode(raw, &r)
}

type reserveResult struct {
	Code    string   `json:"code"`
	Reasons []string `json:"reasons"`
}

func (e *engine) reserve(pod interface{}) (*reserveResult, error) {
	var r reserveResult
	err := e.call(func(p *C.char) *C.char { return C.kth_reserve(e.h, p) }, pod, &r)
	return &r, err
}

func (e *engine) unreserve(pod interface{}) error {
	return e.call(func(p *C.char) *C.char { return C.kth_unreserve(e.h, p) }, pod, nil)
}

func (e *engine) metricsText() string {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	return C.GoString(C.kth_metrics(e.h))
}
