// NOT COMPILED IN THIS REPOSITORY'S ENVIRONMENT (no Go toolchain in the image; see go/README.md).
//
// The kube-scheduler plugin of kube-throttler with its admission hot path on an H100.  Exported surface, plugin name,
// framework statuses, reason strings and events are the reference's (everpeace/kube-throttler pkg/scheduler_plugin/plugin.go:45-279);
// what differs is behind it: instead of two Go controllers that walk listers per pod and per throttle
// (pkg/controllers), informer events are forwarded to the engine behind include/kt_host.h, which keeps the pod /
// throttle / namespace snapshot packed in HBM and answers PreFilter, Reserve and the reconcile of EVERY throttle with
// batched device passes.  Drop-in: `app.WithPlugin(kubethrottler.PluginName, kubethrottler.NewPlugin)` is unchanged.

package scheduler_plugin

import (
	"context"
	"fmt"
	"strings"
	"sync"
	"time"

	schedulev1alpha1 "github.com/everpeace/kube-throttler/pkg/apis/schedule/v1alpha1"
	scheduleclient "github.com/everpeace/kube-throttler/pkg/generated/clientset/versioned"
	scheduleinformers "github.com/everpeace/kube-throttler/pkg/generated/informers/externalversions"
	"github.com/pkg/errors"
	v1 "k8s.io/api/core/v1"
	metav1 "k8s.io/apimachinery/pkg/apis/meta/v1"
	"k8s.io/apimachinery/pkg/runtime"
	"k8s.io/apimachinery/pkg/types"
	utilruntime "k8s.io/apimachinery/pkg/util/runtime"
	"k8s.io/client-go/informers"
	"k8s.io/client-go/kubernetes"
	"k8s.io/client-go/tools/cache"
	"k8s.io/client-go/tools/clientcmd"
	"k8s.io/klog/v2"
	"k8s.io/kubernetes/pkg/scheduler/framework"
)

const (
	// PluginName of the plugin used in the plugin registry and configurations.
	PluginName = "kube-throttler"
)

type KubeThrottler struct {
	fh  framework.Handle
	eng *engine // stands where throttleCtr / clusterThrottleCtr stood (plugin.go:48-52)

	scheduleClientset *scheduleclient.Clientset
	kick              chan struct{} // an informer event happened: reconcile soon (coalesced)
	timerMu           sync.Mutex
	timer             *time.Timer // earliest temporaryThresholdOverride boundary (enqueueAfter, throttle_controller.go:201-208)
}

var _ framework.PreFilterPlugin = &KubeThrottler{}
var _ framework.EnqueueExtensions = &KubeThrottler{}
var _ framework.ReservePlugin = &KubeThrottler{}

func (p *KubeThrottler) Name() string {
	return PluginName
}

// NewPlugin initializes a new plugin and returns it.
func NewPlugin(configuration runtime.Object, fh framework.Handle) (framework.Plugin, error) {
	ctx := context.TODO()

	args, err := DecodePluginArgs(configuration)
	if err != nil {
		return nil, err
	}
	restConfig, err := clientcmd.BuildConfigFromFlags("", args.KubeConifg)
	if err != nil {
		return nil, err
	}
	eng, err := newEngine(args, gpuDevice())
	if err != nil {
		return nil, err
	}
	pl := &KubeThrottler{fh: fh, eng: eng, kick: make(chan struct{}, 1)}
	pl.scheduleClientset = scheduleclient.NewForConfigOrDie(restConfig)

	// Same informers as the reference (own pod informer for the namespace index, plugin.go:81-88); their handlers now only
	// hand the object to the engine, which packs it (labels -> dictionary ids, ResourceAmountOfPod once) into its HBM row.
	scheduleInformerFactory := scheduleinformers.NewSharedInformerFactory(pl.scheduleClientset, 5*time.Minute)
	throttleInformer := scheduleInformerFactory.Schedule().V1alpha1().Throttles().Informer()
	clusterthrottleInformer := scheduleInformerFactory.Schedule().V1alpha1().ClusterThrottles().Informer()
	informerFactory := informers.NewSharedInformerFactory(kubernetes.NewForConfigOrDie(restConfig), 5*time.Minute)
	podInformer := informerFactory.Core().V1().Pods().Informer()
	namespaceInformer := informerFactory.Core().V1().Namespaces().Informer()

	for kind, inf := range map[string]cache.SharedIndexInformer{
		"Namespace": namespaceInformer, "Throttle": throttleInformer, "ClusterThrottle": clusterthrottleInformer, "Pod": podInformer,
	} {
		if _, err := inf.AddEventHandler(pl.handlers(kind)); err != nil {
			panic(fmt.Sprintf("failed to add event handler in %s informer: %v", kind, err)) // as the reference's controllers do
		}
	}

	for _, f := range []interface {
		Start(<-chan struct{})
	}{scheduleInformerFactory, informerFactory} {
		f.Start(ctx.Done())
	}
	for informer, ok := range scheduleInformerFactory.WaitForCacheSync(ctx.Done()) {
		if !ok {
			return nil, errors.Errorf("failed to wait for caches to sync: informer=%v", informer)
		}
		klog.InfoS("Informer cache synched", "Informer", fmt.Sprintf("%v", informer))
	}
	for informer, ok := range informerFactory.WaitForCacheSync(ctx.Done()) {
		if !ok {
			return nil, errors.Errorf("failed to wait for caches to sync: informer=%v", informer)
		}
		klog.InfoS("Informer cache synched", "Informer", fmt.Sprintf("%v", informer))
	}

	// One worker replaces the two controllers' workqueues: a reconcile pass recomputes status.used / throttled /
	// calculatedThreshold of EVERY responsible throttle on the device, so per-key queueing has nothing left to order.
	go pl.reconcileLoop(context.Background(), args.ReconcileTemporaryThresholdInterval)
	pl.poke()
	return pl, nil
}

// withKind fills in the TypeMeta informer objects do not carry: the engine dispatches on "kind".
func withKind(kind string, obj interface{}) interface{} {
	switch o := obj.(type) {
	case *v1.Pod:
		c := o.DeepCopy()
		c.Kind = kind
		return c
	case *v1.Namespace:
		c := o.DeepCopy()
		c.Kind = kind
		return c
	case *schedulev1alpha1.Throttle:
		c := o.DeepCopy()
		c.Kind = kind
		return c
	case *schedulev1alpha1.ClusterThrottle:
		c := o.DeepCopy()
		c.Kind = kind
		return c
	}
	return obj
}

func (pl *KubeThrottler) handlers(kind string) cache.ResourceEventHandlerFuncs {
	upsert := func(obj interface{}) {
		if err := pl.eng.apply(withKind(kind, obj)); err != nil {
			utilruntime.HandleError(errors.Wrapf(err, "kube-throttler engine refused %s", kind))
			return
		}
		pl.poke()
	}
	return cache.ResourceEventHandlerFuncs{
		AddFunc:    upsert,
		UpdateFunc: func(_, newObj interface{}) { upsert(newObj) },
		DeleteFunc: func(obj interface{}) {
			if tomb, ok := obj.(cache.DeletedFinalStateUnknown); ok {
				obj = tomb.Obj
			}
			m, err := metaOf(obj)
			if err != nil {
				utilruntime.HandleError(err)
				return
			}
			if err := pl.eng.delete(kind, m.GetNamespace(), m.GetName()); err != nil {
				utilruntime.HandleError(errors.Wrapf(err, "kube-throttler engine failed to delete %s %s/%s", kind, m.GetNamespace(), m.GetName()))
			}
			pl.poke()
		},
	}
}

func metaOf(obj interface{}) (metav1.Object, error) {
	if m, ok := obj.(metav1.Object); ok {
		return m, nil
	}
	return nil, fmt.Errorf("unexpected object in informer event: %T", obj)
}

func (pl *KubeThrottler) poke() {
	select {
	case pl.kick <- struct{}{}:
	default: // a reconcile is already pending: events coalesce
	}
}

// reconcileLoop is reconcile(key) for every key at once (throttle_controller.go:84-211, clusterthrottle_controller.go:87-214):
// the engine computes the new statuses, the names under "changed" get an UpdateStatus, the override boundaries re-arm
// the timer.  The resync tick stands in for the reference's reconcileTemporaryThresholdInterval.
func (pl *KubeThrottler) reconcileLoop(ctx context.Context, interval time.Duration) {
	tick := time.NewTicker(interval)
	defer tick.Stop()
	for {
		select {
		case <-ctx.Done():
			return
		case <-pl.kick:
		case <-tick.C:
		}
		res, err := pl.eng.reconcileAll(time.Now().UTC().Format(time.RFC3339Nano))
		if err != nil {
			utilruntime.HandleError(errors.Wrap(err, "reconcile pass failed"))
			continue
		}
		for _, nn := range res.Changed {
			if err := pl.updateStatus(ctx, nn); err != nil {
				utilruntime.HandleError(err)
			}
		}
		var soonest time.Duration
		for _, ns := range res.RequeueAfterNanos {
			if d := time.Duration(ns); soonest == 0 || d < soonest {
				soonest = d
			}
		}
		if soonest > 0 {
			pl.timerMu.Lock()
			if pl.timer != nil {
				pl.timer.Stop()
			}
			pl.timer = time.AfterFunc(soonest, pl.poke)
			pl.timerMu.Unlock()
		}
	}
}

// updateStatus sends the status the engine computed for "ns/name" (Throttle) or "/name" (ClusterThrottle).
func (pl *KubeThrottler) updateStatus(ctx context.Context, nn string) error {
	i := strings.IndexByte(nn, '/')
	ns, name := nn[:i], nn[i+1:]
	manifest, err := pl.eng.statusManifest(ns, name)
	if err != nil {
		return err
	}
	patch := []byte(`{"status":` + string(manifest) + `}`)
	if ns != "" {
		_, err = pl.scheduleClientset.ScheduleV1alpha1().Throttles(ns).Patch(ctx, name, types.MergePatchType, patch, metav1.PatchOptions{}, "status")
		return errors.Wrapf(err, "failed to update Throttle '%s' status", nn)
	}
	_, err = pl.scheduleClientset.ScheduleV1alpha1().ClusterThrottles().Patch(ctx, name, types.MergePatchType, patch, metav1.PatchOptions{}, "status")
	return errors.Wrapf(err, "failed to update ClusterThrottle '%s' status", name)
}

func (pl *KubeThrottler) PreFilter(
	ctx context.Context,
	state *framework.CycleState,
	pod *v1.Pod,
) (*framework.PreFilterResult, *framework.Status) {
	r, err := pl.eng.preFilter(withKind("Pod", pod))
	if err != nil {
		return nil, framework.NewStatus(framework.Error, err.Error())
	}
	switch r.Code {
	case "Success":
		return nil, framework.NewStatus(framework.Success)
	case "Error": // a controller error (broken podSelector, unknown namespace): plugin.go:154-156,166-168
		return nil, framework.NewStatus(framework.Error, r.Reasons...)
	}
	if r.Event != nil { // some threshold is below the pod's own requests (plugin.go:189-201)
		pl.fh.EventRecorder().Eventf(pod, nil, r.Event.Type, r.Event.Reason, pl.Name(), r.Event.Message)
	}
	klog.V(2).InfoS("PreFilter: throttled", "Pod", pod.Namespace+"/"+pod.Name, "Reasons", strings.Join(r.Reasons, ";"))
	return nil, framework.NewStatus(framework.UnschedulableAndUnresolvable, r.Reasons...)
}

func (pl *KubeThrottler) Reserve(
	ctx context.Context,
	state *framework.CycleState,
	pod *v1.Pod,
	node string,
) *framework.Status {
	r, err := pl.eng.reserve(withKind("Pod", pod))
	if err != nil {
		return framework.NewStatus(framework.Error, err.Error())
	}
	if r.Code != "Success" {
		return framework.NewStatus(framework.Error, r.Reasons...)
	}
	klog.V(2).InfoS("Reserve: pod is reserved", "pod", pod.Namespace+"/"+pod.Name)
	return framework.NewStatus(framework.Success)
}

func (pl *KubeThrottler) Unreserve(
	ctx context.Context,
	state *framework.CycleState,
	pod *v1.Pod,
	node string,
) {
	if err := pl.eng.unreserve(withKind("Pod", pod)); err != nil { // never fails the cycle (plugin.go:246-254)
		utilruntime.HandleError(errors.Wrapf(err, "Failed to unreserve pod %s/%s", pod.Namespace, pod.Name))
	}
	klog.V(2).InfoS("Unreserve: pod is unreserved", "pod", pod.Namespace+"/"+pod.Name)
}

func (p *KubeThrottler) PreFilterExtensions() framework.PreFilterExtensions {
	return nil
}

func (p *KubeThrottler) EventsToRegister() []framework.ClusterEvent {
	gv := schedulev1alpha1.SchemeGroupVersion
	events := []framework.ClusterEvent{{Resource: framework.Node, ActionType: framework.All}, {Resource: framework.Pod, ActionType: framework.All}}
	for _, plural := range []string{"throttles", "clusterthrottles"} {
		events = append(events, framework.ClusterEvent{Resource: framework.GVK(fmt.Sprintf("%s.%v.%v", plural, gv.Version, gv.Group)), ActionType: framework.All})
	}
	return events
}
