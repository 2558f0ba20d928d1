// NOT COMPILED IN THIS REPOSITORY'S ENVIRONMENT (no Go toolchain in the image; see go/README.md).
//
// Plugin arguments of the kube-throttler scheduler plugin, decoded exactly as the reference does
// (everpeace/kube-throttler pkg/scheduler_plugin/plugin_args.go:33-60): the same struct, the same JSON tags -- misspellings
// included, they are the wire format of existing pluginConfig objects -- the same defaults and error texts.
// The GPU build adds nothing to the wire format: the GPU ordinal comes from the environment (KT_B200_DEVICE).

package scheduler_plugin

import (
	"fmt"
	"os"
	goruntime "runtime"
	"strconv"
	"time"

	"k8s.io/apimachinery/pkg/runtime"
	fwkruntime "k8s.io/kubernetes/pkg/scheduler/framework/runtime"
)

var (
	DefaultReconcileTemporaryThresholdInterval = 15 * time.Second
)

type KubeThrottlerPluginArgs struct {
	Name                                string        `json:"name"`
	KubeConifg                          string        `json:"kubeconfig"`
	ReconcileTemporaryThresholdInterval time.Duration `json:"reconcileTemporaryThresholdInterval"`
	TargetSchedulerName                 string        `json:"targetSchedulerName"`
	ControllerThrediness                int           `json:"controllerThrediness"`
	NumKeyMutex                         int           `json:"numKeyMutex"`
}

func DecodePluginArgs(configuration runtime.Object) (*KubeThrottlerPluginArgs, error) {
	args := &KubeThrottlerPluginArgs{}
	if err := fwkruntime.DecodeInto(configuration, &args); err != nil {
		return nil, fmt.Errorf("Failed to decode into %s PluginConfig", PluginName)
	}
	switch {
	case args.Name == "":
		return nil, fmt.Errorf("Name must not be empty")
	case args.TargetSchedulerName == "":
		return nil, fmt.Errorf("TargetSchedulerName must not be empty")
	}
	if args.ReconcileTemporaryThresholdInterval == 0 {
		args.ReconcileTemporaryThresholdInterval = DefaultReconcileTemporaryThresholdInterval
	}
	if args.ControllerThrediness == 0 {
		// kept for wire compatibility: the device pass reconciles every throttle at once, one worker drives it
		args.ControllerThrediness = goruntime.NumCPU()
	}
	return args, nil
}

// gpuDevice is the CUDA ordinal the plugin's engine is created on.  Not a plugin argument on purpose.
func gpuDevice() int {
	if v, err := strconv.Atoi(os.Getenv("KT_B200_DEVICE")); err == nil && v >= 0 {
		return v
	}
	return 0
}
