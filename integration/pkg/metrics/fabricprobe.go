// fabricprobe.go — addition to pkg/metrics (NVIDIA/k8s-dra-driver-gpu), same conventions as
// dra_requests.go:27-151: namespace nvidia_dra, k8s.io/component-base/metrics, legacyregistry,
// registration behind a sync.Once.  NOT COMPILED IN THIS REPOSITORY (no Go toolchain); the C++ twin
// writes the same series as a Prometheus textfile when FABRIC_PROBE_METRICS_PATH is set
// (k8s-dra-driver-gpu_b200/csrc/daemon_main.cc, asserted by tests/test_daemon.py).
package metrics

import (
	"strconv"
	"sync"
	"time"

	"k8s.io/component-base/metrics"
	"k8s.io/component-base/metrics/legacyregistry"

	"sigs.k8s.io/dra-driver-nvidia-gpu/pkg/fabricprobe"
)

var (
	fabricProbeRegisterOnce sync.Once

	fabricProbeDurationSeconds = metrics.NewGaugeVec(
		&metrics.GaugeOpts{
			Namespace: "nvidia_dra",
			Name:      "fabric_probe_duration_seconds",
			Help:      "Duration of the last all-pairs NVLink fabric probe pass on this node.",
		},
		[]string{"node"},
	)
	fabricProbeOK = metrics.NewGaugeVec(
		&metrics.GaugeOpts{
			Namespace: "nvidia_dra",
			Name:      "fabric_probe_ok",
			Help:      "1 if the last fabric probe pass found every GPU pair reachable and at speed, else 0.",
		},
		[]string{"node"},
	)
	fabricProbeUnreachablePairs = metrics.NewGaugeVec(
		&metrics.GaugeOpts{
			Namespace: "nvidia_dra",
			Name:      "fabric_probe_unreachable_pairs",
			Help:      "Ordered GPU pairs the last fabric probe pass could not read or write over NVLink.",
		},
		[]string{"node"},
	)
	fabricProbeSlowPairs = metrics.NewGaugeVec(
		&metrics.GaugeOpts{
			Namespace: "nvidia_dra",
			Name:      "fabric_probe_slow_pairs",
			Help:      "Ordered GPU pairs that were reachable but under the bandwidth gate in the last pass.",
		},
		[]string{"node"},
	)
	fabricProbePairGBps = metrics.NewGaugeVec(
		&metrics.GaugeOpts{
			Namespace: "nvidia_dra",
			Name:      "fabric_probe_pair_gbps",
			Help:      "Per ordered GPU pair payload bandwidth measured by the last fabric probe pass.",
		},
		[]string{"node", "src", "dst", "op"},
	)
	fabricProbePassesTotal = metrics.NewCounterVec(
		&metrics.CounterOpts{
			Namespace: "nvidia_dra",
			Name:      "fabric_probe_passes_total",
			Help:      "Fabric probe passes by outcome.",
		},
		[]string{"node", "outcome"},
	)
	fabricProbeLinkKiB = metrics.NewGaugeVec(
		&metrics.GaugeOpts{
			Namespace: "nvidia_dra",
			Name:      "fabric_probe_link_kib",
			Help:      "NVLink data a GPU link sent (dir tx) or received (dir rx) over the last fabric probe pass, in KiB, as NVML counts it.",
		},
		[]string{"node", "gpu", "link", "dir"},
	)
	fabricProbeLinkErrors = metrics.NewGaugeVec(
		&metrics.GaugeOpts{
			Namespace: "nvidia_dra",
			Name:      "fabric_probe_link_errors",
			Help:      "NVLink data-link errors (counter replay, recovery or crc) a GPU link counted over the last fabric probe pass.",
		},
		[]string{"node", "gpu", "link", "counter"},
	)
)

func registerFabricProbe() {
	fabricProbeRegisterOnce.Do(func() {
		legacyregistry.MustRegister(
			fabricProbeDurationSeconds,
			fabricProbeOK,
			fabricProbeUnreachablePairs,
			fabricProbeSlowPairs,
			fabricProbePairGBps,
			fabricProbePassesTotal,
			fabricProbeLinkKiB,
			fabricProbeLinkErrors,
		)
	})
}

// ObserveFabricProbe records one pass.  gbpsRead/gbpsWrite are n x n row-major, [issuer*n + target].
func ObserveFabricProbe(node string, d time.Duration, ok bool, unreachable, slow, n int, gbpsRead, gbpsWrite []float32) {
	registerFabricProbe()
	fabricProbeDurationSeconds.WithLabelValues(node).Set(d.Seconds())
	outcome := "failed"
	if ok {
		fabricProbeOK.WithLabelValues(node).Set(1)
		outcome = "ok"
	} else {
		fabricProbeOK.WithLabelValues(node).Set(0)
	}
	fabricProbePassesTotal.WithLabelValues(node, outcome).Inc()
	fabricProbeUnreachablePairs.WithLabelValues(node).Set(float64(unreachable))
	fabricProbeSlowPairs.WithLabelValues(node).Set(float64(slow))
	for i := 0; i < n; i++ {
		for j := 0; j < n; j++ {
			if i == j && n > 1 {
				continue
			}
			if k := i*n + j; k < len(gbpsRead) && k < len(gbpsWrite) {
				fabricProbePairGBps.WithLabelValues(node, strconv.Itoa(i), strconv.Itoa(j), "read").Set(float64(gbpsRead[k]))
				fabricProbePairGBps.WithLabelValues(node, strconv.Itoa(i), strconv.Itoa(j), "write").Set(float64(gbpsWrite[k]))
			}
		}
	}
}

// ObserveFabricProbeLinks records the per-link NVLink counters of one pass, for every GPU NVML could sample.
func ObserveFabricProbeLinks(node string, links fabricprobe.Links) {
	registerFabricProbe()
	for _, d := range links.Devices {
		if d.Status != 0 {
			continue
		}
		for l := range d.TxKiB {
			link := strconv.Itoa(l)
			fabricProbeLinkKiB.WithLabelValues(node, d.UUID, link, "tx").Set(float64(d.TxKiB[l]))
			fabricProbeLinkKiB.WithLabelValues(node, d.UUID, link, "rx").Set(float64(d.RxKiB[l]))
			for c, name := range fabricprobe.LinkCounterNames {
				fabricProbeLinkErrors.WithLabelValues(node, d.UUID, link, name).Set(float64(d.Errors[l][c]))
			}
		}
	}
}
