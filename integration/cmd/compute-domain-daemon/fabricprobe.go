// fabricprobe.go — new file for cmd/compute-domain-daemon (NVIDIA/k8s-dra-driver-gpu).
//
// NOT COMPILED IN THIS REPOSITORY (no Go toolchain in the build image, SURVEY.md F4).  The behaviour
// it specifies is executable as the C++ twin k8s-dra-driver-gpu_b200/csrc/daemon_main.cc
// (`cdprobe-daemon {run,check}`, tests/test_daemon.py).  The two share ONE verdict file schema:
// tests/test_daemon.py parses the json tags of fabricProbeVerdict below and checks every key and JSON
// type of the file the C++ twin writes against them, so either `run` can feed either `check`.
//
// Wiring (INTEGRATION.md §2 has the main.go hunks):
//   newApp(): cliFlags = append(cliFlags, fabricProbeCLIFlags()...)   // next to featureGateConfig.Flags(), main.go:166
//   run():   after addComputeDomainCliqueLabel(), BEFORE the `if flags.cliqueID == ""` early wait
//            (main.go:244-250) so single-node HGX boxes are covered too:
//                prober := startFabricProbe(ctx, flags)
//                defer prober.Stop()
//   update loops (main.go:351-431): the probe is re-run from INSIDE the existing loops, after
//            writeDaemonsConfig / UpdateDNSNameMappings:
//                prober.Kick()
//            GetDaemonInfoUpdateChan() keeps its single receiver — a second `range` over that channel
//            would steal daemon-set updates from the IMEX config / DNS loops (a Go channel delivers each
//            value to exactly one receiver).
//   check(): after the existing IMEX gate (main.go:435-459), and in its cliqueID == "" early return:
//                if err := checkFabricProbeVerdict(flags); err != nil { return err }
package main

import (
	"context"
	"encoding/json"
	"errors"
	"fmt"
	"os"
	"path/filepath"
	"strings"
	"time"

	"github.com/urfave/cli/v2"
	"k8s.io/klog/v2"

	"sigs.k8s.io/dra-driver-nvidia-gpu/pkg/fabricprobe"
	"sigs.k8s.io/dra-driver-nvidia-gpu/pkg/featuregates"
	"sigs.k8s.io/dra-driver-nvidia-gpu/pkg/metrics"
)

const (
	// The per-ComputeDomain bind mount shared by `run` and `check` (computedomain.go:170-177).  It is a
	// host path that outlives pods: run() removes whatever verdict it finds there before probing, and
	// every verdict names the pod and boot that wrote it.
	fabricProbeVerdictPath   = "/imexd/fabricprobe.json"
	fabricProbeVerdictSchema = 2
)

// fabricProbeOptions are the probe's own flags.  They live in this file (package-level, filled by urfave/cli through
// Destination pointers exactly like the fields of Flags, main.go:104-166) so that the patch to main.go stays one
// appended line; podUID and nodeName come from the existing Flags.
type fabricProbeOptions struct {
	bytes        uint64
	mode         string
	minFraction  float64
	linkPeakGBps float64
	intervalS    int
	maxAgeS      int
}

var fpOpts fabricProbeOptions

func fabricProbeCLIFlags() []cli.Flag {
	return []cli.Flag{
		&cli.Uint64Flag{
			Name:        "fabric-probe-bytes",
			Usage:       "Per-GPU buffer the fabric probe moves (bytes).",
			Value:       1 << 30,
			EnvVars:     []string{"FABRIC_PROBE_BYTES"},
			Destination: &fpOpts.bytes,
		},
		&cli.StringFlag{
			Name:        "fabric-probe-mode",
			Usage:       "sliced (bytes split over the peers), full (bytes per ordered pair) or reach-only.",
			Value:       "sliced",
			EnvVars:     []string{"FABRIC_PROBE_MODE"},
			Destination: &fpOpts.mode,
		},
		&cli.Float64Flag{
			Name:        "fabric-probe-min-fraction",
			Usage:       "Bandwidth gate as a fraction of the reference figure; 0 = library default.",
			EnvVars:     []string{"FABRIC_PROBE_MIN_FRACTION"},
			Destination: &fpOpts.minFraction,
		},
		&cli.Float64Flag{
			Name:        "fabric-probe-link-peak-gbps",
			Usage:       "Reference figure of the gate in GB/s; 0 = the library's default (nominal NVLink 4, include/cdprobe.h).",
			EnvVars:     []string{"FABRIC_PROBE_LINK_PEAK_GBPS"},
			Destination: &fpOpts.linkPeakGBps,
		},
		&cli.IntFlag{
			Name:        "fabric-probe-interval",
			Usage:       "Seconds between periodic probe passes; 0 = only at start and on daemon-set changes.",
			EnvVars:     []string{"FABRIC_PROBE_INTERVAL_S"},
			Destination: &fpOpts.intervalS,
		},
		&cli.IntFlag{
			Name:        "fabric-probe-max-age",
			Usage:       "check fails when the verdict is older than this many seconds; 0 = 3 x interval + 60 when an interval is set, else never.",
			EnvVars:     []string{"FABRIC_PROBE_MAX_AGE_S"},
			Destination: &fpOpts.maxAgeS,
		},
	}
}

func (o *fabricProbeOptions) modeID() uint32 {
	switch o.mode {
	case "full":
		return fabricprobe.ModeFull
	case "reach-only":
		return fabricprobe.ModeReachOnly
	default:
		return fabricprobe.ModeSliced
	}
}

func (o *fabricProbeOptions) interval() time.Duration { return time.Duration(o.intervalS) * time.Second }

// fabricProbeVerdict is the file `run` writes and `check` reads.  Reach matrices are 0/1 integers
// (a []bool would marshal as true/false and a []uint8 as base64; the C++ twin prints integers).
type fabricProbeVerdict struct {
	Schema           int       `json:"schema"`
	TimeUnix         int64     `json:"time_unix"`
	PodUID           string    `json:"pod_uid"`
	BootID           string    `json:"boot_id"`
	OK               bool      `json:"ok"`
	N                int       `json:"n"`
	UnreachablePairs int       `json:"unreachable_pairs"`
	SlowPairs        int       `json:"slow_pairs"`
	MinGBpsRead      float32   `json:"min_gbps_read"`
	MinGBpsWrite     float32   `json:"min_gbps_write"`
	GateGBpsRead     float32   `json:"gate_gbps_read"`
	GateGBpsWrite    float32   `json:"gate_gbps_write"`
	ProbeMs          float64   `json:"probe_ms"`
	BytesPerPair     uint64    `json:"bytes_per_pair"`
	ReachRead        []int     `json:"reach_read"`
	ReachWrite       []int     `json:"reach_write"`
	GBpsRead         []float32 `json:"gbps_read"`
	GBpsWrite        []float32 `json:"gbps_write"`
	Error            string    `json:"error"`
}

// fabricProber owns the probe handle.  Kick() asks for another pass and never blocks: the update
// loops call it from their own goroutine.
type fabricProber struct {
	kick chan struct{}
	done chan struct{}
}

func (p *fabricProber) Kick() {
	if p == nil || p.kick == nil {
		return
	}
	select {
	case p.kick <- struct{}{}:
	default: // a pass is already pending
	}
}

func (p *fabricProber) Stop() {
	if p == nil || p.done == nil {
		return
	}
	<-p.done
}

func bootID() string {
	raw, err := os.ReadFile("/proc/sys/kernel/random/boot_id")
	if err != nil {
		return ""
	}
	return strings.TrimSpace(string(raw))
}

func boolsToInts(b []bool) []int {
	out := make([]int, len(b))
	for i, v := range b {
		if v {
			out[i] = 1
		}
	}
	return out
}

// startFabricProbe removes a stale verdict, opens the probe and runs it once; further passes happen on
// Kick() (daemon-set changes) and every FABRIC_PROBE_INTERVAL_S seconds when that is set.  It returns at
// once; Stop() waits for the goroutine (which exits on ctx cancel) and closes the handle.
func startFabricProbe(ctx context.Context, flags *Flags) *fabricProber {
	p := &fabricProber{}
	if !featuregates.Enabled(featuregates.FabricProbe) {
		return p
	}
	// Whatever is in the mount was written by another pod / container instance.
	if err := os.Remove(fabricProbeVerdictPath); err != nil && !errors.Is(err, os.ErrNotExist) {
		klog.Warningf("cannot remove stale %s: %v", fabricProbeVerdictPath, err)
	}
	cfg := fabricprobe.Config{
		Bytes:        fpOpts.bytes,                 // FABRIC_PROBE_BYTES, default 1 GiB
		Mode:         fpOpts.modeID(),              // FABRIC_PROBE_MODE, default sliced
		MinFraction:  float32(fpOpts.minFraction),  // FABRIC_PROBE_MIN_FRACTION, 0 = library default
		LinkPeakGBps: float32(fpOpts.linkPeakGBps), // FABRIC_PROBE_LINK_PEAK_GBPS, 0 = library default reference
		TimeoutMs:    5000,
		Flags:        fabricprobe.FlagFabricHandles | fabricprobe.FlagMigAware,
	}
	probe, err := fabricprobe.Open(cfg)
	switch {
	case errors.Is(err, fabricprobe.ErrUnsupported):
		// No libcdprobe.so / no CUDA driver / not sm_90: there is no CPU stand-in.  No verdict is
		// written and check() does not gate on a missing verdict.
		klog.Infof("fabric probe not supported on this node: %v", err)
		return p
	case err != nil:
		// A node whose probe cannot even be set up is not Ready: leave a failing verdict, not none.
		klog.Errorf("error opening fabric probe: %v", err)
		writeVerdict(fabricprobe.Result{}, fmt.Errorf("cdprobe_open: %w", err), flags)
		return p
	}

	runOnce := func() {
		if probe == nil { // the previous pass left the handle unusable
			if probe, err = fabricprobe.Open(cfg); err != nil {
				klog.Errorf("error reopening fabric probe: %v", err)
				writeVerdict(fabricprobe.Result{}, fmt.Errorf("cdprobe_open: %w", err), flags)
				probe = nil
				return
			}
		}
		t0 := time.Now()
		res, err := probe.Run(ctx)
		d := time.Since(t0)
		klog.V(6).Infof("t_fabric_probe %.6f s", d.Seconds())
		v := writeVerdict(res, err, flags)
		metrics.ObserveFabricProbe(flags.nodeName, d, v.OK, v.UnreachablePairs, v.SlowPairs, res.N, res.GBpsRead, res.GBpsWrite)
		klog.Infof("fabric probe: verdict ok=%t, %d GPU(s), %d unreachable pair(s), %d slow pair(s), min read %.0f GB/s, min write %.0f GB/s, %.3f ms",
			v.OK, v.N, v.UnreachablePairs, v.SlowPairs, v.MinGBpsRead, v.MinGBpsWrite, v.ProbeMs)
		if err != nil && (errors.Is(err, fabricprobe.ErrTimeout) || errors.Is(err, fabricprobe.ErrState) || errors.Is(err, fabricprobe.ErrCUDA)) {
			// a timed-out pass may leave the handle sticky (Run then only returns ErrState): start afresh
			probe.Close()
			probe = nil
		}
	}

	p.kick = make(chan struct{}, 1)
	p.done = make(chan struct{})
	go func() {
		defer close(p.done)
		defer func() {
			if probe != nil {
				probe.Close()
			}
		}()
		var tick <-chan time.Time
		if fpOpts.interval() > 0 {
			t := time.NewTicker(fpOpts.interval())
			defer t.Stop()
			tick = t.C
		}
		runOnce()
		for {
			select {
			case <-ctx.Done():
				return
			case <-p.kick:
				runOnce()
			case <-tick:
				runOnce()
			}
		}
	}()
	return p
}

func writeVerdict(res fabricprobe.Result, runErr error, flags *Flags) fabricProbeVerdict {
	v := fabricProbeVerdict{
		Schema: fabricProbeVerdictSchema, TimeUnix: time.Now().Unix(), PodUID: flags.podUID, BootID: bootID(),
		OK: runErr == nil && res.Verdict, N: res.N,
		UnreachablePairs: res.UnreachablePairs, SlowPairs: res.SlowPairs,
		MinGBpsRead: res.MinGBpsRead, MinGBpsWrite: res.MinGBpsWrite,
		GateGBpsRead: res.GateGBpsRead, GateGBpsWrite: res.GateGBpsWrite,
		ProbeMs: res.ProbeMs, BytesPerPair: res.BytesPerPair,
		ReachRead: boolsToInts(res.ReachRead), ReachWrite: boolsToInts(res.ReachWrite),
		// never nil: an empty result marshals as [] like the C++ twin writes it, not as null
		GBpsRead: append([]float32{}, res.GBpsRead...), GBpsWrite: append([]float32{}, res.GBpsWrite...),
	}
	if runErr != nil {
		v.Error = runErr.Error()
	}
	if err := writeFileAtomic(fabricProbeVerdictPath, v); err != nil {
		klog.Errorf("cannot write %s: %v", fabricProbeVerdictPath, err)
	}
	return v
}

// checkFabricProbeVerdict is the addition to check(): a failed verdict makes the pod NotReady; a missing
// one — or one this pod did not write — does not (same spirit as the reference's no-op when CLIQUE_ID is
// empty, main.go:436-439).
func checkFabricProbeVerdict(flags *Flags) error {
	if !featuregates.Enabled(featuregates.FabricProbe) {
		return nil
	}
	raw, err := os.ReadFile(fabricProbeVerdictPath)
	if errors.Is(err, os.ErrNotExist) {
		return nil
	}
	if err != nil {
		return fmt.Errorf("fabric probe verdict unreadable: %w", err)
	}
	var v fabricProbeVerdict
	if err := json.Unmarshal(raw, &v); err != nil {
		return fmt.Errorf("fabric probe verdict unreadable: %w", err)
	}
	if v.PodUID != "" && flags.podUID != "" && v.PodUID != flags.podUID {
		return nil // another pod's verdict (the mount outlives pods)
	}
	if b := bootID(); v.BootID != "" && b != "" && v.BootID != b {
		return nil
	}
	maxAge := time.Duration(fpOpts.maxAgeS) * time.Second // FABRIC_PROBE_MAX_AGE_S
	if maxAge <= 0 && fpOpts.interval() > 0 {
		maxAge = 3*fpOpts.interval() + time.Minute // periodic re-probe on: a verdict must keep coming
	}
	if age := time.Since(time.Unix(v.TimeUnix, 0)); maxAge > 0 && age > maxAge {
		return fmt.Errorf("fabric probe verdict is stale (%d s old)", int(age.Seconds()))
	}
	if !v.OK {
		msg := fmt.Sprintf("fabric probe failed: %d unreachable pair(s), %d slow pair(s), min read %.0f GB/s, min write %.0f GB/s",
			v.UnreachablePairs, v.SlowPairs, v.MinGBpsRead, v.MinGBpsWrite)
		if v.Error != "" {
			msg += ": " + v.Error
		}
		return errors.New(msg)
	}
	return nil
}

func writeFileAtomic(path string, v any) error {
	raw, err := json.MarshalIndent(v, "", " ")
	if err != nil {
		return err
	}
	tmp := filepath.Join(filepath.Dir(path), "."+filepath.Base(path)+".tmp")
	if err := os.WriteFile(tmp, raw, 0o644); err != nil {
		return err
	}
	return os.Rename(tmp, path)
}
