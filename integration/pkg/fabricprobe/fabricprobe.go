//go:build cgo

// Package fabricprobe binds libcdprobe.so (include/cdprobe.h): the all-pairs NVLink
// reachability + bandwidth probe the compute-domain-daemon runs before it reports its
// node Ready.  It is meant to be dropped into NVIDIA/k8s-dra-driver-gpu as pkg/fabricprobe;
// the only caller is cmd/compute-domain-daemon (run(): main.go:212-347, check(): main.go:435-459).
//
// NOT COMPILED IN THIS REPOSITORY: the build image has no Go toolchain (SURVEY.md F4).  The
// file is a mechanical mirror of the C ABI so it can be reviewed by eye; the same ABI is
// exercised from Python/ctypes by k8s-dra-driver-gpu_b200/fabricprobe.py and tests/.
//
// The library is opened lazily with dlopen at Open(), the pattern go-nvml uses for
// libnvidia-ml.so.1 (vendor/github.com/NVIDIA/go-nvml/pkg/nvml/lib.go:29-80), so the daemon
// binary still starts on nodes that do not ship libcdprobe.so.
package fabricprobe

/*
#cgo CFLAGS: -I${SRCDIR}
#cgo LDFLAGS: -ldl
// cdprobe.h (this repository's include/cdprobe.h) is vendored next to this file.
#include <dlfcn.h>
#include <stdint.h>
#include <stdlib.h>
#include "cdprobe.h"

typedef int (*open_fn)(const cdprobe_config_t*, cdprobe_t**);
typedef int (*run_fn)(cdprobe_t*, cdprobe_result_t*);
typedef void (*close_fn)(cdprobe_t*);
typedef const char* (*str_fn)(int);
typedef const char* (*last_fn)(void);
typedef uint32_t (*abi_fn)(void);

static void* cdp_dl;
static open_fn cdp_open; static run_fn cdp_run; static close_fn cdp_close;
static str_fn cdp_strerror; static last_fn cdp_last; static abi_fn cdp_abi;

static int cdp_load(const char* path) {
  if (cdp_dl) return 0;
  cdp_dl = dlopen(path, RTLD_LAZY | RTLD_GLOBAL);
  if (!cdp_dl) return -1;
  cdp_open = (open_fn)dlsym(cdp_dl, "cdprobe_open");
  cdp_run = (run_fn)dlsym(cdp_dl, "cdprobe_run");
  cdp_close = (close_fn)dlsym(cdp_dl, "cdprobe_close");
  cdp_strerror = (str_fn)dlsym(cdp_dl, "cdprobe_strerror");
  cdp_last = (last_fn)dlsym(cdp_dl, "cdprobe_last_error");
  cdp_abi = (abi_fn)dlsym(cdp_dl, "cdprobe_abi_version");
  if (!cdp_open || !cdp_run || !cdp_close || !cdp_strerror || !cdp_last || !cdp_abi) return -2;
  return cdp_abi() == CDPROBE_ABI_VERSION ? 0 : -3;
}
static int cdp_call_open(const cdprobe_config_t* c, cdprobe_t** h) { return cdp_open(c, h); }
static int cdp_call_run(cdprobe_t* h, cdprobe_result_t* r) { return cdp_run(h, r); }
static void cdp_call_close(cdprobe_t* h) { cdp_close(h); }
static const char* cdp_call_strerror(int rc) { return cdp_strerror(rc); }
static const char* cdp_call_last(void) { return cdp_last(); }
*/
import "C"

import (
	"context"
	"errors"
	"fmt"
	"runtime"
	"unsafe"
)

const (
	ModeReachOnly = 0
	ModeSliced    = 1
	ModeFull      = 2
	OpRead        = 1
	OpWrite       = 2

	FlagFabricHandles = 0x01
	FlagMigAware      = 0x02
	FlagLocalDiag     = 0x04
)

// ErrUnsupported is returned when the probe cannot run on this node (no libcdprobe.so, no CUDA
// driver, no sm_90 GPU).  There is no CPU fallback: callers decide whether that gates Ready.
var ErrUnsupported = errors.New("fabricprobe: not supported on this node")

// Errors a Run can wrap (errors.Is).  After ErrTimeout, ErrState or ErrCUDA the handle may be
// unusable ("sticky"): Close it and Open a new one before the next pass.
var (
	ErrTimeout = errors.New("fabricprobe: probe timed out")        // CDPROBE_ERR_TIMEOUT
	ErrState   = errors.New("fabricprobe: handle is unusable")     // CDPROBE_ERR_STATE
	ErrCUDA    = errors.New("fabricprobe: CUDA call failed")       // CDPROBE_ERR_CUDA
)

type Config struct {
	LibraryPath string // default "libcdprobe.so"
	Ordinals    []int  // nil = every visible GPU
	Bytes       uint64 // per-GPU buffer (FABRIC_PROBE_BYTES, default 1 GiB)
	Mode        uint32 // FABRIC_PROBE_MODE
	Ops         uint32
	TimeoutMs   uint32
	Flags       uint32
	MinFraction float32 // FABRIC_PROBE_MIN_FRACTION; 0 = library default (0.65 of the reference)
	// FABRIC_PROBE_LINK_PEAK_GBPS; 0 = the library's default reference (nominal NVLink 4, include/cdprobe.h),
	// > 0 = absolute: the gate is MinFraction x LinkPeakGBps.
	LinkPeakGBps float32
}

type Result struct {
	N           int
	ReachRead   []bool // N x N row-major, [issuer*N + target]
	ReachWrite  []bool
	GBpsRead    []float32
	GBpsWrite   []float32
	Status      []int32
	ProbeMs     float64
	Verdict     bool
	Aborted     bool
	BytesPerPair uint64
	// Slowest filled off-diagonal pair, the GB/s gate the verdict applied (0: bandwidth not judged), and how
	// many ordered pairs failed it / were unreachable.
	MinGBpsRead, MinGBpsWrite   float32
	GateGBpsRead, GateGBpsWrite float32
	UnreachablePairs, SlowPairs int
}

type Probe struct {
	h *C.cdprobe_t
}

func Open(cfg Config) (*Probe, error) {
	// CUDA contexts are bound per OS thread inside the library; keep the goroutine pinned for
	// the duration of each call (go-nvml does the same around dlopen: pkg/dl/dl.go:68-73).
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	path := cfg.LibraryPath
	if path == "" {
		path = "libcdprobe.so"
	}
	cpath := C.CString(path)
	defer C.free(unsafe.Pointer(cpath))
	if rc := C.cdp_load(cpath); rc != 0 {
		return nil, fmt.Errorf("%w: cannot load %s (rc=%d)", ErrUnsupported, path, int(rc))
	}
	if len(cfg.Ordinals) > C.CDPROBE_MAX_GPUS {
		return nil, fmt.Errorf("fabricprobe: %d ordinals, the ABI carries at most %d", len(cfg.Ordinals), C.CDPROBE_MAX_GPUS)
	}
	var c C.cdprobe_config_t
	c.abi = C.CDPROBE_ABI_VERSION
	c.n_gpus = C.uint32_t(len(cfg.Ordinals))
	for i, o := range cfg.Ordinals {
		c.ordinals[i] = C.int32_t(o)
	}
	c.bytes = C.uint64_t(cfg.Bytes)
	c.mode = C.uint32_t(cfg.Mode)
	c.ops = C.uint32_t(cfg.Ops)
	c.timeout_ms = C.uint32_t(cfg.TimeoutMs)
	c.flags = C.uint32_t(cfg.Flags)
	c.min_fraction = C.float(cfg.MinFraction)
	c.link_peak_gbps = C.float(cfg.LinkPeakGBps)
	var h *C.cdprobe_t
	if rc := C.cdp_call_open(&c, &h); rc != 0 {
		err := fmt.Errorf("cdprobe_open: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_NO_DEVICE || rc == C.CDPROBE_ERR_UNSUPPORTED {
			return nil, fmt.Errorf("%w: %v", ErrUnsupported, err)
		}
		return nil, err
	}
	return &Probe{h: h}, nil
}

// Run executes one probe pass.  ctx is honoured between passes; a pass itself is bounded by
// Config.TimeoutMs (device watchdog + host watchdog), well inside the kubelet probe timeout
// of 10 s (templates/compute-domain-daemon.tmpl.yaml:83,90,97).
func (p *Probe) Run(ctx context.Context) (Result, error) {
	if err := ctx.Err(); err != nil {
		return Result{}, err
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	var r C.cdprobe_result_t
	rc := C.cdp_call_run(p.h, &r)
	n := int(r.n)
	out := Result{N: n, ProbeMs: float64(r.probe_ms), Verdict: r.verdict != 0, Aborted: r.aborted != 0,
		BytesPerPair: uint64(r.bytes_per_pair),
		MinGBpsRead: float32(r.min_gbps_read), MinGBpsWrite: float32(r.min_gbps_write),
		GateGBpsRead: float32(r.gate_gbps_read), GateGBpsWrite: float32(r.gate_gbps_write),
		UnreachablePairs: int(r.unreachable_pairs), SlowPairs: int(r.slow_pairs)}
	out.ReachRead = make([]bool, n*n)
	out.ReachWrite = make([]bool, n*n)
	out.GBpsRead = make([]float32, n*n)
	out.GBpsWrite = make([]float32, n*n)
	out.Status = make([]int32, n*n)
	for i := 0; i < n; i++ {
		for j := 0; j < n; j++ {
			k := i*C.CDPROBE_MAX_GPUS + j
			out.ReachRead[i*n+j] = r.reach_read[k] != 0
			out.ReachWrite[i*n+j] = r.reach_write[k] != 0
			out.GBpsRead[i*n+j] = float32(r.gbps_read[k])
			out.GBpsWrite[i*n+j] = float32(r.gbps_write[k])
			out.Status[i*n+j] = int32(r.status[k])
		}
	}
	if rc != 0 {
		// cdprobe_run zeroes and fills the result before anything can fail, so `out` is well-formed here
		err := fmt.Errorf("cdprobe_run: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
		switch rc {
		case C.CDPROBE_ERR_TIMEOUT:
			err = fmt.Errorf("%w: %v", ErrTimeout, err)
		case C.CDPROBE_ERR_STATE:
			err = fmt.Errorf("%w: %v", ErrState, err)
		case C.CDPROBE_ERR_CUDA:
			err = fmt.Errorf("%w: %v", ErrCUDA, err)
		}
		return out, err
	}
	return out, nil
}

func (p *Probe) Close() {
	if p != nil && p.h != nil {
		runtime.LockOSThread()
		C.cdp_call_close(p.h)
		runtime.UnlockOSThread()
		p.h = nil
	}
}
