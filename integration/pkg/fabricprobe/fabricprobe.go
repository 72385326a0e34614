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
typedef int (*diag_fn)(cdprobe_t*, uint32_t, uint32_t, uint32_t, uint32_t, cdprobe_diag_t*);
typedef int (*lat_fn)(cdprobe_t*, uint32_t, uint32_t, cdprobe_latency_t*);
typedef int (*pp_fn)(cdprobe_t*, uint32_t, uint32_t, uint32_t, cdprobe_pingpong_t*);
typedef int (*at_fn)(cdprobe_t*, uint32_t, uint32_t, uint32_t, cdprobe_atomics_t*);
typedef int (*bw_fn)(cdprobe_t*, uint32_t, cdprobe_bwcurve_t*);
typedef int (*ar_fn)(cdprobe_t*, uint32_t, cdprobe_allreduce_t*);
typedef int (*a2a_fn)(cdprobe_t*, uint32_t, cdprobe_alltoall_t*);
typedef int (*mc_fn)(cdprobe_t*, uint32_t, uint32_t, cdprobe_memcpy_t*);
typedef int (*cea_fn)(cdprobe_t*, uint32_t, uint32_t, cdprobe_ce_alltoall_t*);
typedef int (*opt_fn)(cdprobe_t*, uint32_t, uint64_t);
typedef int (*links_fn)(cdprobe_t*, cdprobe_links_t*);

static void* cdp_dl;
static open_fn cdp_open; static run_fn cdp_run; static close_fn cdp_close;
static str_fn cdp_strerror; static last_fn cdp_last; static abi_fn cdp_abi;
static diag_fn cdp_diag;  // optional: absent from libraries that predate cdprobe_diagnose
static lat_fn cdp_lat;    // optional: absent from libraries that predate cdprobe_latency
static pp_fn cdp_pp;      // optional: absent from libraries that predate cdprobe_pingpong
static at_fn cdp_at;      // optional: absent from libraries that predate cdprobe_atomics
static bw_fn cdp_bw;      // optional: absent from libraries that predate cdprobe_bwcurve
static ar_fn cdp_ar;      // optional: absent from libraries that predate cdprobe_allreduce
static a2a_fn cdp_a2a;    // optional: absent from libraries that predate cdprobe_alltoall
static ar_fn cdp_ar2;     // optional: absent from libraries that predate cdprobe_allreduce_twoshot
static ar_fn cdp_arll;    // optional: absent from libraries that predate cdprobe_allreduce_ll
static ar_fn cdp_arring;  // optional: absent from libraries that predate cdprobe_allreduce_ring
static ar_fn cdp_arpush;  // optional: absent from libraries that predate cdprobe_allreduce_push
static ar_fn cdp_arnvls;  // optional: absent from libraries that predate cdprobe_allreduce_nvls
static mc_fn cdp_mc;      // optional: absent from libraries that predate cdprobe_memcpy
static cea_fn cdp_cea;    // optional: absent from libraries that predate cdprobe_ce_alltoall
static opt_fn cdp_opt;    // optional: this binding did not need cdprobe_set_option before the link counters
static links_fn cdp_links;  // optional: absent from libraries that predate cdprobe_links

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
  cdp_diag = (diag_fn)dlsym(cdp_dl, "cdprobe_diagnose");
  cdp_lat = (lat_fn)dlsym(cdp_dl, "cdprobe_latency");
  cdp_pp = (pp_fn)dlsym(cdp_dl, "cdprobe_pingpong");
  cdp_at = (at_fn)dlsym(cdp_dl, "cdprobe_atomics");
  cdp_bw = (bw_fn)dlsym(cdp_dl, "cdprobe_bwcurve");
  cdp_ar = (ar_fn)dlsym(cdp_dl, "cdprobe_allreduce");
  cdp_a2a = (a2a_fn)dlsym(cdp_dl, "cdprobe_alltoall");
  cdp_ar2 = (ar_fn)dlsym(cdp_dl, "cdprobe_allreduce_twoshot");
  cdp_arll = (ar_fn)dlsym(cdp_dl, "cdprobe_allreduce_ll");
  cdp_arring = (ar_fn)dlsym(cdp_dl, "cdprobe_allreduce_ring");
  cdp_arpush = (ar_fn)dlsym(cdp_dl, "cdprobe_allreduce_push");
  cdp_arnvls = (ar_fn)dlsym(cdp_dl, "cdprobe_allreduce_nvls");
  cdp_mc = (mc_fn)dlsym(cdp_dl, "cdprobe_memcpy");
  cdp_cea = (cea_fn)dlsym(cdp_dl, "cdprobe_ce_alltoall");
  cdp_opt = (opt_fn)dlsym(cdp_dl, "cdprobe_set_option");
  cdp_links = (links_fn)dlsym(cdp_dl, "cdprobe_links");
  if (!cdp_open || !cdp_run || !cdp_close || !cdp_strerror || !cdp_last || !cdp_abi) return -2;
  return cdp_abi() == CDPROBE_ABI_VERSION ? 0 : -3;
}
static int cdp_call_open(const cdprobe_config_t* c, cdprobe_t** h) { return cdp_open(c, h); }
static int cdp_call_run(cdprobe_t* h, cdprobe_result_t* r) { return cdp_run(h, r); }
static void cdp_call_close(cdprobe_t* h) { cdp_close(h); }
static const char* cdp_call_strerror(int rc) { return cdp_strerror(rc); }
static const char* cdp_call_last(void) { return cdp_last(); }
static int cdp_has_diagnose(void) { return cdp_diag != NULL; }
static int cdp_call_diagnose(cdprobe_t* h, uint32_t op, uint32_t i, uint32_t j, uint32_t reader, cdprobe_diag_t* d) {
  return cdp_diag(h, op, i, j, reader, d);
}
static int cdp_has_latency(void) { return cdp_lat != NULL; }
static int cdp_call_latency(cdprobe_t* h, uint32_t hops, uint32_t reps, cdprobe_latency_t* l) {
  return cdp_lat(h, hops, reps, l);
}
static int cdp_has_pingpong(void) { return cdp_pp != NULL; }
static int cdp_call_pingpong(cdprobe_t* h, uint32_t trips, uint32_t reps, uint32_t fenced, cdprobe_pingpong_t* pp) {
  return cdp_pp(h, trips, reps, fenced, pp);
}
static int cdp_has_atomics(void) { return cdp_at != NULL; }
static int cdp_call_atomics(cdprobe_t* h, uint32_t kind, uint32_t ops, uint32_t reps, cdprobe_atomics_t* at) {
  return cdp_at(h, kind, ops, reps, at);
}
static int cdp_has_bwcurve(void) { return cdp_bw != NULL; }
static int cdp_call_bwcurve(cdprobe_t* h, uint32_t reps, cdprobe_bwcurve_t* bw) { return cdp_bw(h, reps, bw); }
static int cdp_has_allreduce(void) { return cdp_ar != NULL; }
static int cdp_call_allreduce(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* ar) { return cdp_ar(h, reps, ar); }
static int cdp_has_alltoall(void) { return cdp_a2a != NULL; }
static int cdp_call_alltoall(cdprobe_t* h, uint32_t reps, cdprobe_alltoall_t* aa) { return cdp_a2a(h, reps, aa); }
static int cdp_has_allreduce_twoshot(void) { return cdp_ar2 != NULL; }
static int cdp_call_allreduce_twoshot(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* ar) {
  return cdp_ar2(h, reps, ar);
}
static int cdp_has_allreduce_ll(void) { return cdp_arll != NULL; }
static int cdp_call_allreduce_ll(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* ar) { return cdp_arll(h, reps, ar); }
static int cdp_has_allreduce_ring(void) { return cdp_arring != NULL; }
static int cdp_call_allreduce_ring(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* ar) {
  return cdp_arring(h, reps, ar);
}
static int cdp_has_allreduce_push(void) { return cdp_arpush != NULL; }
static int cdp_call_allreduce_push(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* ar) {
  return cdp_arpush(h, reps, ar);
}
static int cdp_has_allreduce_nvls(void) { return cdp_arnvls != NULL; }
static int cdp_call_allreduce_nvls(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* ar) {
  return cdp_arnvls(h, reps, ar);
}
static int cdp_has_memcpy(void) { return cdp_mc != NULL; }
static int cdp_call_memcpy(cdprobe_t* h, uint32_t op, uint32_t reps, cdprobe_memcpy_t* mc) {
  return cdp_mc(h, op, reps, mc);
}
static int cdp_has_ce_alltoall(void) { return cdp_cea != NULL; }
static int cdp_call_ce_alltoall(cdprobe_t* h, uint32_t op, uint32_t reps, cdprobe_ce_alltoall_t* ca) {
  return cdp_cea(h, op, reps, ca);
}
static int cdp_has_set_option(void) { return cdp_opt != NULL; }
static int cdp_call_set_option(cdprobe_t* h, uint32_t option, uint64_t value) { return cdp_opt(h, option, value); }
static int cdp_has_links(void) { return cdp_links != NULL; }
static int cdp_call_links(cdprobe_t* h, cdprobe_links_t* l) { return cdp_links(h, l); }
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

	// OptLinkCounters (value 0/1, default 0) samples every local GPU's per-link NVLink counters around each Run,
	// for Links (CDPROBE_OPT_LINK_COUNTERS).
	OptLinkCounters = 27
)

// The error counters of LinkDevice.Errors, in order (CDPROBE_LINK_*).
var LinkCounterNames = [3]string{"replay", "recovery", "crc"}

// LinkDevice is one local GPU's row of Links (cdprobe_link_device_t).  Per-link slices have 18 entries, index = link.
type LinkDevice struct {
	Status                        int32       // 0 ok; CDPROBE_ERR_UNSUPPORTED: no NVLink fields; > 0: the failing nvmlReturn_t
	RankMask                      uint32      // ranks on this GPU
	UUID                          string
	LinkMask, LostMask, ErrorMask uint32      // enabled at the first sample; enabled then but not at the second; an error rose
	ExpectedTxKiB, ExpectedRxKiB  uint64      // payload the pass's plan moved to / from other GPUs
	TxKiB, RxKiB                  []uint64
	Errors                        [][3]uint64 // [link][replay, recovery, crc]
	FailedFields                  []uint32    // CDPROBE_LINK_FIELD_* bits
	RemoteBusID                   []string    // "" when NVML does not say
}

// Links is the per-link NVLink counter report of the last Run taken with OptLinkCounters on (cdprobe_links_t).
type Links struct {
	RunSeq   uint64 // 0: no sampled run yet
	SampleMs float64
	Devices  []LinkDevice
}

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

// DiagKinds names the classes of a bad word, indexed by CDPROBE_DIAG_*.
var DiagKinds = [5]string{"flip", "zero", "displaced", "stale", "foreign"}

// DiagSample is one bad word (cdprobe_diag_sample_t).
type DiagSample struct {
	Offset             uint64 // bytes from the region start
	Expected, Observed uint64
	Word               uint64 // displaced/stale/foreign: the pattern index that produced Observed
	RunSeq             uint64 // stale: the run that wrote it
	Kind               string // one of DiagKinds
	Rank               int    // whose pattern it is (-1 for flip/zero)
}

// Diagnosis is what Diagnose found in one cell's region (cdprobe_diag_t).
type Diagnosis struct {
	Op                     string // "read" or "write"
	Issuer, Target, Reader int
	RunSeq                 uint64
	Words                  uint64 // 64-bit words in the region
	BadWords, BadGranules  uint64
	ZeroWords              uint64
	FirstBad, LastBad      uint64    // byte offsets of the first / last bad word (meaningless when BadWords == 0)
	KindCount              [5]uint64 // indexed like DiagKinds
	BitFlips               [64]uint64 // flip words only: how often bit b differed
	Ms                     float64
	Samples                []DiagSample // the lowest-offset bad words, in offset order
}

// Latency is the dependent-load latency matrix of the local rows (cdprobe_latency_t).  Matrices are N x N
// row-major, [issuer*N + target]; the Ns* entries are 0 where a cell was not measured or its chase timed out.
type Latency struct {
	N                      int
	RowMask                uint32    // rows of this process's ranks
	Hops, Reps             int       // as applied
	RegionBytes            uint64    // bytes one chase ranges over
	Measured               []bool
	Status                 []int32   // 0 ok; CDPROBE_ERR_INTEGRITY; CDPROBE_ERR_TIMEOUT; else the mapping's status
	NsMin, NsMedian, NsMax []float32 // ns per hop over the timed reps
	Digest                 []uint64  // xor of every loaded word
	Ms                     float64
}

// PingPong is the signal round-trip matrix of the local rows (cdprobe_pingpong_t).  Matrices are N x N row-major,
// [initiator*N + target]; the Ns* entries are 0 where a cell was not measured or its round trips timed out.
type PingPong struct {
	N                      int
	RowMask                uint32    // rows of this process's ranks
	Trips, Reps            int       // as applied
	Fenced                 bool      // a fence.sys before every store
	CallSeq                uint64    // 1-based count of PingPong calls, equal in every process
	Measured               []bool
	Status                 []int32   // 0 ok; CDPROBE_ERR_INTEGRITY; CDPROBE_ERR_TIMEOUT; else the pair's mapping status
	NsMin, NsMedian, NsMax []float32 // ns per round trip over the timed reps
	Digest                 []uint64  // xor of every echo word the initiator received
	Ms                     float64
}

// Kinds of Atomics (CDPROBE_ATOMIC_*).
const (
	AtomicFetchAdd  = 0 // one lane: a dependent atom.add chain
	AtomicCAS       = 1 // one lane: a dependent atom.cas chain, every CAS must succeed
	AtomicContended = 2 // 32 lanes of one warp: fetch-add chains on the same word
)

// Atomics is the remote-atomics matrix of the local rows (cdprobe_atomics_t).  Matrices are N x N row-major,
// [issuer*N + target]; the Ns* entries are 0 where a cell was not measured or timed out.
type Atomics struct {
	N                      int
	RowMask                uint32    // rows of this process's ranks
	Kind                   int       // AtomicFetchAdd, AtomicCAS or AtomicContended
	Ops, Reps, Lanes       int       // as applied; ops per lane
	CallSeq                uint64    // 1-based count of Atomics calls on this handle
	Native                 []uint8   // 1 native atomics (or same device); 0 none reported: not run; 2 peer device not visible
	Measured               []bool
	Status                 []int32   // 0 ok; CDPROBE_ERR_INTEGRITY; CDPROBE_ERR_TIMEOUT; CDPROBE_ERR_UNSUPPORTED; else the mapping's status
	NsMin, NsMedian, NsMax []float32 // ns per atomic over the timed reps
	Digest                 []uint64  // xor of every value the atomics returned
	Ms                     float64
}

// BwCurve is the bandwidth-versus-size curve of the local rows (cdprobe_bwcurve_t).  Per-cell slices are N x N
// row-major, [issuer*N + target]; the per-size ones hold one entry per Sizes element, and every timing is 0 where a
// cell was not measured or timed out.
type BwCurve struct {
	N                      int
	RowMask                uint32      // rows of this process's ranks
	Reps                   int         // timed reps per size, as applied
	Path                   int         // the read data path (CDPROBE_OPT_PATH)
	CallSeq                uint64      // 1-based count of BwCurve calls on this handle, equal in every process
	Sizes                  []uint64    // bytes read per rep
	Measured               []bool
	Status                 []int32     // 0 ok; CDPROBE_ERR_INTEGRITY; CDPROBE_ERR_TIMEOUT; else the mapping's status
	BadSizes               []uint32    // bit k: a rep of Sizes[k] read a checksum other than the pattern's
	T0Ns, PeakGBps         []float32   // median ns of the smallest size; max over sizes of size / median ns
	HalfBytes              []uint64    // the smallest size reaching half the peak
	NsMin, NsMedian, NsMax [][]float32 // [cell][size]: ns per rep over the timed reps
	Sum, Xr                [][]uint64  // [cell][size]: (S, X) of the last timed rep
	Ms                     float64
}

// AllReduce is the one-shot all-reduce of the local rows (cdprobe_allreduce_t), or the two-shot's (AllReduceTwoShot),
// the low-latency one's (AllReduceLL), the ring's (AllReduceRing), the push one's (AllReducePush) or the multicast one's
// (AllReduceNVLS).
// Every slice is indexed by rank; the per-size ones hold one entry per Sizes element, and every timing is 0 where a
// rank was not measured or timed out.
type AllReduce struct {
	N                      int
	RowMask                uint32      // rows of this process's ranks
	Reps                   int         // timed reps per size, as applied
	Path                   int         // the read data path (CDPROBE_OPT_PATH)
	CallSeq                uint64      // 1-based count of AllReduce calls on this handle, equal in every process
	Sizes                  []uint64    // bytes per input and of the output per rep
	Measured               []bool
	Status                 []int32     // 0 ok; CDPROBE_ERR_INTEGRITY; CDPROBE_ERR_TIMEOUT; else the first down cell's status
	BadSizes               []uint32    // bit k: Sizes[k] failed the checksum or the word check
	T0Ns, PeakGBps         []float32   // median ns of the smallest size; max over sizes of size / median ns (algbw)
	HalfBytes              []uint64    // the smallest size reaching half the peak
	NsMin, NsMedian, NsMax [][]float32 // [rank][size]: ns per rep over the timed reps
	Sum, Xr                [][]uint64  // [rank][size]: (S, X) of the output of the last timed rep
	BadWords, FirstBad     [][]uint64  // [rank][size]: the word check; FirstBad is MaxUint64 when clean
	Ms                     float64
}

// AllToAll is the one-shot all-to-all (cdprobe_alltoall_t).  Per-rank slices are indexed by the sender and filled for
// this process's ranks; per-cell ones are [sender][receiver] and filled for the cells this process's ranks receive.  The
// per-size ones hold one entry per Sizes element; every timing is 0 where a rank was not measured or timed out.
type AllToAll struct {
	N                      int
	RowMask                uint32      // this process's ranks
	Reps                   int         // timed reps per size, as applied
	Path                   int         // the write data path (CDPROBE_OPT_PATH)
	CallSeq                uint64      // 1-based count of AllToAll calls on this handle, equal in every process
	AreaBytes              uint64      // this rank's exchange area
	Sizes                  []uint64    // bytes per block per rep
	Measured               []bool      // [rank]
	Status                 []int32     // [rank]: 0 ok; CDPROBE_ERR_TIMEOUT
	Blocks                 []uint32    // [rank]: blocks pushed per rep
	T0Ns, PeakGBps         []float32   // [rank]: median ns of the smallest size; max over sizes of egress GB/s
	HalfBytes              []uint64    // [rank]: the smallest size reaching half the peak
	NsMin, NsMedian, NsMax [][]float32 // [rank][size]: ns per rep over the timed reps
	CellMeasured           [][]bool    // [sender][receiver]
	CellStatus             [][]int32   // [sender][receiver]: 0 ok; CDPROBE_ERR_INTEGRITY; CDPROBE_ERR_TIMEOUT; else the mapping status
	BadSizes               [][]uint32  // [sender][receiver]: bit k: Sizes[k] delivered a bad word
	BadWords, FirstBad     [][][]uint64 // [sender][receiver][size]: the word check; FirstBad is MaxUint64 when clean
	Sum, Xr                [][][]uint64 // [sender][receiver][size]: (S, X) of the block in the last timed rep
	Ms                     float64
}

// Memcpy is the copy-engine bandwidth curve of the local rows (cdprobe_memcpy_t), pulled (Op CDPROBE_OP_READ) or pushed
// (CDPROBE_OP_WRITE).  Cells are [issuer * N + target], as in BwCurve; the per-size slices hold one entry per Sizes
// element.
type Memcpy struct {
	N                      int
	RowMask                uint32      // rows of this process's ranks
	Reps                   int         // timed reps per size, as applied
	Op                     uint32      // CDPROBE_OP_READ (pull) or CDPROBE_OP_WRITE (push)
	CallSeq                uint64      // 1-based count of Memcpy calls on this handle, equal in every process
	AreaBytes              uint64      // this rank's exchange area, where the copies land
	Sizes                  []uint64    // bytes copied per rep
	Measured               []bool
	Status                 []int32     // 0 ok; CDPROBE_ERR_INTEGRITY; CDPROBE_ERR_TIMEOUT; else the mapping's status
	BadSizes               []uint32    // bit k: a rep of Sizes[k] landed a bad word or checksum
	T0Ns, PeakGBps         []float32   // median ns of the smallest size; max over sizes of size / median ns
	HalfBytes              []uint64    // the smallest size reaching half the peak
	NsMin, NsMedian, NsMax [][]float32 // [cell][size]: ns per copy over the timed reps, by CUDA events
	Sum, Xr                [][]uint64  // [cell][size]: (S, X) of the destination in the last timed rep
	BadWords, FirstBad     [][]uint64  // [cell][size]: the word check over every rep; FirstBad is MaxUint64 when clean
	Ms                     float64
}

// CeAllToAll is the copy-engine all-to-all (cdprobe_ce_alltoall_t), pulled (Op CDPROBE_OP_READ) or pushed
// (CDPROBE_OP_WRITE).  Per-rank slices are filled for this process's ranks; per-cell ones are [issuer][target]: the
// check fields for the blocks this process's ranks own (the issuer's on a pull, the target's on a push), CopyNsMedian
// for the cells they issue.  The per-size ones hold one entry per Sizes element; every timing is 0 where a rank did
// not run.
type CeAllToAll struct {
	N                      int
	RowMask                uint32       // this process's ranks
	Reps                   int          // timed reps per size, as applied
	Op                     uint32       // CDPROBE_OP_READ (pull) or CDPROBE_OP_WRITE (push)
	CallSeq                uint64       // 1-based count of CeAllToAll calls on this handle, equal in every process
	AreaBytes              uint64       // this rank's exchange area, where the blocks land
	Sizes                  []uint64     // bytes per block per rep
	Measured               []bool       // [rank]
	Status                 []int32      // [rank]: 0 ok; else the status of the domain's first down mapping
	Blocks                 []uint32     // [rank]: blocks copied per rep (the cells it issues)
	T0Ns, PeakGBps         []float32    // [rank]: median ns of the smallest size; max over sizes of blocks x size / ns
	HalfBytes              []uint64     // [rank]: the smallest size reaching half the peak
	NsMin, NsMedian, NsMax [][]float32  // [rank][size]: ns per rep, release to every block landed, over the timed reps
	CellMeasured           [][]bool     // [issuer][target]
	CellStatus             [][]int32    // [issuer][target]: 0 ok; CDPROBE_ERR_INTEGRITY; CDPROBE_ERR_TIMEOUT; else a mapping status
	BadSizes               [][]uint32   // [issuer][target]: bit k: Sizes[k] landed a bad word or checksum
	CopyNsMedian           [][][]float32 // [issuer][target][size]: median ns of the cell's copy, by CUDA events
	BadWords, FirstBad     [][][]uint64 // [issuer][target][size]: the word check; FirstBad is MaxUint64 when clean
	Sum, Xr                [][][]uint64 // [issuer][target][size]: (S, X) of the block in the last timed rep
	Ms                     float64
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

// Diagnose re-reads cell (op, issuer, target) of the last Run on reader's GPU and diffs it word for word against
// the pattern: reader = issuer is what crossed the fabric, reader = target what is at rest.  ErrUnsupported when
// the library predates cdprobe_diagnose.
func (p *Probe) Diagnose(op uint32, issuer, target, reader int) (Diagnosis, error) {
	if C.cdp_has_diagnose() == 0 {
		return Diagnosis{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_diagnose", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	var d C.cdprobe_diag_t
	rc := C.cdp_call_diagnose(p.h, C.uint32_t(op), C.uint32_t(issuer), C.uint32_t(target), C.uint32_t(reader), &d)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_diagnose: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return Diagnosis{}, err
	}
	out := Diagnosis{Op: "read", Issuer: int(d.issuer), Target: int(d.target), Reader: int(d.reader),
		RunSeq: uint64(d.run_seq), Words: uint64(d.bytes) / 8, BadWords: uint64(d.bad_words),
		BadGranules: uint64(d.bad_granules), ZeroWords: uint64(d.zero_words),
		FirstBad: uint64(d.first_bad), LastBad: uint64(d.last_bad), Ms: float64(d.ms)}
	if d.op == C.CDPROBE_OP_WRITE {
		out.Op = "write"
	}
	for k := range out.KindCount {
		out.KindCount[k] = uint64(d.kind_count[k])
	}
	for b := range out.BitFlips {
		out.BitFlips[b] = uint64(d.bit_flips[b])
	}
	for k := 0; k < int(d.n_samples); k++ {
		s := d.sample[k]
		out.Samples = append(out.Samples, DiagSample{Offset: uint64(s.offset), Expected: uint64(s.expected),
			Observed: uint64(s.observed), Word: uint64(s.word), RunSeq: uint64(s.run_seq),
			Kind: DiagKinds[int(s.kind)%len(DiagKinds)], Rank: int(s.rank)})
	}
	return out, nil
}

// Latency chases hops dependent 8-byte loads from every local issuer through its mapping of each target's source
// slice and reports ns per hop (0, 0: 1024 hops, 8 timed reps).  One-sided: only the local rows are filled.
// ErrUnsupported when the library predates cdprobe_latency.
func (p *Probe) Latency(hops, reps int) (Latency, error) {
	if C.cdp_has_latency() == 0 {
		return Latency{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_latency", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	var lt C.cdprobe_latency_t
	rc := C.cdp_call_latency(p.h, C.uint32_t(hops), C.uint32_t(reps), &lt)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_latency: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return Latency{}, err
	}
	n := int(lt.n)
	out := Latency{N: n, RowMask: uint32(lt.row_mask), Hops: int(lt.hops), Reps: int(lt.reps),
		RegionBytes: uint64(lt.region_bytes), Ms: float64(lt.ms)}
	out.Measured = make([]bool, n*n)
	out.Status = make([]int32, n*n)
	out.NsMin = make([]float32, n*n)
	out.NsMedian = make([]float32, n*n)
	out.NsMax = make([]float32, n*n)
	out.Digest = make([]uint64, n*n)
	for i := 0; i < n; i++ {
		for j := 0; j < n; j++ {
			k := i*C.CDPROBE_MAX_GPUS + j
			out.Measured[i*n+j] = lt.measured[k] != 0
			out.Status[i*n+j] = int32(lt.status[k])
			out.NsMin[i*n+j] = float32(lt.ns_min[k])
			out.NsMedian[i*n+j] = float32(lt.ns_median[k])
			out.NsMax[i*n+j] = float32(lt.ns_max[k])
			out.Digest[i*n+j] = uint64(lt.digest[k])
		}
	}
	return out, nil
}

// PingPong times the barrier's cross-GPU signal as a round trip over every pair of the tournament and reports ns
// per round trip (0, 0: 256 round trips, 8 timed reps); fenced puts a fence.sys before every store.  Collective when
// the domain spans processes: every process calls it with the same arguments and gets its own rows.
// ErrUnsupported when the library predates cdprobe_pingpong.
func (p *Probe) PingPong(trips, reps int, fenced bool) (PingPong, error) {
	if C.cdp_has_pingpong() == 0 {
		return PingPong{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_pingpong", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	f := 0
	if fenced {
		f = 1
	}
	var pp C.cdprobe_pingpong_t
	rc := C.cdp_call_pingpong(p.h, C.uint32_t(trips), C.uint32_t(reps), C.uint32_t(f), &pp)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_pingpong: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return PingPong{}, err
	}
	n := int(pp.n)
	out := PingPong{N: n, RowMask: uint32(pp.row_mask), Trips: int(pp.trips), Reps: int(pp.reps),
		Fenced: pp.fenced != 0, CallSeq: uint64(pp.call_seq), Ms: float64(pp.ms)}
	out.Measured = make([]bool, n*n)
	out.Status = make([]int32, n*n)
	out.NsMin = make([]float32, n*n)
	out.NsMedian = make([]float32, n*n)
	out.NsMax = make([]float32, n*n)
	out.Digest = make([]uint64, n*n)
	for i := 0; i < n; i++ {
		for j := 0; j < n; j++ {
			k := i*C.CDPROBE_MAX_GPUS + j
			out.Measured[i*n+j] = pp.measured[k] != 0
			out.Status[i*n+j] = int32(pp.status[k])
			out.NsMin[i*n+j] = float32(pp.ns_min[k])
			out.NsMedian[i*n+j] = float32(pp.ns_median[k])
			out.NsMax[i*n+j] = float32(pp.ns_max[k])
			out.Digest[i*n+j] = uint64(pp.digest[k])
		}
	}
	return out, nil
}

// Atomics runs system-scope 64-bit atomics from every local issuer on each cell's own word in the target's memory
// and reports ns per atomic (ops, reps 0, 0: 1024 ops per lane, 8 timed reps); every returned value is checked.
// One-sided: only the local rows are filled and no process waits on another.  ErrUnsupported when the library
// predates cdprobe_atomics.
func (p *Probe) Atomics(kind, ops, reps int) (Atomics, error) {
	if C.cdp_has_atomics() == 0 {
		return Atomics{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_atomics", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	var at C.cdprobe_atomics_t
	rc := C.cdp_call_atomics(p.h, C.uint32_t(kind), C.uint32_t(ops), C.uint32_t(reps), &at)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_atomics: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return Atomics{}, err
	}
	n := int(at.n)
	out := Atomics{N: n, RowMask: uint32(at.row_mask), Kind: int(at.kind), Ops: int(at.ops), Reps: int(at.reps),
		Lanes: int(at.lanes), CallSeq: uint64(at.call_seq), Ms: float64(at.ms)}
	out.Native = make([]uint8, n*n)
	out.Measured = make([]bool, n*n)
	out.Status = make([]int32, n*n)
	out.NsMin = make([]float32, n*n)
	out.NsMedian = make([]float32, n*n)
	out.NsMax = make([]float32, n*n)
	out.Digest = make([]uint64, n*n)
	for i := 0; i < n; i++ {
		for j := 0; j < n; j++ {
			k := i*C.CDPROBE_MAX_GPUS + j
			out.Native[i*n+j] = uint8(at.native[k])
			out.Measured[i*n+j] = at.measured[k] != 0
			out.Status[i*n+j] = int32(at.status[k])
			out.NsMin[i*n+j] = float32(at.ns_min[k])
			out.NsMedian[i*n+j] = float32(at.ns_median[k])
			out.NsMax[i*n+j] = float32(at.ns_max[k])
			out.Digest[i*n+j] = uint64(at.digest[k])
		}
	}
	return out, nil
}

// BwCurve reads growing prefixes of every local issuer's source slices on the probe's read path and grid, in the
// tournament's rounds, and reports ns per rep for each size (reps 0: 8 timed reps); every rep's checksum is checked.
// Collective when the domain spans processes.  ErrUnsupported when the library predates cdprobe_bwcurve.
func (p *Probe) BwCurve(reps int) (BwCurve, error) {
	if C.cdp_has_bwcurve() == 0 {
		return BwCurve{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_bwcurve", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	bw := new(C.cdprobe_bwcurve_t)
	rc := C.cdp_call_bwcurve(p.h, C.uint32_t(reps), bw)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_bwcurve: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return BwCurve{}, err
	}
	n, ns := int(bw.n), int(bw.n_sizes)
	out := BwCurve{N: n, RowMask: uint32(bw.row_mask), Reps: int(bw.reps), Path: int(bw.path),
		CallSeq: uint64(bw.call_seq), Ms: float64(bw.ms)}
	out.Sizes = make([]uint64, ns)
	for s := 0; s < ns; s++ {
		out.Sizes[s] = uint64(bw.size[s])
	}
	out.Measured = make([]bool, n*n)
	out.Status = make([]int32, n*n)
	out.BadSizes = make([]uint32, n*n)
	out.T0Ns = make([]float32, n*n)
	out.PeakGBps = make([]float32, n*n)
	out.HalfBytes = make([]uint64, n*n)
	out.NsMin = make([][]float32, n*n)
	out.NsMedian = make([][]float32, n*n)
	out.NsMax = make([][]float32, n*n)
	out.Sum = make([][]uint64, n*n)
	out.Xr = make([][]uint64, n*n)
	for i := 0; i < n; i++ {
		for j := 0; j < n; j++ {
			k, c := i*C.CDPROBE_MAX_GPUS+j, i*n+j
			out.Measured[c] = bw.measured[k] != 0
			out.Status[c] = int32(bw.status[k])
			out.BadSizes[c] = uint32(bw.bad_sizes[k])
			out.T0Ns[c] = float32(bw.t0_ns[k])
			out.PeakGBps[c] = float32(bw.peak_gbps[k])
			out.HalfBytes[c] = uint64(bw.half_bytes[k])
			out.NsMin[c], out.NsMedian[c], out.NsMax[c] = make([]float32, ns), make([]float32, ns), make([]float32, ns)
			out.Sum[c], out.Xr[c] = make([]uint64, ns), make([]uint64, ns)
			for s := 0; s < ns; s++ {
				out.NsMin[c][s] = float32(bw.ns_min[k][s])
				out.NsMedian[c][s] = float32(bw.ns_median[k][s])
				out.NsMax[c][s] = float32(bw.ns_max[k][s])
				out.Sum[c][s] = uint64(bw.sum[k][s])
				out.Xr[c][s] = uint64(bw.xr[k][s])
			}
		}
	}
	return out, nil
}

// AllReduce runs the one-shot all-reduce of every rank's source buffer on every rank at once, at each size of the
// bwcurve ladder, and reports ns per rep for each size (reps 0: 8 timed reps); every rep's checksum and the last rep's
// every word are checked.  Collective when the domain spans processes.  ErrUnsupported when the library predates
// cdprobe_allreduce.
func (p *Probe) AllReduce(reps int) (AllReduce, error) {
	if C.cdp_has_allreduce() == 0 {
		return AllReduce{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_allreduce", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	ar := new(C.cdprobe_allreduce_t)
	rc := C.cdp_call_allreduce(p.h, C.uint32_t(reps), ar)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_allreduce: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return AllReduce{}, err
	}
	return allReduceOf(ar), nil
}

// AllReduceTwoShot runs the two-shot all-reduce of every rank's source buffer on every rank at once, a reduce-scatter
// then a pushed all-gather, at each size of the bwcurve ladder, and reports ns per rep for each size (reps 0: 8 timed
// reps).  Every rep's output is read back, checked word for word and cleared: BadWords and FirstBad cover every rep.
// PeakGBps is the algorithm bandwidth; the nccl-tests bus bandwidth is PeakGBps x 2(N - 1)/N.  Collective when the
// domain spans processes.  ErrUnsupported when the library predates cdprobe_allreduce_twoshot.
func (p *Probe) AllReduceTwoShot(reps int) (AllReduce, error) {
	if C.cdp_has_allreduce_twoshot() == 0 {
		return AllReduce{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_allreduce_twoshot", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	ar := new(C.cdprobe_allreduce_t)
	rc := C.cdp_call_allreduce_twoshot(p.h, C.uint32_t(reps), ar)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_allreduce_twoshot: %s: %s", C.GoString(C.cdp_call_strerror(rc)),
			C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return AllReduce{}, err
	}
	return allReduceOf(ar), nil
}

// AllReduceLL runs the low-latency all-reduce of every rank's source buffer on every rank at once: every input word
// travels to every peer in a flag-carrying 16-byte packet, with no barrier or fence per rep, at each size of the LL
// ladder (the bwcurve ladder up to 1 MiB), and reports ns per rep for each size (reps 0: 8 timed reps), timed from
// the end of the rank's previous rep.  Path is CDPROBE_ALLREDUCE_PATH_LL.  Collective when the domain spans processes.
// ErrUnsupported when the library predates cdprobe_allreduce_ll.
func (p *Probe) AllReduceLL(reps int) (AllReduce, error) {
	if C.cdp_has_allreduce_ll() == 0 {
		return AllReduce{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_allreduce_ll", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	ar := new(C.cdprobe_allreduce_t)
	rc := C.cdp_call_allreduce_ll(p.h, C.uint32_t(reps), ar)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_allreduce_ll: %s: %s", C.GoString(C.cdp_call_strerror(rc)),
			C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return AllReduce{}, err
	}
	ll := allReduceOf(ar)
	return ll, nil
}

// AllReduceRing runs the ring all-reduce of every rank's source buffer on every rank at once: each rank passes every
// 8 KiB unit to the next rank under its own flag, 2(N - 1) steps of reduce-scatter and all-gather with no barrier or
// fence between them, at each size of the bwcurve ladder, and reports ns per rep for each size (reps 0: 8 timed reps),
// timed from the rep's opening barrier to the moment the rank's output is complete.  Path is
// CDPROBE_ALLREDUCE_PATH_RING.  Collective when the domain spans processes.  ErrUnsupported when the library predates
// cdprobe_allreduce_ring.
func (p *Probe) AllReduceRing(reps int) (AllReduce, error) {
	if C.cdp_has_allreduce_ring() == 0 {
		return AllReduce{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_allreduce_ring", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	res := new(C.cdprobe_allreduce_t)
	rc := C.cdp_call_allreduce_ring(p.h, C.uint32_t(reps), res)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_allreduce_ring: %s: %s", C.GoString(C.cdp_call_strerror(rc)),
			C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return AllReduce{}, err
	}
	ring := allReduceOf(res)
	return ring, nil
}

// AllReducePush runs the push all-reduce of every rank's source buffer on every rank at once, every byte moved as a
// write: each rank reduces every 8 KiB unit of its input into the unit's owner (bulk reductions on the TMA path,
// red.global per word on ld/st), then each owner pushes its finished chunk to every peer, at each size of the bwcurve
// ladder, and reports ns per rep for each size (reps 0: 8 timed reps), timed from the rep's opening barrier to its
// closing barrier.  Path is the handle's data path.  Collective when the domain spans processes.  ErrUnsupported when
// the library predates cdprobe_allreduce_push.
func (p *Probe) AllReducePush(reps int) (AllReduce, error) {
	if C.cdp_has_allreduce_push() == 0 {
		return AllReduce{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_allreduce_push", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	res := new(C.cdprobe_allreduce_t)
	rc := C.cdp_call_allreduce_push(p.h, C.uint32_t(reps), res)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_allreduce_push: %s: %s", C.GoString(C.cdp_call_strerror(rc)),
			C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return AllReduce{}, err
	}
	push := allReduceOf(res)
	return push, nil
}

// AllReduceNVLS runs the multicast (NVLS) all-reduce of every rank's source buffer on every rank at once: each rank
// sums its chunk of 8 KiB units with multimem.ld_reduce through one multicast object that spans the domain and stores
// each sum to every rank with one multimem.st, at each size of the bwcurve ladder, and reports ns per rep for each size
// (reps 0: 8 timed reps), timed from the rep's opening barrier to its closing barrier.  Path is
// CDPROBE_ALLREDUCE_PATH_NVLS.  Rows are CDPROBE_ERR_UNSUPPORTED, with nothing run, when a device or the driver lacks
// multicast or two ranks share a device.  Collective when the domain spans processes.  ErrUnsupported when the library
// predates cdprobe_allreduce_nvls.
func (p *Probe) AllReduceNVLS(reps int) (AllReduce, error) {
	if C.cdp_has_allreduce_nvls() == 0 {
		return AllReduce{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_allreduce_nvls", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	res := new(C.cdprobe_allreduce_t)
	rc := C.cdp_call_allreduce_nvls(p.h, C.uint32_t(reps), res)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_allreduce_nvls: %s: %s", C.GoString(C.cdp_call_strerror(rc)),
			C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return AllReduce{}, err
	}
	nvls := allReduceOf(res)
	return nvls, nil
}

// allReduceOf copies a cdprobe_allreduce_t into an AllReduce.
func allReduceOf(ar *C.cdprobe_allreduce_t) AllReduce {
	n, ns := int(ar.n), int(ar.n_sizes)
	out := AllReduce{N: n, RowMask: uint32(ar.row_mask), Reps: int(ar.reps), Path: int(ar.path),
		CallSeq: uint64(ar.call_seq), Ms: float64(ar.ms)}
	out.Sizes = make([]uint64, ns)
	for s := 0; s < ns; s++ {
		out.Sizes[s] = uint64(ar.size[s])
	}
	out.Measured = make([]bool, n)
	out.Status = make([]int32, n)
	out.BadSizes = make([]uint32, n)
	out.T0Ns = make([]float32, n)
	out.PeakGBps = make([]float32, n)
	out.HalfBytes = make([]uint64, n)
	out.NsMin, out.NsMedian, out.NsMax = make([][]float32, n), make([][]float32, n), make([][]float32, n)
	out.Sum, out.Xr = make([][]uint64, n), make([][]uint64, n)
	out.BadWords, out.FirstBad = make([][]uint64, n), make([][]uint64, n)
	for r := 0; r < n; r++ {
		out.Measured[r] = ar.measured[r] != 0
		out.Status[r] = int32(ar.status[r])
		out.BadSizes[r] = uint32(ar.bad_sizes[r])
		out.T0Ns[r] = float32(ar.t0_ns[r])
		out.PeakGBps[r] = float32(ar.peak_gbps[r])
		out.HalfBytes[r] = uint64(ar.half_bytes[r])
		out.NsMin[r], out.NsMedian[r], out.NsMax[r] = make([]float32, ns), make([]float32, ns), make([]float32, ns)
		out.Sum[r], out.Xr[r] = make([]uint64, ns), make([]uint64, ns)
		out.BadWords[r], out.FirstBad[r] = make([]uint64, ns), make([]uint64, ns)
		for s := 0; s < ns; s++ {
			out.NsMin[r][s] = float32(ar.ns_min[r][s])
			out.NsMedian[r][s] = float32(ar.ns_median[r][s])
			out.NsMax[r][s] = float32(ar.ns_max[r][s])
			out.Sum[r][s] = uint64(ar.sum[r][s])
			out.Xr[r][s] = uint64(ar.xr[r][s])
			out.BadWords[r][s] = uint64(ar.bad_words[r][s])
			out.FirstBad[r][s] = uint64(ar.first_bad[r][s])
		}
	}
	return out
}

// AllToAll runs the one-shot all-to-all: every rank pushes a block to every peer at once, at each size of the bwcurve
// ladder, and every receiver checks every word (reps 0: 8 timed reps).  Collective when the domain spans processes.
// ErrUnsupported when the library predates cdprobe_alltoall.
func (p *Probe) AllToAll(reps int) (AllToAll, error) {
	if C.cdp_has_alltoall() == 0 {
		return AllToAll{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_alltoall", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	aa := new(C.cdprobe_alltoall_t)
	rc := C.cdp_call_alltoall(p.h, C.uint32_t(reps), aa)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_alltoall: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return AllToAll{}, err
	}
	n, ns := int(aa.n), int(aa.n_sizes)
	out := AllToAll{N: n, RowMask: uint32(aa.row_mask), Reps: int(aa.reps), Path: int(aa.path),
		CallSeq: uint64(aa.call_seq), AreaBytes: uint64(aa.area_bytes), Ms: float64(aa.ms)}
	out.Sizes = make([]uint64, ns)
	for s := 0; s < ns; s++ {
		out.Sizes[s] = uint64(aa.size[s])
	}
	out.Measured, out.Status, out.Blocks = make([]bool, n), make([]int32, n), make([]uint32, n)
	out.T0Ns, out.PeakGBps, out.HalfBytes = make([]float32, n), make([]float32, n), make([]uint64, n)
	out.NsMin, out.NsMedian, out.NsMax = make([][]float32, n), make([][]float32, n), make([][]float32, n)
	out.CellMeasured, out.CellStatus, out.BadSizes = make([][]bool, n), make([][]int32, n), make([][]uint32, n)
	out.BadWords, out.FirstBad = make([][][]uint64, n), make([][][]uint64, n)
	out.Sum, out.Xr = make([][][]uint64, n), make([][][]uint64, n)
	for r := 0; r < n; r++ {
		out.Measured[r] = aa.measured[r] != 0
		out.Status[r] = int32(aa.status[r])
		out.Blocks[r] = uint32(aa.blocks[r])
		out.T0Ns[r] = float32(aa.t0_ns[r])
		out.PeakGBps[r] = float32(aa.peak_gbps[r])
		out.HalfBytes[r] = uint64(aa.half_bytes[r])
		out.NsMin[r], out.NsMedian[r], out.NsMax[r] = make([]float32, ns), make([]float32, ns), make([]float32, ns)
		for s := 0; s < ns; s++ {
			out.NsMin[r][s] = float32(aa.ns_min[r][s])
			out.NsMedian[r][s] = float32(aa.ns_median[r][s])
			out.NsMax[r][s] = float32(aa.ns_max[r][s])
		}
		out.CellMeasured[r], out.CellStatus[r], out.BadSizes[r] = make([]bool, n), make([]int32, n), make([]uint32, n)
		out.BadWords[r], out.FirstBad[r] = make([][]uint64, n), make([][]uint64, n)
		out.Sum[r], out.Xr[r] = make([][]uint64, n), make([][]uint64, n)
		for d := 0; d < n; d++ {
			c := r*C.CDPROBE_MAX_GPUS + d
			out.CellMeasured[r][d] = aa.cell_measured[c] != 0
			out.CellStatus[r][d] = int32(aa.cell_status[c])
			out.BadSizes[r][d] = uint32(aa.bad_sizes[c])
			out.BadWords[r][d], out.FirstBad[r][d] = make([]uint64, ns), make([]uint64, ns)
			out.Sum[r][d], out.Xr[r][d] = make([]uint64, ns), make([]uint64, ns)
			for s := 0; s < ns; s++ {
				out.BadWords[r][d][s] = uint64(aa.bad_words[c][s])
				out.FirstBad[r][d][s] = uint64(aa.first_bad[c][s])
				out.Sum[r][d][s] = uint64(aa.sum[c][s])
				out.Xr[r][d][s] = uint64(aa.xr[c][s])
			}
		}
	}
	return out, nil
}

// Memcpy runs the copy-engine bandwidth curve: cudaMemcpyAsync of each size of the bwcurve ladder per cell, pulled from
// the target into the issuer's exchange area (op CDPROBE_OP_READ) or pushed into the target's (CDPROBE_OP_WRITE), timed
// by CUDA events, every landed word checked (reps 0: 8 timed reps).  Collective when the domain spans processes.
// ErrUnsupported when the library predates cdprobe_memcpy.
func (p *Probe) Memcpy(op uint32, reps int) (Memcpy, error) {
	if C.cdp_has_memcpy() == 0 {
		return Memcpy{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_memcpy", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	mc := new(C.cdprobe_memcpy_t)
	rc := C.cdp_call_memcpy(p.h, C.uint32_t(op), C.uint32_t(reps), mc)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_memcpy: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
		if rc == C.CDPROBE_ERR_STATE {
			err = fmt.Errorf("%w: %v", ErrState, err)
		}
		return Memcpy{}, err
	}
	n, ns := int(mc.n), int(mc.n_sizes)
	out := Memcpy{N: n, RowMask: uint32(mc.row_mask), Reps: int(mc.reps), Op: uint32(mc.op),
		CallSeq: uint64(mc.call_seq), AreaBytes: uint64(mc.area_bytes), Ms: float64(mc.ms)}
	out.Sizes = make([]uint64, ns)
	for s := 0; s < ns; s++ {
		out.Sizes[s] = uint64(mc.size[s])
	}
	out.Measured, out.Status, out.BadSizes = make([]bool, n*n), make([]int32, n*n), make([]uint32, n*n)
	out.T0Ns, out.PeakGBps, out.HalfBytes = make([]float32, n*n), make([]float32, n*n), make([]uint64, n*n)
	out.NsMin, out.NsMedian, out.NsMax = make([][]float32, n*n), make([][]float32, n*n), make([][]float32, n*n)
	out.Sum, out.Xr = make([][]uint64, n*n), make([][]uint64, n*n)
	out.BadWords, out.FirstBad = make([][]uint64, n*n), make([][]uint64, n*n)
	for i := 0; i < n; i++ {
		for j := 0; j < n; j++ {
			k, c := i*C.CDPROBE_MAX_GPUS+j, i*n+j
			out.Measured[c] = mc.measured[k] != 0
			out.Status[c] = int32(mc.status[k])
			out.BadSizes[c] = uint32(mc.bad_sizes[k])
			out.T0Ns[c] = float32(mc.t0_ns[k])
			out.PeakGBps[c] = float32(mc.peak_gbps[k])
			out.HalfBytes[c] = uint64(mc.half_bytes[k])
			out.NsMin[c], out.NsMedian[c], out.NsMax[c] = make([]float32, ns), make([]float32, ns), make([]float32, ns)
			out.Sum[c], out.Xr[c] = make([]uint64, ns), make([]uint64, ns)
			out.BadWords[c], out.FirstBad[c] = make([]uint64, ns), make([]uint64, ns)
			for s := 0; s < ns; s++ {
				out.NsMin[c][s] = float32(mc.ns_min[k][s])
				out.NsMedian[c][s] = float32(mc.ns_median[k][s])
				out.NsMax[c][s] = float32(mc.ns_max[k][s])
				out.Sum[c][s] = uint64(mc.sum[k][s])
				out.Xr[c][s] = uint64(mc.xr[k][s])
				out.BadWords[c][s] = uint64(mc.bad_words[k][s])
				out.FirstBad[c][s] = uint64(mc.first_bad[k][s])
			}
		}
	}
	return out, nil
}

// CeAllToAll runs the copy-engine all-to-all: in every rep every cell copies its block at once on a copy stream of its
// own, pulled (op CDPROBE_OP_READ) or pushed (CDPROBE_OP_WRITE), the ranks signalling each other with stream memory
// operations, at each size of the bwcurve ladder; the owner of every block checks every word (reps 0: 8 timed reps).
// Collective when the domain spans processes.  ErrUnsupported when the library predates cdprobe_ce_alltoall.
func (p *Probe) CeAllToAll(op uint32, reps int) (CeAllToAll, error) {
	if C.cdp_has_ce_alltoall() == 0 {
		return CeAllToAll{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_ce_alltoall", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	ca := new(C.cdprobe_ce_alltoall_t)
	rc := C.cdp_call_ce_alltoall(p.h, C.uint32_t(op), C.uint32_t(reps), ca)
	if rc != 0 {
		err := fmt.Errorf("cdprobe_ce_alltoall: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
		switch rc {
		case C.CDPROBE_ERR_STATE:
			err = fmt.Errorf("%w: %v", ErrState, err)
		case C.CDPROBE_ERR_UNSUPPORTED:
			err = fmt.Errorf("%w: %v", ErrUnsupported, err)
		}
		return CeAllToAll{}, err
	}
	n, ns := int(ca.n), int(ca.n_sizes)
	out := CeAllToAll{N: n, RowMask: uint32(ca.row_mask), Reps: int(ca.reps), Op: uint32(ca.op),
		CallSeq: uint64(ca.call_seq), AreaBytes: uint64(ca.area_bytes), Ms: float64(ca.ms)}
	out.Sizes = make([]uint64, ns)
	for s := 0; s < ns; s++ {
		out.Sizes[s] = uint64(ca.size[s])
	}
	out.Measured, out.Status, out.Blocks = make([]bool, n), make([]int32, n), make([]uint32, n)
	out.T0Ns, out.PeakGBps, out.HalfBytes = make([]float32, n), make([]float32, n), make([]uint64, n)
	out.NsMin, out.NsMedian, out.NsMax = make([][]float32, n), make([][]float32, n), make([][]float32, n)
	out.CellMeasured, out.CellStatus, out.BadSizes = make([][]bool, n), make([][]int32, n), make([][]uint32, n)
	out.CopyNsMedian = make([][][]float32, n)
	out.BadWords, out.FirstBad = make([][][]uint64, n), make([][][]uint64, n)
	out.Sum, out.Xr = make([][][]uint64, n), make([][][]uint64, n)
	for r := 0; r < n; r++ {
		out.Measured[r] = ca.measured[r] != 0
		out.Status[r] = int32(ca.status[r])
		out.Blocks[r] = uint32(ca.blocks[r])
		out.T0Ns[r] = float32(ca.t0_ns[r])
		out.PeakGBps[r] = float32(ca.peak_gbps[r])
		out.HalfBytes[r] = uint64(ca.half_bytes[r])
		out.NsMin[r], out.NsMedian[r], out.NsMax[r] = make([]float32, ns), make([]float32, ns), make([]float32, ns)
		for s := 0; s < ns; s++ {
			out.NsMin[r][s] = float32(ca.ns_min[r][s])
			out.NsMedian[r][s] = float32(ca.ns_median[r][s])
			out.NsMax[r][s] = float32(ca.ns_max[r][s])
		}
		out.CellMeasured[r], out.CellStatus[r], out.BadSizes[r] = make([]bool, n), make([]int32, n), make([]uint32, n)
		out.CopyNsMedian[r] = make([][]float32, n)
		out.BadWords[r], out.FirstBad[r] = make([][]uint64, n), make([][]uint64, n)
		out.Sum[r], out.Xr[r] = make([][]uint64, n), make([][]uint64, n)
		for d := 0; d < n; d++ {
			c := r*C.CDPROBE_MAX_GPUS + d
			out.CellMeasured[r][d] = ca.cell_measured[c] != 0
			out.CellStatus[r][d] = int32(ca.cell_status[c])
			out.BadSizes[r][d] = uint32(ca.bad_sizes[c])
			out.CopyNsMedian[r][d] = make([]float32, ns)
			out.BadWords[r][d], out.FirstBad[r][d] = make([]uint64, ns), make([]uint64, ns)
			out.Sum[r][d], out.Xr[r][d] = make([]uint64, ns), make([]uint64, ns)
			for s := 0; s < ns; s++ {
				out.CopyNsMedian[r][d][s] = float32(ca.copy_ns_median[c][s])
				out.BadWords[r][d][s] = uint64(ca.bad_words[c][s])
				out.FirstBad[r][d][s] = uint64(ca.first_bad[c][s])
				out.Sum[r][d][s] = uint64(ca.sum[c][s])
				out.Xr[r][d][s] = uint64(ca.xr[c][s])
			}
		}
	}
	return out, nil
}

// SetOption sets one run option (CDPROBE_OPT_*).  ErrUnsupported when the library lacks cdprobe_set_option.
func (p *Probe) SetOption(option uint32, value uint64) error {
	if C.cdp_has_set_option() == 0 {
		return fmt.Errorf("%w: libcdprobe.so has no cdprobe_set_option", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	if rc := C.cdp_call_set_option(p.h, C.uint32_t(option), C.uint64_t(value)); rc != 0 {
		return fmt.Errorf("cdprobe_set_option: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
	}
	return nil
}

// Links returns the per-link NVLink counters of the last Run taken with OptLinkCounters on, one row per local GPU.
// One-sided, not collective.  ErrUnsupported when the library predates cdprobe_links.
func (p *Probe) Links() (Links, error) {
	if C.cdp_has_links() == 0 {
		return Links{}, fmt.Errorf("%w: libcdprobe.so has no cdprobe_links", ErrUnsupported)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	t := new(C.cdprobe_links_t)
	if rc := C.cdp_call_links(p.h, t); rc != 0 {
		return Links{}, fmt.Errorf("cdprobe_links: %s: %s", C.GoString(C.cdp_call_strerror(rc)), C.GoString(C.cdp_call_last()))
	}
	out := Links{RunSeq: uint64(t.run_seq), SampleMs: float64(t.sample_ms)}
	const nl = C.CDPROBE_NVLINK_MAX_LINKS
	for k := 0; k < int(t.n_devices); k++ {
		d := &t.dev[k]
		x := LinkDevice{Status: int32(d.status), RankMask: uint32(d.rank_mask), UUID: C.GoString(&d.uuid[0]),
			LinkMask: uint32(d.link_mask), LostMask: uint32(d.lost_mask), ErrorMask: uint32(d.error_mask),
			ExpectedTxKiB: uint64(d.expected_tx_kib), ExpectedRxKiB: uint64(d.expected_rx_kib)}
		x.TxKiB, x.RxKiB = make([]uint64, nl), make([]uint64, nl)
		x.Errors, x.FailedFields, x.RemoteBusID = make([][3]uint64, nl), make([]uint32, nl), make([]string, nl)
		for l := 0; l < nl; l++ {
			x.TxKiB[l], x.RxKiB[l] = uint64(d.tx_kib[l]), uint64(d.rx_kib[l])
			for c := 0; c < 3; c++ {
				x.Errors[l][c] = uint64(d.errors[l][c])
			}
			x.FailedFields[l] = uint32(d.failed_fields[l])
			x.RemoteBusID[l] = C.GoString(&d.remote_bus_id[l][0])
		}
		out.Devices = append(out.Devices, x)
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
