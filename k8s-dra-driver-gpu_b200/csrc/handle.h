// handle.h — the probe handle and the helpers its C entry points share: handle.cc (open, close, mapping, options,
// the run path) and measure.cc (the on-demand measurements).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <time.h>

#include <string>

#include "../../include/cdprobe.h"
#include "plan.h"
#include "probe_types.h"
#include "rendezvous.h"
#include "timed_rep.cuh"
#include "vmm.h"

namespace cdp {

struct CopyHost;
struct LinkCounters;

inline thread_local std::string g_last_error;

inline void set_err(const std::string& s) { g_last_error = s; }

inline double now_ms() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec * 1e3 + ts.tv_nsec / 1e6;
}

constexpr int32_t kStatusUnmapped = CDPROBE_ERR_STATE;  // fault-injected / torn-down mapping

struct LocalRank {
  uint32_t grank = 0;
  int ordinal = -1;
  int sm_count = 0;
  uint32_t ctas = 0;
  bool coop = false;
  bool mig = false;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int max_ctas = 0;
  ResultRow* row = nullptr;
  char uuid[48] = {};
  Phase phases[kMaxPhases];
  uint32_t n_phases = 0;
  uint32_t peer_mask = 0;
  void* scratch = nullptr;  // device output of the on-demand measurements (measure.cc), grown on demand
  size_t scratch_bytes = 0;
  // cdprobe_memcpy and cdprobe_ce_alltoall, made on the first call of either: rep r is timed from [2r] to [2r + 1]
  cudaEvent_t rep_ev[2 * kRepSlots] = {};
  // cdprobe_ce_alltoall, made on its first call and kept until close: one copy stream per cell the rank issues, each
  // with the events of its copy ([0] to [1]) and of its join ([2])
  cudaStream_t cea_stream[kMaxRanks] = {};
  cudaEvent_t cea_copy_ev[kMaxRanks][3] = {};
};

// One allocation per local rank, shared with the whole domain: each process creates its local ranks' allocations,
// exports them, takes the other processes' over the rendezvous, imports them and maps every rank's into every local
// rank (handle.cc, share_alloc).  The probe allocation and the measurements' unicast areas are SharedAllocs (the
// cdprobe members say which, how large and whose).
struct SharedAlloc {
  size_t bytes = 0;                                       // of each allocation; 0: not created
  CUdeviceptr va[kMaxRanks][kMaxRanks] = {};              // [local rank][rank] rank j's allocation as mapped there
  bool mapped[kMaxRanks][kMaxRanks] = {};
  CUmemGenericAllocationHandle own[kMaxRanks] = {};       // [local rank]
  bool has_own[kMaxRanks] = {};
  int own_fd[kMaxRanks];                                  // [local rank] exported POSIX fd, -1: none
  CUmemGenericAllocationHandle imported[kMaxRanks] = {};  // [rank] of another process
  bool has_import[kMaxRanks] = {};
  int32_t status[kMaxRanks][kMaxRanks] = {};  // an area's [issuer][owner] mapping status, all ranks, once it exists
                                              // (the probe allocation's is cdprobe::status)
  bool stale = false;  // an area that must start zeroed must be zeroed before its next use: it is new, or a local
                       // rank's kernel timed out and it may hold packets, data, flags or partial sums of any earlier call
  SharedAlloc() {
    for (int& f : own_fd) f = -1;
  }
};

// The NVLS area (handle.cc, ensure_nvls): one multicast object of `bytes` that spans the domain, and per local rank an
// allocation of `bytes` on its device, bound into the object at offset 0, mapped into the rank both through the object
// (multicast) and on its own (unicast).  Peers never map another rank's allocation.
struct NvlsArea {
  size_t bytes = 0;                         // of the object and of each allocation; 0: not created
  CUmemGenericAllocationHandle mc = 0;      // the multicast object, created here or imported from rank 0's process
  bool has_mc = false;
  CUmemGenericAllocationHandle own[kMaxRanks] = {};  // [local rank]
  bool has_own[kMaxRanks] = {}, bound[kMaxRanks] = {};
  CUdeviceptr mc_va[kMaxRanks] = {}, uc_va[kMaxRanks] = {};  // [local rank] its multicast and unicast mappings
  bool mc_mapped[kMaxRanks] = {}, uc_mapped[kMaxRanks] = {};
};

// The measurements that keep a record on the handle (cdprobe::meas), one per entry point; the all-reduces are
// cdprobe_allreduce, cdprobe_allreduce_twoshot, _ll, _ring, _push and _nvls.
enum Measurement : uint32_t {
  kMeasPingPong, kMeasAtomics, kMeasBwCurve,
  kMeasAllReduce, kMeasTwoShot, kMeasLl, kMeasRing, kMeasPush, kMeasNvls,
  kMeasAllToAll, kMeasMemcpy, kMeasCeAllToAll,
  kMeasCount
};

// What a measurement keeps on the handle between calls.  `calls` counts its calls that ran, so it is the call_seq of
// the last one; the words, flags and values its kernels exchange derive from it.  `fault` is its armed test fault, the
// value of its CDPROBE_OPT_*_FAULT option (handle.cc, kFaultOptions), 0: disarmed; the call checks it.
// cdprobe_bwcurve has no fault option, so its fault stays 0.
struct MeasRecord {
  uint64_t calls = 0;
  uint64_t fault = 0;
};

}  // namespace cdp

struct cdprobe {
  cdprobe_config_t cfg;
  cdp::Plan plan;
  cdp::Driver drv;
  cdp::Rendezvous rdv;
  uint32_t n_total = 0, n_local = 0, first = 0;
  uint32_t handle_type = 0;  // 0 none, 1 posix fd, 8 fabric
  cdp::LocalRank lr[cdp::kMaxRanks];
  // The device memory shared across the domain, per rank.  The probe allocation is made at open; every other area on
  // the first call of the measurement that owns it (ensure_area, ensure_nvls), rounded up to the VMM granule.  All are
  // kept until close.
  cdp::SharedAlloc mem;     // the probe allocation: plan.alloc_bytes
  cdp::SharedAlloc area;    // cdprobe_alltoall's exchange area: n_total x bytes_per_pair
  cdp::SharedAlloc gather;  // cdprobe_allreduce_twoshot's gather area: bytes_per_pair
  cdp::SharedAlloc ll;      // cdprobe_allreduce_ll's LL area: 2 x n_total x 2 x the LL ladder's largest size
  cdp::SharedAlloc ring;    // cdprobe_allreduce_ring's ring area: bytes_per_pair and one flag per 8 KiB of it
  cdp::SharedAlloc push;    // cdprobe_allreduce_push's push area: bytes_per_pair
  // cdprobe_allreduce_nvls's multicast object and NVLS areas: 2 x bytes_per_pair, also rounded up to the multicast
  // granularity
  cdp::NvlsArea nvls;
  int32_t status[cdp::kMaxRanks][cdp::kMaxRanks];  // [issuer][owner] mapping status, all ranks
  uint64_t launch_seq = 0;
  uint64_t last_run_seq = 0;  // launch_seq of the last cdprobe_run (0: none yet); the run a diagnosis checks
  uint64_t seed = 0;
  uint64_t src_sum[cdp::kMaxRanks][cdp::kMaxRanks] = {};
  uint64_t src_xor[cdp::kMaxRanks][cdp::kMaxRanks] = {};
  bool sticky = false;
  bool event_timing = false;
  uint32_t path = 0;          // 0 TMA bulk, 1 ld/st 128-bit, 2 ld/st 256-bit
  uint32_t warm_mode = 1;     // 0 never, 1 auto (after an idle gap), 2 always
  uint64_t warm_bytes = 8ull << 20;   // untimed wake-up prefix per rank
  double warm_idle_ms = 5.0;  // auto: wake the links when the previous run ended longer ago than this
  double last_run_end_ms = -1.0;
  bool warm_now = false;
  uint32_t debug_skip_rank = 0;  // 1-based local rank whose kernel is NOT launched (fault injection)
  uint32_t solo_rank = 0;        // 1-based local rank that runs alone, no cross-GPU barrier (ncu captures)
  double last_probe_ms = 0.0;    // host wall clock of the previous run (wait_rows: how long to spin hot)
  uint32_t verify_ctas = 32;  // CTAs that verify landing slots under CDPROBE_FLAG_OVERLAP_VERIFY
  int32_t fault_local = -1;   // local rank whose Ctrl holds the armed landing fault (cdprobe_corrupt_landing), -1: none
  cdp::MeasRecord meas[cdp::kMeasCount];  // [Measurement]
  // the pinned host block of cdprobe_memcpy and cdprobe_ce_alltoall (measure.cc), made by the first call of either:
  // the tickets their streams wait on and what their checks leave
  cdp::CopyHost* copy_host = nullptr;
  uint32_t max_connections = 8;       // CUDA_DEVICE_MAX_CONNECTIONS as read at open: hardware queues per device
  char rank_uuid[cdp::kMaxRanks][48] = {};  // every rank's device UUID, exchanged at open (cdprobe_links' payload)
  bool link_counters = false;               // CDPROBE_OPT_LINK_COUNTERS
  cdp::LinkCounters* links = nullptr;       // NVML, the local devices and the last report, from the option's first
                                            // enabling until close
  double open_ms = 0, fill_ms = 0;
};

namespace cdp {

inline int fail_cuda(const char* what, cudaError_t e) {
  set_err(std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")");
  if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver || e == cudaErrorInitializationError ||
      e == cudaErrorSystemDriverMismatch || e == cudaErrorSystemNotReady || e == cudaErrorNotSupported)
    return CDPROBE_ERR_NO_DEVICE;
  if (e == cudaErrorNoKernelImageForDevice || e == cudaErrorInvalidDeviceFunction ||
      e == cudaErrorCooperativeLaunchTooLarge)
    return CDPROBE_ERR_UNSUPPORTED;
  if (e == cudaErrorMemoryAllocation) return CDPROBE_ERR_NOMEM;
  return CDPROBE_ERR_CUDA;
}

#define CDP_RT(call)                                       \
  do {                                                     \
    cudaError_t e_ = (call);                               \
    if (e_ != cudaSuccess) return cdp::fail_cuda(#call, e_);    \
  } while (0)

// CDPROBE_ERR_STATE once a timeout or CUDA error has made the handle sticky.
inline int require_usable(const cdprobe* h) {
  if (!h->sticky) return CDPROBE_OK;
  set_err("handle is unusable after an earlier timeout or CUDA error: close it and open a new one");
  return CDPROBE_ERR_STATE;
}

// The device deadline every kernel gets, counted from its entry: timeout_ms.
inline uint64_t timeout_ns(const cdprobe* h) { return (uint64_t)h->cfg.timeout_ms * 1000000ull; }

// Whether local rank L's grid kernels (the probe and the ladder measurements) launch cooperatively: when its device
// can and CDPROBE_FLAG_NO_COOPERATIVE is clear.
inline bool launch_cooperatively(const cdprobe* h, const LocalRank& L) {
  return L.coop && !(h->cfg.flags & CDPROBE_FLAG_NO_COOPERATIVE);
}

// A measurement's unicast shared area m (handle.cc).  On the first call, every local rank creates `bytes` of device
// memory (rounded up to the VMM granule), shared like the probe allocation and mapped into every local rank wherever
// the probe mapping is then up; m.status gets every rank's mapping statuses.  Collective.  If creating it fails in any
// process, every process returns the first failure in process order, with that process's message; nothing is kept,
// and the next call tries again.  Kept until close.
int ensure_area(cdprobe* h, SharedAlloc& m, size_t bytes);

// The NVLS area (h->nvls, DESIGN §5m): on the first call, `bytes` rounded up to the VMM granule and to the multicast
// granularity.  The process hosting rank 0 creates the multicast object with the probe allocation's handle type
// (POSIX fd within one process, which has none) and hands it to the others over the rendezvous; every process adds
// its devices; once every process has reported that, each local rank creates its allocation, binds it at offset 0 and
// maps the object and its allocation.  Collective, and only for a domain that agree() found able to run it.  If a step
// fails in any process, every process returns the first failure as ensure_area does (cdprobe_last_error names the
// step and the CUresult); nothing is kept, and the next call tries again.  *refused: the failure is the
// driver refusing a multicast object of one device (cuMulticastCreate, CUDA_ERROR_INVALID_VALUE, n_total == 1), which
// the caller reports as CDPROBE_ERR_UNSUPPORTED rows.  Kept until close.
int ensure_nvls(cdprobe* h, size_t bytes, bool* refused);

// The mapping status of local rank li's cell [its rank][j]: kStatusUnmapped when that status is 0 but the peer is not
// mapped.  Non-zero: never read or write through that mapping.
inline int32_t cell_status(const cdprobe* h, uint32_t li, uint32_t j) {
  const int32_t s = h->status[h->lr[li].grank][j];
  return s == 0 && !h->mem.mapped[li][j] ? kStatusUnmapped : s;
}

}  // namespace cdp
