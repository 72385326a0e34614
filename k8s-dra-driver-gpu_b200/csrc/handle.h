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
#include "vmm.h"

namespace cdp {

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
  CUmemGenericAllocationHandle own = 0;
  bool has_own = false;
  int own_fd = -1;
  CUdeviceptr va[kMaxRanks] = {};
  bool mapped[kMaxRanks] = {};
  ResultRow* row = nullptr;
  char uuid[48] = {};
  Phase phases[kMaxPhases];
  uint32_t n_phases = 0;
  uint32_t peer_mask = 0;
  void* scratch = nullptr;  // device output of the on-demand measurements (measure.cc), grown on demand
  size_t scratch_bytes = 0;
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
  CUmemGenericAllocationHandle imported[cdp::kMaxRanks] = {};
  bool has_import[cdp::kMaxRanks] = {};
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
  uint64_t pp_calls = 0;      // cdprobe_pingpong calls that ran (call_seq of the last one)
  uint64_t pp_fault = 0;      // CDPROBE_OPT_PINGPONG_FAULT value, 0: disarmed
  uint64_t at_calls = 0;      // cdprobe_atomics calls that ran (call_seq of the last one)
  uint64_t at_fault = 0;      // CDPROBE_OPT_ATOMICS_FAULT value, 0: disarmed
  uint64_t bw_calls = 0;      // cdprobe_bwcurve calls that ran (call_seq of the last one)
  uint64_t ar_calls = 0;      // cdprobe_allreduce calls that ran (call_seq of the last one)
  uint64_t ar_fault = 0;      // CDPROBE_OPT_ALLREDUCE_FAULT value, 0: disarmed
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

// The mapping status of local rank li's cell [its rank][j]: kStatusUnmapped when that status is 0 but the peer is not
// mapped.  Non-zero: never read or write through that mapping.
inline int32_t cell_status(const cdprobe* h, uint32_t li, uint32_t j) {
  const int32_t s = h->status[h->lr[li].grank][j];
  return s == 0 && !h->lr[li].mapped[j] ? kStatusUnmapped : s;
}

}  // namespace cdp
