// latency.h — host-callable launcher of the dependent-load chase in latency_kernels.cu (cdprobe_latency).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "probe_types.h"
#include "timed_rep.cuh"

namespace cdp {

constexpr uint32_t kLatencyDefaultHops = 1024;
constexpr uint32_t kLatencyDefaultReps = 8;
constexpr uint32_t kLatencyMaxHops = 1u << 20;

struct LatencyCell {
  const uint8_t* region;  // the source slice the issuer reads, through the issuer's mapping of the target
  uint64_t lines;         // 128-byte lines in it
  uint32_t issuer, target;
};

struct LatencyParams {
  LatencyCell cell[kMaxRanks];  // one 32-thread block per cell
  uint64_t seed;
  uint64_t timeout_ns;          // device deadline from kernel entry, checked every 64 hops
  uint32_t n_cells, hops, reps; // reps: timed reps (rep 0, the warm-up, comes on top)
};

// Enqueues the chases of p.n_cells cells on `stream`; cell k leaves its reps at out[k * kRepSlots + rep], each with a
// status of 0 or CDPROBE_ERR_TIMEOUT.  Returns a cudaError_t.
int latency_launch(const LatencyParams& p, TimedRep* out, cudaStream_t stream);

}  // namespace cdp
