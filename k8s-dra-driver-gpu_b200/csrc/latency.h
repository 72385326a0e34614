// latency.h — host-callable launcher of the dependent-load chase in latency_kernels.cu (cdprobe_latency).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "probe_types.h"

namespace cdp {

constexpr uint32_t kLatencyDefaultHops = 1024;
constexpr uint32_t kLatencyDefaultReps = 8;
constexpr uint32_t kLatencyMaxHops = 1u << 20;
constexpr uint32_t kLatencyMaxReps = 64;              // timed reps; one untimed warm-up rep runs before them
constexpr uint32_t kLatencyRepSlots = kLatencyMaxReps + 1;

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

struct LatencyRep {             // what the kernel leaves per cell and rep, at [cell * kLatencyRepSlots + rep]
  unsigned long long ns;        // %globaltimer: last load returned - chase started
  unsigned long long digest;    // xor of the words this rep loaded
  int32_t status;               // 0, or CDPROBE_ERR_TIMEOUT (the chase stopped; later reps did not run)
  uint32_t pad;
};

// Enqueues the chases of p.n_cells cells on `stream`.  Returns a cudaError_t.
int latency_launch(const LatencyParams& p, LatencyRep* out, cudaStream_t stream);

}  // namespace cdp
