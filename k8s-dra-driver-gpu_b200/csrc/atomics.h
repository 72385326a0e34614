// atomics.h — host-callable launcher of the remote-atomic chains in atomics_kernels.cu (cdprobe_atomics).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "probe_types.h"
#include "timed_rep.cuh"

namespace cdp {

constexpr uint32_t kAtomicsDefaultOps = 1024;
constexpr uint32_t kAtomicsDefaultReps = 8;
constexpr uint32_t kAtomicsMaxOps = 1u << 16;
constexpr uint32_t kAtomicsNoFault = 0xFFFFFFFFu;

struct AtomicsCell {
  unsigned long long* word;  // word 0 of atom[issuer] in the target's Ctrl granule, through the issuer's mapping
  uint32_t issuer, target;
};

struct AtomicsParams {
  AtomicsCell cell[kMaxRanks];  // one 32-thread block per cell
  uint64_t call_seq;
  uint64_t timeout_ns;          // device deadline from kernel entry, checked every 64 ops
  uint32_t n_cells, ops, reps;  // ops per lane; reps: timed reps (rep 0, the warm-up, comes on top)
  uint32_t fault_cell;          // test-only: the cell whose first op of timed rep 1 adds 2 (kAtomicsNoFault: none)
};

// Enqueues the atomics of p.n_cells cells of kind `kind` (CDPROBE_ATOMIC_*) on `stream`; cell k leaves its reps at
// out[k * kRepSlots + rep], CDPROBE_ERR_INTEGRITY marking a rep whose returns or read-back differ from the expected
// values and CDPROBE_ERR_TIMEOUT one that passed the deadline (later reps do not run).  Returns a cudaError_t.
int atomics_launch(const AtomicsParams& p, uint32_t kind, TimedRep* out, cudaStream_t stream);

}  // namespace cdp
