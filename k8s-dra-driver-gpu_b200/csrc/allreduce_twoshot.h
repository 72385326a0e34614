// allreduce_twoshot.h — host-callable launcher of the two-shot all-reduce kernel in allreduce_twoshot_kernels.cu
// (cdprobe_allreduce_twoshot).  Its scratch head is the one-shot's ArScratch (allreduce.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "allreduce.h"
#include "probe_types.h"

namespace cdp {

struct TwoShotParams {
  const uint8_t* src[kMaxRanks];  // the n inputs in the order this rank adds them: rank + t (mod n) at src[t], each
                                  // through this rank's mapping, src[0] its own source buffer
  uint8_t* dst[kMaxRanks];        // the gather area of rank + t (mod n) at dst[t], through this rank's mapping: where a
                                  // summed unit goes, in that order; dst[0] is this rank's own, its output
  DomainLines dom;                // the domain barrier: push to and wait for every other rank through the kAr2Off lines
  ArScratch* scratch;
  uint64_t size[kBwMaxSizes];     // the ladder (bwcurve_ladder)
  uint64_t seed;                  // the pattern seed (the word check)
  uint64_t timeout_ns;            // device deadline from kernel entry
  uint64_t fault_word;            // the armed fault: in timed rep 1 of size fault_k, the store of this output word to
  uint32_t fault_k;               //   dst[fault_dst] is xored with 1 (fault_drop 0), or every store of its unit to
  uint32_t fault_dst, fault_drop; //   dst[fault_dst] is skipped (1); fault_k kArNoFault: disarmed
  uint32_t rank, n, n_sizes, reps;
  uint32_t path;                  // ProbeParams::path: the read side
};

// Launches allreduce_twoshot_kernel on `stream` of the current device: `grid` CTAs of the probe kernel's shape,
// cooperative or not as the probe launches them.  For every size, one warm-up and p.reps timed reps; each rep is a
// domain barrier, the reduction of this rank's chunk pushed to every rank, a fenced domain barrier, and the word check
// and clear of this rank's output (DESIGN §5i).  Returns a cudaError_t.
int allreduce_twoshot_launch(const TwoShotParams& p, unsigned grid, bool cooperative, cudaStream_t stream);

}  // namespace cdp
