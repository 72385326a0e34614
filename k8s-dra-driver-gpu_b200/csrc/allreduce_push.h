// allreduce_push.h — host-callable launcher of the push all-reduce kernel in allreduce_push_kernels.cu
// (cdprobe_allreduce_push).  Its scratch head is the one-shot's ArScratch (allreduce.h); its output is the first part of
// the rank's own push area.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "allreduce.h"
#include "probe_types.h"

namespace cdp {

struct PushParams {
  const uint8_t* src;             // this rank's own source buffer
  uint8_t* dst[kMaxRanks];        // the push area of rank + t (mod n) at dst[t], through this rank's mapping; dst[0] is
                                  // this rank's own, its output
  DomainLines dom;                // the three domain barriers of every rep, through the kPushOff lines
  ArScratch* scratch;
  uint64_t size[kBwMaxSizes];     // the ladder (bwcurve_ladder)
  uint64_t seed;                  // the pattern seed (the word check)
  uint64_t timeout_ns;            // device deadline from kernel entry
  uint64_t fault_word;            // the armed fault, in timed rep 1 of size fault_k (kArNoFault: disarmed), on output
  uint32_t fault_k;               //   word fault_word: mode 0, this rank's contribution is its source word + 1; mode 1,
  uint32_t fault_mode;            //   the word's unit is not reduced; mode 2, it is reduced twice; mode 3 (this rank
  uint32_t fault_dst;             //   owns the word), the all-gather pushes it xored with 1 to dst[fault_dst]
  uint32_t rank, n, n_sizes, reps;
  uint32_t path;                  // ProbeParams::path: 0 bulk reductions, 1 and 2 red.global per word
};

// Launches allreduce_push_kernel on `stream` of the current device: `grid` CTAs of the probe kernel's shape,
// cooperative or not as the probe launches them.  For every size, one warm-up and p.reps timed reps; each rep is a
// fenced domain barrier, every unit of this rank's input reduced into its owner's push area, a fenced domain barrier,
// this rank's own chunk pushed to every peer, a fenced domain barrier, and the word check and clear of this rank's
// output (DESIGN §5l).  Returns a cudaError_t.
int allreduce_push_launch(const PushParams& p, unsigned grid, bool cooperative, cudaStream_t stream);

}  // namespace cdp
