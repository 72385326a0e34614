// allreduce.h — host-callable launchers of the one-shot all-reduce kernels in allreduce_kernels.cu (cdprobe_allreduce),
// and the layout of the scratch buffer they share with the host.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "bwcurve.h"
#include "probe_types.h"

namespace cdp {

constexpr uint32_t kArDefaultReps = 8;

// The head of a local rank's scratch buffer during one allreduce_kernel launch; the host zeroes it before the launch
// and reads it back after.  `rep` holds what a bwcurve_kernel launch holds (abort word, grid barrier, per-rep stamps
// and (S, X)) for the reps of every size; the word checks of size k add their bad words into bad_words[k] and keep
// ~(the lowest bad byte offset) in first_bad_n[k] (0: none).  The output of the one-shot and the LL follows at
// kArOutOff.
struct ArScratch {
  BwScratch rep;
  alignas(128) unsigned long long bad_words[kBwMaxSizes];
  unsigned long long first_bad_n[kBwMaxSizes];
};
constexpr size_t kArOutOff = (sizeof(ArScratch) + 255) / 256 * 256;

struct AllReduceParams {
  const uint8_t* src[kMaxRanks];  // the n inputs in the order this rank adds them: rank + t (mod n) at src[t], each
                                  // through this rank's mapping, src[0] its own source buffer
  DomainLines dom;                // the domain barrier: push to and wait for every other rank through the kArOff lines
  ArScratch* scratch;
  uint8_t* out;                   // the output, in this rank's scratch
  uint64_t size[kBwMaxSizes];     // the ladder (bwcurve_ladder)
  uint64_t seed;                  // the pattern seed (the word check)
  uint64_t timeout_ns;            // device deadline from kernel entry
  uint64_t fault_word;            // the armed fault: timed rep 1 of size fault_k adds 1 to this output word, or
  uint32_t fault_k;               //   (fault_drop) stores nothing of its 8 KiB unit; kArNoFault: disarmed
  uint32_t fault_drop;
  uint32_t rank, n, n_sizes, reps;
  uint32_t path;                  // ProbeParams::path: the read side
};

// Launches allreduce_kernel on `stream` of the current device: `grid` CTAs of the probe kernel's shape, cooperative or
// not as the probe launches them.  For every size, one warm-up and p.reps timed reps, each opened by a domain barrier
// and followed by the word check and clear of its output.  Returns a cudaError_t.
int allreduce_launch(const AllReduceParams& p, unsigned grid, bool cooperative, cudaStream_t stream);
// The expected output's per-granule sums come from granules_launch (bwcurve.h) with AllReduceWord.

}  // namespace cdp
