// allreduce.h — host-callable launchers of the one-shot all-reduce kernels in probe_kernels.cu (cdprobe_allreduce), and
// the layout of the scratch buffer they share with the host.
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
// and (S, X)) for the reps of every size; the word check of size k adds its bad words into bad_words[k] and keeps
// ~(the lowest bad byte offset) in first_bad_n[k] (0: none).  The output follows at kArOutOff.
struct ArScratch {
  BwScratch rep;
  alignas(128) unsigned long long bad_words[kBwMaxSizes];
  unsigned long long first_bad_n[kBwMaxSizes];
};
constexpr size_t kArOutOff = (sizeof(ArScratch) + 255) / 256 * 256;

struct AllReduceParams {
  const uint8_t* src[kMaxRanks];  // the n inputs in the order this rank adds them: rank + t (mod n) at src[t], each
                                  // through this rank's mapping, src[0] its own source buffer
  uint64_t* sig_out[kMaxRanks];   // this rank's line in rank j's Ctrl granule (null for j == rank)
  const FlagLine* sig_in;         // this rank's own lines: sig_in[j].v is the last barrier value rank j signalled
  ArScratch* scratch;
  uint8_t* out;                   // the output, in this rank's scratch
  uint64_t size[kBwMaxSizes];     // the ladder (bwcurve_ladder)
  uint64_t seed;                  // the pattern seed (the word check)
  uint64_t call_seq;              // the barrier values' high bits
  uint64_t timeout_ns;            // device deadline from kernel entry
  uint64_t fault_word;            // the armed fault: timed rep 1 of size fault_k adds 1 to this output word
  uint32_t fault_k;               // kArNoFault: disarmed
  uint32_t rank, n, n_sizes, reps;
  uint32_t path;                  // ProbeParams::path: the read side
};

// Launches allreduce_kernel on `stream` of the current device: `grid` CTAs of the probe kernel's shape, cooperative or
// not as the probe launches them.  For every size, one warm-up and p.reps timed reps, each opened by a domain barrier,
// then the word check of the last one.  Returns a cudaError_t.
int allreduce_launch(const AllReduceParams& p, unsigned grid, bool cooperative, cudaStream_t stream);
// Writes gsum[g] / gxor[g], the sum and the xor of the words of whole granule g of the n-rank all-reduce output, for
// its first n_granules granules, computed from allreduce_word.  Returns a cudaError_t.
int allreduce_granules_launch(uint64_t* gsum, uint64_t* gxor, uint64_t seed, uint32_t n, uint64_t n_granules,
                              unsigned grid, cudaStream_t stream);

}  // namespace cdp
