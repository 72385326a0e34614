// alltoall.h — host-callable launcher of the one-shot all-to-all kernel in alltoall_kernels.cu (cdprobe_alltoall), and
// the layout of the scratch buffer it shares with the host.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "bwcurve.h"
#include "probe_types.h"

namespace cdp {

constexpr uint32_t kA2aDefaultReps = 8;
constexpr uint32_t kA2aNoFault = ~0u;

// The head of a local rank's scratch buffer during one alltoall_kernel launch; the host zeroes it before the launch and
// reads it back after.  `rep` holds what a bwcurve_kernel launch holds (abort word, grid barrier, per-rep stamps) for
// the reps of every size; its checksums stay 0.  The word checks of the blocks from sender s at size k add their bad
// words into bad_words[s][k] and keep ~(the lowest bad byte offset) in first_bad_n[s][k] (0: none); the last timed
// rep's words are folded into sum[s][k] and xr[s][k].
struct A2aScratch {
  BwScratch rep;
  alignas(128) unsigned long long bad_words[kMaxRanks][kBwMaxSizes];
  unsigned long long first_bad_n[kMaxRanks][kBwMaxSizes];
  unsigned long long sum[kMaxRanks][kBwMaxSizes];
  unsigned long long xr[kMaxRanks][kBwMaxSizes];
};

struct AllToAllParams {
  DomainLines dom;                // the domain barrier, over the kA2aOff lines
  uint8_t* dst[kMaxRanks];        // block b: this rank's block in receiver to[b]'s exchange area, through its mapping
  const uint8_t* in[kMaxRanks];   // incoming block i: sender from[i]'s block in this rank's own exchange area
  A2aScratch* scratch;
  uint64_t size[kBwMaxSizes];     // the ladder (bwcurve_ladder)
  uint64_t seed;                  // the pattern seed
  uint64_t timeout_ns;            // device deadline from kernel entry
  uint64_t fault_word;            // the armed fault: timed rep 1 of size fault_k stores this word of block fault_block
  uint32_t fault_k, fault_block;  //   xored with 1; fault_k kA2aNoFault: disarmed
  uint32_t to[kMaxRanks], from[kMaxRanks];
  uint32_t rank, blocks, n_in, n_sizes, reps;
  uint32_t path;                  // ProbeParams::path: the write side
};

// Launches alltoall_kernel on `stream` of the current device: `grid` CTAs of the probe kernel's shape, cooperative or
// not as the probe launches them.  For every size, one warm-up and p.reps timed reps, each a domain barrier, the push
// of p.blocks blocks, an untimed domain barrier and the word check of the p.n_in incoming blocks.  Returns a
// cudaError_t.
int alltoall_launch(const AllToAllParams& p, unsigned grid, bool cooperative, cudaStream_t stream);

}  // namespace cdp
