// allreduce_ll.h — host-callable launcher of the low-latency all-reduce kernel in allreduce_ll_kernels.cu
// (cdprobe_allreduce_ll).  Its scratch head is the one-shot's ArScratch (allreduce.h), its output at kArOutOff.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "allreduce.h"
#include "probe_types.h"

namespace cdp {

struct LlParams {
  const uint8_t* src;             // this rank's own source buffer
  uint8_t* dst[kMaxRanks];        // the LL area of rank + t (mod n) at dst[t], t >= 1, through this rank's mapping:
                                  // where this rank's packets go, in that order
  const uint8_t* in;              // this rank's own LL area: where every peer's packets arrive
  DomainLines dom;                // the opening barrier of every size, through the kLlOff lines; dom.call_seq is the
                                  // call number the packet flags carry (ll_flag)
  ArScratch* scratch;
  uint8_t* out;                   // the output, in this rank's scratch at kArOutOff
  uint64_t size[kBwMaxSizes];     // the ladder (ll_ladder)
  uint64_t s_max;                 // its largest size: the LL area's slot layout (ll_slot)
  uint64_t seed;                  // the pattern seed (the inputs, the salts and the word check)
  uint64_t timeout_ns;            // device deadline from kernel entry
  uint64_t fault_arg;             // the armed fault, in size fault_k (kArNoFault: disarmed): in timed rep 1, mode 0,
  uint32_t fault_k;               //   the packet of word fault_arg to dst[fault_dst] carries its data xored with 1;
  uint32_t fault_mode, fault_dst; //   mode 1, this rank waits fault_arg us before its first push; in every rep,
                                  //   mode 2, this rank makes no store to output word fault_arg
  uint32_t rank, n, n_sizes, reps;
  uint32_t ctas;                  // the domain's smallest grid: only CTAs below it move words
  uint32_t path;                  // set for every ladder kernel; LL has one data path and ignores it
};

// Launches allreduce_ll_kernel on `stream` of the current device: `grid` (>= p.ctas) CTAs of the probe kernel's shape,
// cooperative or not as the probe launches them.  For every size, one domain barrier, then one warm-up and p.reps
// timed reps back to back, each pushing this rank's words as flag-carrying packets to every peer and summing the
// packets that arrive, then the word check and clear of the last one's output (DESIGN §5j).  Returns a cudaError_t.
int allreduce_ll_launch(const LlParams& p, unsigned grid, bool cooperative, cudaStream_t stream);

}  // namespace cdp
