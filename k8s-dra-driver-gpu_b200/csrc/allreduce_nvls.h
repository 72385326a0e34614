// allreduce_nvls.h — host-callable launcher of the multicast all-reduce kernel in allreduce_nvls_kernels.cu
// (cdprobe_allreduce_nvls).  Its scratch head is the one-shot's ArScratch (allreduce.h); its input and output are the
// two halves of the rank's NVLS area, bound into one multicast object that spans the domain.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "allreduce.h"
#include "probe_types.h"

namespace cdp {

struct NvlsParams {
  const uint8_t* mc_in;           // the multicast object's input half as mapped here (multimem.ld_reduce)
  uint8_t* mc_out;                // its output half as mapped here (multimem.st)
  uint8_t* out;                   // this rank's own output half through its unicast mapping (the word check)
  DomainLines dom;                // the two domain barriers of every rep, through the kNvlsOff lines
  ArScratch* scratch;
  uint64_t size[kBwMaxSizes];     // the ladder (bwcurve_ladder)
  uint64_t seed;                  // the pattern seed (the word check)
  uint64_t timeout_ns;            // device deadline from kernel entry
  uint64_t fault_word;            // the armed fault, in timed rep 1 of size fault_k (kArNoFault: disarmed; this rank
  uint32_t fault_k;               //   owns the word): mode 0, the word is stored xored with 1; mode 1, the word's unit
  uint32_t fault_mode;            //   is not stored
  uint32_t rank, n, n_sizes, reps;
  uint32_t path;                  // ProbeParams::path, unused: every path issues the same multimem instructions
};

// Launches allreduce_nvls_kernel on `stream` of the current device: `grid` CTAs of the probe kernel's shape,
// cooperative or not as the probe launches them.  For every size, one warm-up and p.reps timed reps; each rep is a
// fenced domain barrier, this rank's chunk reduced by multimem.ld_reduce and stored to every rank by multimem.st, a
// fenced domain barrier, and the word check and clear of this rank's output (DESIGN §5m).  Returns a cudaError_t.
int allreduce_nvls_launch(const NvlsParams& p, unsigned grid, bool cooperative, cudaStream_t stream);

}  // namespace cdp
