// allreduce_ring.h — host-callable launcher of the ring all-reduce kernel in allreduce_ring_kernels.cu
// (cdprobe_allreduce_ring).  Its scratch head is the one-shot's ArScratch (allreduce.h); its output is the first part of
// the rank's own ring area.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "allreduce.h"
#include "probe_types.h"

namespace cdp {

struct RingParams {
  const uint8_t* src;             // this rank's own source buffer
  uint8_t* out;                   // this rank's own ring area: its output, then its flags (ring_flags_off)
  uint8_t* next;                  // the ring area of rank + 1 (mod n), through this rank's mapping: where it pushes
  DomainLines dom;                // the opening barrier of every rep, through the kRingOff lines; dom.call_seq is the
                                  // call number the flags carry (ring_flag)
  ArScratch* scratch;
  uint64_t size[kBwMaxSizes];     // the ladder (bwcurve_ladder)
  uint64_t s_max;                 // its largest size: the ring area's layout
  uint64_t seed;                  // the pattern seed (the inputs and the word check)
  uint64_t timeout_ns;            // device deadline from kernel entry
  uint64_t fault_arg;             // the armed fault, in timed rep 1 of size fault_k (kArNoFault: disarmed): mode 0,
  uint32_t fault_k;               //   this rank's push of word fault_arg in phase fault_phase carries it xored with 1;
  uint32_t fault_mode;            //   mode 1, that push stores nothing of the word's flag grain but publishes its
  uint32_t fault_phase;           //   flag; mode 2, this rank waits fault_arg us before its first push of the rep
  uint32_t rank, n, n_sizes, reps;
  uint32_t path;                  // set for every ladder kernel; the ring has one data path and ignores it
};

// Launches allreduce_ring_kernel on `stream` of the current device: `grid` CTAs of the probe kernel's shape,
// cooperative or not as the probe launches them.  For every size, one warm-up and p.reps timed reps; each rep is a
// fenced domain barrier, the 2 (n - 1) steps of the ring in which every unit is passed to rank + 1 under a per-unit
// flag, a grid barrier, and the word check and clear of this rank's output (DESIGN §5k).  Returns a cudaError_t.
int allreduce_ring_launch(const RingParams& p, unsigned grid, bool cooperative, cudaStream_t stream);

}  // namespace cdp
