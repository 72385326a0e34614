// timed_rep.cuh — the per-rep record the timed measurements leave in device memory (cdprobe_latency,
// cdprobe_pingpong, cdprobe_atomics), and the %globaltimer reads their kernels time a rep with.
#pragma once
#include <stdint.h>

namespace cdp {

constexpr uint32_t kMaxTimedReps = 64;  // timed reps; one untimed warm-up rep runs before them
constexpr uint32_t kRepSlots = kMaxTimedReps + 1;

struct TimedRep {             // what a kernel leaves per cell and rep, at [cell * kRepSlots + rep]
  unsigned long long ns;      // %globaltimer: the rep's closing read - its opening read
  unsigned long long digest;  // xor of the words this rep received
  int32_t status;             // 0 or a CDPROBE_ERR_*; CDPROBE_ERR_TIMEOUT: a wait passed the deadline and later reps
                              // did not run
  uint32_t pad;
};
static_assert(sizeof(TimedRep) == 24, "timed rep slot");

#if defined(__CUDACC__)
__device__ __forceinline__ uint64_t globaltimer() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)::"memory");
  return t;
}
// The closing timer read.  `v`, the last word the rep received, is an operand, so the compiler cannot place the read
// ahead of the load that returned it.  In the SASS the read follows the rep's loop, whose use of v (the digest xor,
// the echo compare) waits for the load, and instructions issue in order: the read cannot issue before the last load
// has returned (tests/test_latency_cpu.py and tests/test_pingpong_cpu.py check that order in the compiled kernels).
__device__ __forceinline__ uint64_t globaltimer_after(uint64_t v) {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t) : "l"(v) : "memory");
  return t;
}
#endif

}  // namespace cdp
