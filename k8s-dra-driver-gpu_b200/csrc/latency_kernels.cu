// latency_kernels.cu — sm_90a kernel of cdprobe_latency: dependent 8-byte loads through one mapping, timed with
// %globaltimer on the issuing GPU.
//
// One 32-thread block per cell; lane 0 chases and the other lanes exit, so a chase has exactly one load in flight.
// Every load is ld.relaxed.sys.global (LDG.E.64.STRONG.SYS): it bypasses L1 and is served by the owner's L2 or HBM,
// at the scope the probe's barrier polls use.  The chase (probe_types.h, latency_start / latency_next) computes its
// first line, so the opening timer read waits on nothing; the closing one comes after the last loaded word has been
// used, so it cannot issue before that load has returned.  The device deadline (timeout_ms) is checked every 64 hops.
//
// probe_kernels.cu is untouched: the probe kernel's code generation does not depend on this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cdprobe.h"
#include "latency.h"

namespace cdp {
namespace {

__device__ __forceinline__ uint64_t ld_relaxed_sys(const uint8_t* p) {
  uint64_t v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__global__ void __launch_bounds__(32) latency_kernel(const __grid_constant__ LatencyParams p, TimedRep* out) {
  if (threadIdx.x != 0) return;
  const LatencyCell c = p.cell[blockIdx.x];
  TimedRep* o = out + (size_t)blockIdx.x * kRepSlots;
  const uint64_t deadline = globaltimer() + p.timeout_ns;
  for (uint32_t r = 0; r <= p.reps; ++r) {
    uint64_t line = latency_start(p.seed, c.issuer, c.target, r, c.lines);
    uint64_t digest = 0, v = 0;
    int32_t status = 0;
    const uint64_t t0 = globaltimer();
    for (uint32_t h = 0; h < p.hops; ++h) {
      v = ld_relaxed_sys(c.region + line * (kLineWords * 8));
      digest ^= v;
      line = latency_next(v, h, c.lines);
      if ((h & 63u) == 63u && globaltimer() > deadline) {
        status = CDPROBE_ERR_TIMEOUT;
        break;
      }
    }
    const uint64_t t1 = globaltimer_after(v);
    o[r].ns = t1 - t0;
    o[r].digest = digest;
    o[r].status = status;
    if (status != 0) return;
  }
}

}  // namespace

int latency_launch(const LatencyParams& p, TimedRep* out, cudaStream_t stream) {
  if (p.n_cells == 0) return (int)cudaSuccess;
  latency_kernel<<<p.n_cells, 32, 0, stream>>>(p, out);
  return (int)cudaGetLastError();
}

}  // namespace cdp
