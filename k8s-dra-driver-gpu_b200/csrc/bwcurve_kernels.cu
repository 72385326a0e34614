// bwcurve_kernels.cu — sm_90a kernels of cdprobe_bwcurve: reads of growing prefixes of one source slice through the
// probe's K1 read path (datapath.cuh), one launch per cell, each rep between two grid barriers (bwcurve_kernel); and
// the per-granule sums of a source slice that the expected checksums are folded from (granules_kernel<SrcRegionWord>).
//
// probe_kernels.cu is untouched: the probe kernel's code generation does not depend on this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "bwcurve.h"
#include "datapath.cuh"

namespace cdp {

// One cell of cdprobe_bwcurve: for every size of the ladder, one warm-up and P.reps timed reps, each reading the first
// size bytes of the cell's source slice with every warp of the grid (the strided walk of a probe phase, on the data
// path the probe uses) and folding them into the (S, X) checksum.  Reps are separated by grid barriers, so a rep is
// timed as a probe phase is: from the barrier's release stamp to the latest CTA completion stamp.  Every piece of
// state (barrier, stamps, checksums, abort word) is in the rank's scratch buffer; Ctrl is not touched.
__global__ void __launch_bounds__(kThreads, 1) bwcurve_kernel(const __grid_constant__ BwCurveParams P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  BwScratch* bs = P.scratch;
  uint64_t* red;
  Ctx c = enter(smem, &bs->abort_flag, P.timeout_ns, &red);

  const uint32_t gwarp = blockIdx.x * kWarpsPerCta + c.warp;
  const uint32_t nwarps = gridDim.x * kWarpsPerCta;
  uint32_t b = 0;
  for (uint32_t k = 0; k < P.n_sizes; ++k) {
    const uint64_t bytes = P.size[k];
    for (uint32_t r = 0; r <= P.reps; ++r, ++b) {
      if (!grid_barrier(c, bs, b, &bs->t_rel[k][r], nullptr, false)) return;
      Sum a{0ull, 0ull, 0ull};
      read_units(c, P.path, P.region, bytes, strided(bytes, gwarp, nwarps), a);
      Acc* const acc = &bs->rep[k][r];
      cta_reduce<1>(c, red, &a, &acc);
      if (threadIdx.x == 0) atomicMax(&acc->t_end, (unsigned long long)gtimer());
    }
  }
}

int bwcurve_launch(const BwCurveParams& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  return grid_launch(bwcurve_kernel, p, grid, cooperative, stream);
}

template int granules_launch(uint64_t*, uint64_t*, const SrcRegionWord&, uint64_t, unsigned, cudaStream_t);

}  // namespace cdp
