// allreduce_twoshot_kernels.cu — sm_90a kernel of cdprobe_allreduce_twoshot's two-shot all-reduce: every rank sums its
// chunk of units of all n source buffers with the one-shot's read-and-add side (allreduce_path.cuh) and pushes each
// summed unit with st.global.v4 into every rank's gather area; a fenced domain barrier closes the rep, and every rank
// then checks and clears its own gather area (allreduce_twoshot_kernel, with allreduce_path.cuh's ar_check_clear).
//
// probe_kernels.cu is untouched: the probe kernel's code generation does not depend on this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "allreduce_path.cuh"
#include "allreduce_twoshot.h"

namespace cdp {
namespace {
// The two-shot's store policy (allreduce_path.cuh): a summed unit goes to every rank's gather area, dst[0] (this
// rank's own) first.  The armed fault (fw, an output word index; ~0 when none) acts on the stores to dst[fault_dst]
// only: the word leaves xored with 1, or (fault_drop) nothing of its unit leaves.  Nothing is folded into (S, X); the
// word check reads the output back.
struct ToGather {
  template <uint32_t kLaneBytes>
  __device__ __forceinline__ static void put(const Ctx& c, const TwoShotParams& P, uint64_t u, uint32_t len,
                                             uint64_t fw, uint64_t (&acc)[kArWords], Sum&) {
    put_ranks<kLaneBytes, true>(c, P, 0u, u, len, fw, acc);
  }
};
}  // namespace

// One rank of cdprobe_allreduce_twoshot: for every size of the ladder, one warm-up and P.reps timed reps.  A rep opens
// with a domain barrier whose leader fences first (the previous check's clearing stores precede every peer's pushes),
// sums this rank's chunk (twoshot_chunk) of all P.n inputs with every warp of the grid and pushes each summed unit to
// every rank (ToGather).  Every CTA then passes a CTA barrier and issues one fence.sys, and a fenced domain barrier
// closes the rep: its release, stamped into rep[k][r].t_end, is when this rank's output is complete, so the rep runs
// from the opening release to the closing release.  The word check and clear follow, untimed (DESIGN §5i).  State
// lives in the rank's scratch buffer; outside it, only the gather areas and the barrier lines are written.
__global__ void __launch_bounds__(kThreads, 1) allreduce_twoshot_kernel(const __grid_constant__ TwoShotParams P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  ArScratch* as = P.scratch;
  BwScratch* bs = &as->rep;
  uint64_t* red;
  Ctx c = enter(smem, &bs->abort_flag, P.timeout_ns, &red);

  const uint32_t gwarp = blockIdx.x * kWarpsPerCta + c.warp;
  const uint32_t nwarps = gridDim.x * kWarpsPerCta;
  uint32_t b = 0;
  for (uint32_t k = 0; k < P.n_sizes; ++k) {
    const uint64_t bytes = P.size[k];
    uint64_t lo, hi;
    twoshot_chunk(units_of(bytes), P.n, P.rank, &lo, &hi);
    for (uint32_t r = 0; r <= P.reps; ++r) {
      if (!grid_barrier(c, bs, b++, &bs->t_rel[k][r], &P.dom, true)) return;
      const uint64_t fw = (r == 1u && k == P.fault_k) ? P.fault_word : ~0ull;
      Sum a{0ull, 0ull, 0ull};
      ar_units<ToGather>(c, P, bytes, Walk<false>{hi, lo + gwarp, 0ull, nwarps, nullptr}, fw, a);
      if (!close_fenced(c, bs, b++, &bs->rep[k][r].t_end, &P.dom)) return;
      ar_check_clear(c, P, reinterpret_cast<uint4*>(P.dst[0]), as, red, k, r, bytes, gwarp, nwarps);
    }
  }
}

int allreduce_twoshot_launch(const TwoShotParams& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  return grid_launch(allreduce_twoshot_kernel, p, grid, cooperative, stream);
}

}  // namespace cdp
