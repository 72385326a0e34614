// allreduce_kernels.cu — sm_90a kernels of cdprobe_allreduce's one-shot all-reduce: every warp streams one output unit
// of all n ranks' source buffers (TMA ring or ld.global.v4), adds them in registers and stores the sum with
// st.global.v4; each rep opens with a domain barrier (allreduce_kernel).  And the per-granule sums of the output that
// the expected checksums are folded from (granules_kernel<AllReduceWord>).  The shared data path is in datapath.cuh,
// the read-and-add side in allreduce_path.cuh.
//
// probe_kernels.cu is untouched: the probe kernel's code generation does not depend on this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "allreduce.h"
#include "allreduce_path.cuh"

namespace cdp {
namespace {
// Unit u of the output is complete in the accumulators: the armed fault goes in (fw, an output word index; ~0 when
// none), every vector of the unit leaves with st.global.v4, and the accumulators are cleared for the next unit.  The
// fault adds 1 to its word, or (P.fault_drop) nothing of its unit is stored.  Nothing is folded into (S, X): the word
// check reads the output back.
template <uint32_t kLaneBytes>
__device__ __forceinline__ void ar_store(const Ctx& c, const AllReduceParams& P, uint64_t u, uint32_t len, uint64_t fw,
                                         uint64_t (&acc)[kArWords]) {
  const bool hit = fw / (kUnitBytes / 8) == u;  // rare: this unit holds the armed word
  if (hit) {
    const uint32_t fb = (uint32_t)(fw % (kUnitBytes / 8)) * 8u;
#pragma unroll
    for (int i = 0; i < kArWords / 2; ++i) {
      if (ar_vec_off<kLaneBytes>(c.lane, i) != (fb & ~15u)) continue;
      if (fb & 8u) acc[2 * i + 1] += 1ull;
      else acc[2 * i] += 1ull;
    }
  }
  if (hit && P.fault_drop) len = 0;  // no vector of the unit is stored
  uint8_t* base = P.out + u * kUnitBytes;
  if (len == kUnitBytes) {  // a whole unit: every lane stores every vector, with no guard
#pragma unroll
    for (int i = 0; i < kArWords / 2; ++i)
      stg_pair(base + ar_vec_off<kLaneBytes>(c.lane, i), acc[2 * i], acc[2 * i + 1]);
  } else {
#pragma unroll
    for (int i = 0; i < kArWords / 2; ++i)
      if (ar_vec_off<kLaneBytes>(c.lane, i) < len)
        stg_pair(base + ar_vec_off<kLaneBytes>(c.lane, i), acc[2 * i], acc[2 * i + 1]);
  }
#pragma unroll
  for (int i = 0; i < kArWords; ++i) acc[i] = 0ull;
}

// The one-shot's store policy (allreduce_path.cuh): a summed unit goes to the rank's own output, P.out.
struct ToOut {
  template <uint32_t kLaneBytes>
  __device__ __forceinline__ static void put(const Ctx& c, const AllReduceParams& P, uint64_t u, uint32_t len,
                                             uint64_t fw, uint64_t (&acc)[kArWords], Sum&) {
    ar_store<kLaneBytes>(c, P, u, len, fw, acc);
  }
};
}  // namespace

// One rank of cdprobe_allreduce: for every size of the ladder, one warm-up and P.reps timed reps, each summing the
// first size bytes of all P.n inputs into P.out with every warp of the grid (the strided walk of a probe phase).  A
// domain barrier opens every rep, so a rep is timed as a probe phase is, per rank: from this rank's release stamp to its
// latest CTA completion stamp (ranks see a release one signal latency apart).  After every rep and a grid barrier, the
// word check and clear of the output (allreduce_path.cuh's ar_check_clear), untimed: the rep's (S, X) is folded from
// what the check read back, and a unit that a later rep does not store reads as 0s (DESIGN §5g).  Its state (barrier,
// stamps, checksums, word-check counters, abort word) is in the rank's scratch buffer; outside it only its barrier
// lines are written.
__global__ void __launch_bounds__(kThreads, 1) allreduce_kernel(const __grid_constant__ AllReduceParams P) {
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
    for (uint32_t r = 0; r <= P.reps; ++r) {
      if (!grid_barrier(c, bs, b++, &bs->t_rel[k][r], &P.dom, false)) return;
      const uint64_t fw = (r == 1u && k == P.fault_k) ? P.fault_word : ~0ull;
      Sum a{0ull, 0ull, 0ull};
      ar_units<ToOut>(c, P, bytes, strided(bytes, gwarp, nwarps), fw, a);
      __threadfence();  // this warp's stores are performed before the CTA's completion stamp
      __syncthreads();
      if (threadIdx.x == 0) atomicMax(&bs->rep[k][r].t_end, (unsigned long long)gtimer());
      if (!grid_barrier(c, bs, b++, nullptr, nullptr, false)) return;
      ar_check_clear(c, P, reinterpret_cast<uint4*>(P.out), as, red, k, r, bytes, gwarp, nwarps);
    }
  }
}

int allreduce_launch(const AllReduceParams& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  return grid_launch(allreduce_kernel, p, grid, cooperative, stream);
}

template int granules_launch(uint64_t*, uint64_t*, const AllReduceWord&, uint64_t, unsigned, cudaStream_t);

}  // namespace cdp
