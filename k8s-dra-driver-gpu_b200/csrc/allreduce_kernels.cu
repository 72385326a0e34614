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
// none), every vector of the unit leaves with st.global.v4 and is folded into the (S, X) by its place in the output,
// and the accumulators are cleared for the next unit.
template <uint32_t kLaneBytes>
__device__ __forceinline__ void ar_store(const Ctx& c, uint8_t* out, uint64_t u, uint32_t len, uint64_t fw,
                                         uint64_t (&acc)[kArWords], Sum& a) {
  if (fw / (kUnitBytes / 8) == u) {  // rare: this unit holds the armed word
    const uint32_t fb = (uint32_t)(fw % (kUnitBytes / 8)) * 8u;
#pragma unroll
    for (int i = 0; i < kArWords / 2; ++i) {
      if (ar_vec_off<kLaneBytes>(c.lane, i) != (fb & ~15u)) continue;
      if (fb & 8u) acc[2 * i + 1] += 1ull;
      else acc[2 * i] += 1ull;
    }
  }
  uint8_t* base = out + u * kUnitBytes;
  uint64_t ux = 0;
#pragma unroll
  for (int i = 0; i < kArWords / 2; ++i) {
    const uint32_t off = ar_vec_off<kLaneBytes>(c.lane, i);
    const uint64_t w0 = acc[2 * i], w1 = acc[2 * i + 1];
    if (off < len) {
      stg_v4(reinterpret_cast<uint4*>(base + off),
             make_uint4((uint32_t)w0, (uint32_t)(w0 >> 32), (uint32_t)w1, (uint32_t)(w1 >> 32)));
      add_pair(a, ux, w0, w1);
    }
    acc[2 * i] = 0ull;
    acc[2 * i + 1] = 0ull;
  }
  fold_unit(a, ux, u);
}

// The one-shot's store policy (allreduce_path.cuh): a summed unit goes to the rank's own output, P.out.
struct ToOut {
  template <uint32_t kLaneBytes>
  __device__ __forceinline__ static void put(const Ctx& c, const AllReduceParams& P, uint64_t u, uint32_t len,
                                             uint64_t fw, uint64_t (&acc)[kArWords], Sum& a) {
    ar_store<kLaneBytes>(c, P.out, u, len, fw, acc, a);
  }
};
}  // namespace

// One rank of cdprobe_allreduce: for every size of the ladder, one warm-up and P.reps timed reps, each summing the
// first size bytes of all P.n inputs into P.out with every warp of the grid (the strided walk of a probe phase) and
// folding the sum into the (S, X) checksum.  A domain barrier opens every rep, so a rep is timed as a probe phase is,
// per rank: from this rank's release stamp to its latest CTA completion stamp (ranks see a release one signal latency
// apart).  After the last rep of a size and a grid barrier, the word check.  Its state (barrier, stamps, checksums,
// word-check counters, abort word) is in the rank's scratch buffer; outside it only its barrier lines are written.
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
      const Walk<false> walk = strided(bytes, gwarp, nwarps);
      ar_units<ToOut>(c, P, bytes, walk, fw, a);
      __threadfence();  // this warp's stores are performed before the CTA's completion stamp
      Acc* const acc = &bs->rep[k][r];
      cta_reduce<1>(c, red, &a, &acc);
      if (threadIdx.x == 0) atomicMax(&acc->t_end, (unsigned long long)gtimer());
    }
    if (!grid_barrier(c, bs, b++, nullptr, nullptr, false)) return;
    ar_check(c, P, as, k, bytes, gwarp, nwarps);
  }
}

int allreduce_launch(const AllReduceParams& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  return grid_launch(allreduce_kernel, p, grid, cooperative, stream);
}

template int granules_launch(uint64_t*, uint64_t*, const AllReduceWord&, uint64_t, unsigned, cudaStream_t);

}  // namespace cdp
