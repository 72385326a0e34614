// allreduce_nvls_kernels.cu — sm_90a kernel of cdprobe_allreduce_nvls's multicast all-reduce: every rank reduces its
// chunk of units (the two-shot's) by multimem.ld_reduce .add.u64 through the multicast object's input half, so the
// fabric returns the sum of the word across every member's memory, and writes each summed 16 bytes to every member at
// once with one multimem.st through the object's output half; a fenced domain barrier closes the rep, and every rank
// checks and clears its own output half through its unicast mapping (allreduce_nvls_kernel, with allreduce_path.cuh's
// ar_check_clear).  Unicast and multicast addresses alias the same memory, so every hand-over between them passes a
// fence.proxy.alias (DESIGN §5m).
//
// probe_kernels.cu is untouched: the probe kernel's code generation does not depend on this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "allreduce_nvls.h"
#include "allreduce_path.cuh"

namespace cdp {
namespace {
// The wrapping 64-bit sum of the word at mc over every member of the multicast object.  There is no vector form of
// the integer reduction (the .v2/.v4 forms take floating-point types only), so the exact sum costs one 8-byte request
// per word.
__device__ __forceinline__ uint64_t mc_ld_reduce_add_u64(const void* mc) {
  uint64_t v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.u64 %0, [%1];" : "=l"(v) : "l"(mc) : "memory");
  return v;
}
// One 16-byte store into every member's memory at mc.  The .f32 type only names the vector's width: the bits are
// stored as they are, and no arithmetic touches them.
__device__ __forceinline__ void mc_st_v4(void* mc, uint64_t w0, uint64_t w1) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "r"((uint32_t)w0),
               "r"((uint32_t)(w0 >> 32)), "r"((uint32_t)w1), "r"((uint32_t)(w1 >> 32))
               : "memory");
}
// Orders this thread's accesses through one virtual address before its later accesses to the same memory through an
// aliasing one (the multicast and the unicast mapping of the output half, the copied input).
__device__ __forceinline__ void fence_proxy_alias() { asm volatile("fence.proxy.alias;" ::: "memory"); }

// The reduce and store of one rank's chunk, by one warp over the units of `walk`: each lane reduces the two words of
// each of its 16-byte vectors of the unit (the ld/st layout, ar_vec_off<16>), all of them before the first store, and
// stores each pair with one multimem.st.  The armed fault (fw, an output word index; ~0 when none) stores that word
// xored with 1 (mode 0) or skips every store of its unit (mode 1).
__device__ void reduce_store(const Ctx& c, const NvlsParams& P, uint64_t bytes, Walk<false> walk, uint64_t fw) {
  const uint64_t fu = fw / (kUnitBytes / 8);
  const uint32_t fb = (uint32_t)(fw % (kUnitBytes / 8)) * 8u;
  for (uint64_t u; walk.take(c, u);) {
    const uint32_t len = unit_len(bytes, u);
    const bool hit = u == fu;
    if (hit && P.fault_mode == 1u) continue;
    const uint8_t* const in = P.mc_in + u * kUnitBytes;
    uint8_t* const out = P.mc_out + u * kUnitBytes;
    uint64_t w[2 * kLdstVecs];
#pragma unroll
    for (int i = 0; i < (int)kLdstVecs; ++i) {
      const uint32_t off = ar_vec_off<16>(c.lane, i);
      w[2 * i] = w[2 * i + 1] = 0ull;
      if (off < len) {
        w[2 * i] = mc_ld_reduce_add_u64(in + off);
        w[2 * i + 1] = mc_ld_reduce_add_u64(in + off + 8);
      }
    }
#pragma unroll
    for (int i = 0; i < (int)kLdstVecs; ++i) {
      const uint32_t off = ar_vec_off<16>(c.lane, i);
      if (off >= len) continue;
      uint64_t w0 = w[2 * i], w1 = w[2 * i + 1];
      if (hit && off == (fb & ~15u)) {
        if (fb & 8u) w1 ^= 1ull;
        else w0 ^= 1ull;
      }
      mc_st_v4(out + off, w0, w1);
    }
  }
}
}  // namespace

// One rank of cdprobe_allreduce_nvls: for every size of the ladder, one warm-up and P.reps timed reps.  A rep opens
// with a domain barrier whose leader fences first (every rank's previous check and clear precede every multicast
// store), whose release is stamped into t_rel[k][r].  Every warp then reduces and stores its strided units of this
// rank's chunk (twoshot_chunk).  Every thread passes a fence.proxy.alias, the CTA a CTA barrier and one fence.sys,
// and a fenced domain barrier closes the rep: its release, stamped into rep[k][r].t_end, is when this rank's output
// is complete, in every rank's memory.  That fence.proxy.alias is inside the timed window, so its cost is part of
// every reported time.  The word check and clear follow through the unicast mapping, untimed, and one more
// fence.proxy.alias per thread (DESIGN §5m).  State lives in the rank's scratch buffer; outside it, only the output
// halves and the barrier lines are written.
__global__ void __launch_bounds__(kThreads, 1) allreduce_nvls_kernel(const __grid_constant__ NvlsParams P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  ArScratch* as = P.scratch;
  BwScratch* bs = &as->rep;
  uint64_t* red;
  Ctx c = enter(smem, &bs->abort_flag, P.timeout_ns, &red);
  fence_proxy_alias();  // the host copied the input and zeroed the output through the unicast mapping

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
      reduce_store(c, P, bytes, Walk<false>{hi, lo + gwarp, 0ull, nwarps, nullptr}, fw);
      fence_proxy_alias();  // the multicast stores, before the unicast check reads the same memory
      __syncthreads();
      if (threadIdx.x == 0) __threadfence_system();  // every store of this CTA has reached every member
      if (!grid_barrier(c, bs, b++, &bs->rep[k][r].t_end, &P.dom, true)) return;
      ar_check_clear(c, P, reinterpret_cast<uint4*>(P.out), as, red, k, r, bytes, gwarp, nwarps);
      fence_proxy_alias();  // the unicast clear, before the next rep stores through the multicast address
    }
  }
}

int allreduce_nvls_launch(const NvlsParams& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  return grid_launch(allreduce_nvls_kernel, p, grid, cooperative, stream);
}

}  // namespace cdp
