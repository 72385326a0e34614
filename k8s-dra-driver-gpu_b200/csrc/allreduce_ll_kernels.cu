// allreduce_ll_kernels.cu — sm_90a kernel of cdprobe_allreduce_ll's low-latency all-reduce: every 64-bit input word
// travels to every peer as one 16-byte packet of two flag-carrying 8-byte elements (st.relaxed.sys.v2.u64), and the
// receiver polls its own LL area (ld.relaxed.sys.v2.u64) until both flags of each packet are the rep's; no barrier and
// no fence inside a size (allreduce_ll_kernel).  The word check and clear of the output after each size is
// allreduce_path.cuh's ar_check.
//
// probe_kernels.cu is untouched: the probe kernel's code generation does not depend on this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "allreduce_ll.h"
#include "allreduce_path.cuh"

namespace cdp {
namespace {
// One packet: two 8-byte elements, each single-copy atomic on its own (DESIGN §5j).
__device__ __forceinline__ void st_packet(uint8_t* p, uint64_t e0, uint64_t e1) {
  asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(e0), "l"(e1) : "memory");
}
__device__ __forceinline__ void ld_packet(const uint8_t* p, uint64_t& e0, uint64_t& e1) {
  asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];" : "=l"(e0), "=l"(e1) : "l"(p) : "memory");
}

// Rep r of size k at this rank, by warp gwarp of the nwarps = kWarpsPerCta x P.ctas that move words: lane l of the warp
// owns word 32 i + l of every line i = gwarp, gwarp + nwarps, ... of the size, the same words at every rank.  Pushes
// them to every peer, then sums this rank's input and every peer's packets into the output, folded into a.  Returns
// false once the launch is aborted (a poll passed the deadline or saw the abort).
__device__ bool ll_rep(const Ctx& c, const LlParams& P, uint32_t k, uint32_t r, uint64_t bytes, uint32_t gwarp,
                       uint32_t nwarps, Sum& a) {
  const uint64_t words = bytes / 8, lines = (words + 31) / 32;
  const uint32_t p = r & 1u, n = P.n, g = P.rank;
  const uint32_t flag = ll_flag(P.dom.call_seq, k, r);
  const uint64_t hi = (uint64_t)flag << 32;
  const uint64_t salt = ll_salt(P.seed, g, flag);
  const unsigned long long* src = reinterpret_cast<const unsigned long long*>(P.src);
  const bool armed = r == 1u && k == P.fault_k;
  if (armed && P.fault_mode == 1u) delay_us(P.fault_arg);
  const uint64_t fw = armed && P.fault_mode == 0u ? P.fault_arg : ~0ull;
  const uint64_t nw = k == P.fault_k && P.fault_mode == 2u ? P.fault_arg : ~0ull;  // mode 2: the word left unstored

  // 1. push: one packet per owned word to rank g + 1, g + 2, ... (mod n)
  for (uint64_t i = gwarp; i < lines; i += nwarps) {
    const uint64_t w = i * 32u + (uint32_t)c.lane;
    if (w >= words) break;
    const uint64_t v = __ldg(src + w) + salt;
    const uint64_t off = ll_slot(p, n, g, P.s_max, w);
    for (uint32_t t = 1; t < n; ++t) {
      const uint64_t d = (w == fw && t == P.fault_dst) ? v ^ 1ull : v;
      st_packet(P.dst[t] + off, (d & 0xffffffffull) | hi, (d >> 32) | hi);
    }
  }

  // 2-5. this rank's input, then every peer's packets as they arrive (rank g - 1, g - 2, ...: the order in which
  // they push to g), less the salts, into the output and (S, X)
  uint64_t salts = 0;
  for (uint32_t j = 0; j < n; ++j) salts += ll_salt(P.seed, j, flag);
  uint64_t* out = reinterpret_cast<uint64_t*>(P.out);
  for (uint64_t i = gwarp; i < lines; i += nwarps) {
    const uint64_t w = i * 32u + (uint32_t)c.lane;
    if (w >= words) break;
    uint64_t acc = __ldg(src + w) + salt;
    for (uint32_t t = 1; t < n; ++t) {
      const uint8_t* q = P.in + ll_slot(p, n, g >= t ? g - t : g + n - t, P.s_max, w);
      uint64_t e0, e1;
      uint32_t spins = 0;
      for (;;) {
        ld_packet(q, e0, e1);
        if ((uint32_t)(e0 >> 32) == flag && (uint32_t)(e1 >> 32) == flag) break;
        if ((++spins & 63u) == 0u && check_abort(c)) return false;
      }
      acc += (e0 & 0xffffffffull) | (e1 << 32);
    }
    const uint64_t v = acc - salts;
    if (w != nw) out[w] = v;
    a.s0 += v;
    a.x ^= rotl64(v, fold6((uint32_t)(i / (kGranuleWords / 32))));
  }
  return true;
}
}  // namespace

// One rank of cdprobe_allreduce_ll: for every size of the ladder, a domain barrier whose release stamps t_rel[k][0],
// then one warm-up and P.reps timed reps back to back with no barrier between them (ll_rep; rep r uses parity r % 2 of
// the LL area).  A CTA's rep ends when its stores of the output are performed: its stamp goes into rep[k][r].t_end and
// into t_rel[k][r + 1], where the next rep is timed from, so a rep runs from the end of this rank's previous rep to the
// end of its own.  After the last rep of a size and a grid barrier, the word check and clear of the output (ar_check),
// so the next size, and the next call, finds 0s wherever it stores nothing.  CTAs from P.ctas on only join the
// barriers and the check.  State lives in the rank's scratch buffer; outside it, only the peers' LL areas
// and the barrier lines are written.
__global__ void __launch_bounds__(kThreads, 1) allreduce_ll_kernel(const __grid_constant__ LlParams P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  ArScratch* as = P.scratch;
  BwScratch* bs = &as->rep;
  uint64_t* red;
  Ctx c = enter(smem, &bs->abort_flag, P.timeout_ns, &red);

  const uint32_t gwarp = blockIdx.x * kWarpsPerCta + c.warp;
  const bool moves = blockIdx.x < P.ctas;
  uint32_t b = 0;
  for (uint32_t k = 0; k < P.n_sizes; ++k) {
    const uint64_t bytes = P.size[k];
    if (!grid_barrier(c, bs, b++, &bs->t_rel[k][0], &P.dom, false)) return;
    for (uint32_t r = 0; moves && r <= P.reps; ++r) {
      Sum a{0ull, 0ull, 0ull};
      const bool ok = ll_rep(c, P, k, r, bytes, gwarp, P.ctas * kWarpsPerCta, a);
      if (__syncthreads_or(!ok)) return;  // the deadline passed or a peer's CTA aborted: every CTA stops
      __threadfence();                    // this CTA's output stores are performed before its completion stamp
      Acc* const acc = &bs->rep[k][r];
      cta_reduce<1>(c, red, &a, &acc);
      if (threadIdx.x == 0) {
        const unsigned long long t = gtimer();
        atomicMax(&acc->t_end, t);
        if (r < P.reps) atomicMax(&bs->t_rel[k][r + 1], t);
      }
    }
    if (!grid_barrier(c, bs, b++, nullptr, nullptr, false)) return;
    ar_check(c, P, as, k, bytes, gwarp, gridDim.x * kWarpsPerCta);
  }
}

int allreduce_ll_launch(const LlParams& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  return grid_launch(allreduce_ll_kernel, p, grid, cooperative, stream);
}

}  // namespace cdp
