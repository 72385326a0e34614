// allreduce_ring_kernels.cu — sm_90a kernel of cdprobe_allreduce_ring's ring all-reduce: rank g passes every 8 KiB
// unit of the two-shot's chunks to rank g + 1 in 2 (n - 1) dependent steps, a reduce-scatter and then an all-gather.
// A unit's data goes with st.global.v4 into the successor's ring area and is published by a per-unit flag
// (st.release.sys) that the successor polls (ld.acquire.sys); no barrier and no fence across the domain between the
// steps (allreduce_ring_kernel).  The word check and clear is the two-shot's (allreduce_path.cuh).
//
// probe_kernels.cu is untouched: the probe kernel's code generation does not depend on this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "allreduce_path.cuh"
#include "allreduce_ring.h"

namespace cdp {
namespace {
__device__ __forceinline__ void st_flag(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_flag(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Lane 0 polls the flag at p until it holds `want`, checking the abort and the deadline every 64 spins; the warp
// barrier then orders every lane's reads of the grain after that acquire.  Returns false in every lane once the launch
// is aborted.
__device__ __forceinline__ bool wait_flag(const Ctx& c, const uint32_t* p, uint32_t want) {
  bool ok = true;
  if (c.lane == 0) {
    uint32_t spins = 0;
    while (ld_flag(p) != want) {
      if ((++spins & 63u) == 0u && check_abort(c)) {
        ok = false;
        break;
      }
    }
  }
  __syncwarp();
  return __shfl_sync(0xffffffffu, ok, 0);
}

// What one step does with a unit at this rank: add what the predecessor pushed into this rank's area (recv) and this
// rank's own input (src), store the sum into this rank's output (own), push it to the successor's area (push) in
// `phase` (0 the reduce-scatter, 1 the all-gather).
struct Step {
  bool recv, src, own, push;
  uint32_t phase;
};

// Unit u of a step, by the warp: lane l moves the 16-byte vectors at ar_vec_off<16>(l, i).  The push of word xw
// (~0: none) leaves xored with 1; drop: the push stores nothing.
__device__ __forceinline__ void ring_unit(const Ctx& c, const RingParams& P, uint64_t bytes, uint64_t u,
                                          const Step& st, uint64_t xw, bool drop) {
  const uint32_t len = unit_len(bytes, u);
  const uint64_t base = u * kUnitBytes;
  const uint32_t hit = xw / (kUnitBytes / 8) == u ? (uint32_t)(xw % (kUnitBytes / 8)) * 8u : ~0u;
  uint64_t acc[kArWords];
#pragma unroll
  for (int i = 0; i < kArWords; ++i) acc[i] = 0ull;
#pragma unroll
  for (int i = 0; i < kArWords / 2; ++i) {
    const uint32_t off = ar_vec_off<16>(c.lane, i);
    if (off >= len) continue;
    if (st.recv) ar_add(acc, i, __ldcg(reinterpret_cast<const uint4*>(P.out + base + off)));
    if (st.src) ar_add(acc, i, ldg_stream_v4(reinterpret_cast<const uint4*>(P.src + base + off)));
  }
#pragma unroll
  for (int i = 0; i < kArWords / 2; ++i) {
    const uint32_t off = ar_vec_off<16>(c.lane, i);
    if (off >= len) continue;
    uint64_t w0 = acc[2 * i], w1 = acc[2 * i + 1];
    if (st.own) stg_pair(P.out + base + off, w0, w1);
    if (!st.push || drop) continue;
    if (off == (hit & ~15u)) {
      if (hit & 8u) w1 ^= 1ull;
      else w0 ^= 1ull;
    }
    stg_pair(P.next + base + off, w0, w1);
  }
}

// Rep r of size k at this rank g, by warp gwarp of nwarps.  Steps s = 0 .. 2 (n - 1), on chunk (g - 1 - s) mod n in
// the reduce-scatter (s < n - 1) and chunk (g - (s - n + 1)) mod n from then on:
//   s = 0:               push this rank's input;
//   0 < s < n - 1:       wait for the partial, push it plus this rank's input;
//   s = n - 1:           wait for the partial, store it plus this rank's input (the full sum of chunk g) into the
//                        output and push it, the all-gather's first push;
//   n - 1 < s < 2 (n-1): wait for the full chunk, which landed in the output, and push it on;
//   s = 2 (n - 1):       wait for the last full chunk (g + 1); nothing to push.
// At n = 1 the one step stores this rank's input into its output.  The warp owns grains j = gwarp, gwarp + nwarps, ...
// of kRingFlagUnits units counted from each chunk's start, and takes its (j, s) in lexicographic order; item (g, j, s)
// waits only on (g - 1, j, s - 1) (DESIGN §5k).  Returns false once the launch is aborted.
__device__ bool ring_rep(const Ctx& c, const RingParams& P, uint32_t k, uint32_t r, uint64_t bytes, uint32_t gwarp,
                         uint32_t nwarps) {
  const uint32_t n = P.n, g = P.rank, rs = n - 1, last = 2 * rs;
  const uint64_t units = units_of(bytes), span = (units + n - 1) / n;  // the longest chunk
  const uint32_t f0 = ring_flag(P.dom.call_seq, k, r, 0), f1 = ring_flag(P.dom.call_seq, k, r, 1);
  const uint32_t* const in_flags = reinterpret_cast<const uint32_t*>(P.out + ring_flags_off(P.s_max));
  uint32_t* const out_flags = reinterpret_cast<uint32_t*>(P.next + ring_flags_off(P.s_max));
  const bool armed = r == 1u && k == P.fault_k;
  if (armed && P.fault_mode == 2u) delay_us(P.fault_arg);
  const uint64_t fw = armed && P.fault_mode < 2u ? P.fault_arg : ~0ull;
  for (uint64_t j = gwarp; j * kRingFlagUnits < span; j += nwarps) {
    for (uint32_t s = 0; s <= last; ++s) {
      const uint32_t ch = s < rs ? (g + n - 1 - s) % n : (g + n - (s - rs)) % n;
      uint64_t lo, hi;
      twoshot_chunk(units, n, ch, &lo, &hi);
      const uint64_t u0 = lo + j * kRingFlagUnits;
      if (u0 >= hi) continue;  // this chunk is shorter than the longest
      const uint64_t u1 = min(hi, u0 + kRingFlagUnits);
      const Step st{s > 0, s <= rs, s == rs, s < last, s >= rs ? 1u : 0u};
      if (st.recv && !wait_flag(c, in_flags + u0, s > rs ? f1 : f0)) return false;
      if (s == last && s != rs) continue;  // the last chunk has arrived in the output
      const uint64_t xw = st.push && st.phase == P.fault_phase ? fw : ~0ull;
      const bool drop = P.fault_mode == 1u && xw / (kUnitBytes / 8) - u0 < u1 - u0;
      for (uint64_t u = u0; u < u1; ++u) ring_unit(c, P, bytes, u, st, P.fault_mode == 0u ? xw : ~0ull, drop);
      if (st.push) {
        __syncwarp();  // every lane's stores of the grain precede lane 0's release
        if (c.lane == 0) st_flag(out_flags + u0, st.phase ? f1 : f0);
      }
    }
  }
  return true;
}
}  // namespace

// One rank of cdprobe_allreduce_ring: for every size of the ladder, one warm-up and P.reps timed reps.  A rep opens
// with a domain barrier whose leader fences first (the previous check's clearing stores precede every peer's pushes)
// and whose release is stamped into t_rel[k][r]; the ring's steps follow (ring_rep).  A CTA's part of the rep ends
// when its pushes are issued and its output stores performed: its stamp goes into rep[k][r].t_end, so a rep runs
// from the opening release to the moment this rank's output is complete.  After a grid barrier, the word check and
// clear of the output, untimed (DESIGN §5k).  State lives in the rank's scratch buffer; outside it, only the
// successor's ring area and the barrier lines are written.
__global__ void __launch_bounds__(kThreads, 1) allreduce_ring_kernel(const __grid_constant__ RingParams P) {
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
      if (!grid_barrier(c, bs, b++, &bs->t_rel[k][r], &P.dom, true)) return;
      const bool ok = ring_rep(c, P, k, r, bytes, gwarp, nwarps);
      if (__syncthreads_or(!ok)) return;  // the deadline passed or a peer's CTA aborted: every CTA stops
      __threadfence();                    // this CTA's output stores are performed before its completion stamp
      if (threadIdx.x == 0) atomicMax(&bs->rep[k][r].t_end, gtimer());
      if (!grid_barrier(c, bs, b++, nullptr, nullptr, false)) return;
      ar_check_clear(c, P, reinterpret_cast<uint4*>(P.out), as, red, k, r, bytes, gwarp, nwarps);
    }
  }
}

int allreduce_ring_launch(const RingParams& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  return grid_launch(allreduce_ring_kernel, p, grid, cooperative, stream);
}

}  // namespace cdp
