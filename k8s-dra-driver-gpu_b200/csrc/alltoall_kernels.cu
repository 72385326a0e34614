// alltoall_kernels.cu — sm_90a kernel of cdprobe_alltoall's one-shot all-to-all: every warp pushes interleaved units of
// the rank's blocks into the receivers' exchange areas through the probe's K2 write path (datapath.cuh); each rep sits
// between two domain barriers and is followed by the word check of the blocks received (alltoall_kernel).
//
// probe_kernels.cu is untouched: the probe kernel's code generation does not depend on this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "alltoall.h"
#include "datapath.cuh"

namespace cdp {
namespace {
// The all-to-all's push: one strided walk over blocks x units_of(bytes) units, interleaved so that every target is in
// flight at once.  Walk unit t is unit t / blocks of block t % blocks, which goes to P.dst[b] with the write salt of
// (rank -> to[b]) in rep `seq`.  take() stops once the launch is aborted (checked every 16 units per warp), so a rank
// whose peer is gone stops issuing; the write job then drains what it issued.
struct BlockWalk {
  static constexpr bool kSpread = true;
  Walk<false> w;
  const AllToAllParams* P;
  uint64_t seq;
  uint32_t taken;
  __device__ __forceinline__ bool take(const Ctx& c, uint64_t& t) {
    if ((++taken & 15u) == 0u) {
      bool ab = false;
      if (c.lane == 0) ab = check_abort(c);
      if (__shfl_sync(0xffffffffu, ab, 0)) return false;
    }
    return w.take(c, t);
  }
  __device__ __forceinline__ void place(uint64_t& u, uint8_t*& base, uint64_t& salt) const {
    const uint32_t t = (uint32_t)u, b = t % P->blocks;
    u = t / P->blocks;
    base = P->dst[b];
    salt = write_salt(P->seed, P->rank, P->to[b], seq);
  }
};

// The armed fault: after its stores of timed rep 1 of size fault_k are complete, the warp that wrote word fault_word
// of block fault_block stores that word again xored with 1, so the receiver reads it as a fault in transit.  The
// strided walk hands walk unit t to warp t % nwarps.
__device__ __noinline__ void a2a_fault(const AllToAllParams& P, uint64_t seq, uint32_t gwarp, uint32_t nwarps,
                                       int lane) {
  const uint64_t t = (P.fault_word / (kUnitBytes / 8)) * P.blocks + P.fault_block;
  if (t % nwarps != gwarp || lane != 0) return;
  fence_proxy_async_global();  // the word may have been stored by a bulk copy
  const uint64_t salt = write_salt(P.seed, P.rank, P.to[P.fault_block], seq);
  *reinterpret_cast<volatile uint64_t*>(P.dst[P.fault_block] + 8 * P.fault_word) = write_word(salt, P.fault_word) ^ 1ull;
}

// Adds what one warp found in the blocks of sender slot i into the receiver's counters: bad words, the lowest bad
// offset and, on the last timed rep (fold), the (S, X) parts.
__device__ __forceinline__ void a2a_flush(const AllToAllParams& P, A2aScratch* as, uint32_t i, uint32_t k, bool fold,
                                          int lane, uint64_t bad, uint64_t first, uint64_t s, uint64_t x) {
  bad = warp_sum64(bad);
  if (bad != 0) first = warp_min64(first);
  if (fold) {
    s = warp_sum64(s);
    x = warp_xor64(x);
  }
  if (lane != 0) return;
  const uint32_t from = P.from[i];
  if (bad != 0) {
    atomicAdd(&as->bad_words[from][k], (unsigned long long)bad);
    atomicMax(&as->first_bad_n[from][k], (unsigned long long)~first);
  }
  if (fold) {
    atomicAdd(&as->sum[from][k], (unsigned long long)s);
    atomicXor(&as->xr[from][k], (unsigned long long)x);
  }
}

// The word check of rep r of size k: every word of every incoming block is compared with the pattern its sender
// stored.  Walk unit t is unit t % units of incoming block t / units, so a warp's units mostly share a sender and its
// counters are flushed when the sender changes.  Loads go to L2 (peers stored the words).  On the last timed rep the
// words are also folded into the cell's (S, X): the X part of unit u is rotl64(xor of its words, fold6(u / 2)), which
// is fold_unit's, so the parts xor together into the checksum of the block.
__device__ void a2a_check(const Ctx& c, const AllToAllParams& P, A2aScratch* as, uint32_t k, uint32_t r,
                          uint64_t bytes, uint32_t gwarp, uint32_t nwarps) {
  const uint32_t units = (uint32_t)units_of(bytes);
  const bool fold = r == P.reps;
  const uint64_t seq = alltoall_seq(P.dom.call_seq, k, r);
  Walk<false> walk{(uint64_t)P.n_in * units, gwarp, 0ull, nwarps, nullptr};
  uint32_t cur = ~0u;
  uint64_t bad = 0, first = ~0ull, s = 0, x = 0, salt = 0;
  for (uint64_t t; walk.take(c, t);) {
    const uint32_t i = (uint32_t)t / units, u = (uint32_t)t % units;
    if (i != cur) {
      if (cur != ~0u) a2a_flush(P, as, cur, k, fold, c.lane, bad, first, s, x);
      if (aborted(c)) return;
      cur = i;
      bad = s = x = 0;
      first = ~0ull;
      salt = write_salt(P.seed, P.from[i], P.rank, seq);
    }
    const uint4* p = reinterpret_cast<const uint4*>(P.in[i] + (uint64_t)u * kUnitBytes);
    const uint32_t nvec = unit_len(bytes, u) / 16;
    const uint64_t w_base = (uint64_t)u * (kUnitBytes / 8);
    uint64_t ux = 0;
#pragma unroll 4
    for (uint32_t v = c.lane; v < nvec; v += 32) {
      const uint4 q = ldg_stream_v4(p + v);
      const uint64_t w0 = pack64(q.x, q.y), w1 = pack64(q.z, q.w), k0 = w_base + 2 * v;
      if (w0 != write_word(salt, k0)) {
        ++bad;
        first = min(first, 8 * k0);
      }
      if (w1 != write_word(salt, k0 + 1)) {
        ++bad;
        first = min(first, 8 * k0 + 8);
      }
      s += w0 + w1;
      ux ^= w0 ^ w1;
    }
    x ^= rotl64(ux, fold6(u / (kGranuleBytes / kUnitBytes)));
  }
  if (cur != ~0u) a2a_flush(P, as, cur, k, fold, c.lane, bad, first, s, x);
}
}  // namespace

// One rank of cdprobe_alltoall: for every size of the ladder, one warm-up and P.reps timed reps.  A rep opens with a
// domain barrier, pushes the first size bytes of each of the rank's blocks into its receivers' exchange areas with every
// warp of the grid (BlockWalk, on the probe's write path), and is timed as a probe write phase is: every CTA completes
// its stores, passes a CTA barrier and issues one fence.sys, then stamps; the rep runs from the release stamp to the
// latest CTA stamp.  An untimed domain barrier, whose leader fences before signalling, then makes the blocks this rank
// receives visible, and the word check reads them (DESIGN §5h).  State lives in the rank's scratch buffer; outside it,
// only its blocks and its barrier lines are written.
__global__ void __launch_bounds__(kThreads, 1) alltoall_kernel(const __grid_constant__ AllToAllParams P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  A2aScratch* as = P.scratch;
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
      const uint64_t seq = alltoall_seq(P.dom.call_seq, k, r);
      Sum a{0ull, 0ull, 0ull};
      if (P.blocks != 0) {
        const BlockWalk walk{{(uint64_t)P.blocks * units_of(bytes), gwarp, 0ull, nwarps, nullptr}, &P, seq, 0u};
        write_units(c, P.path, nullptr, bytes, walk, 0ull, a);
        if (c.lane == 0) fence_proxy_async_global();  // bulk stores, then generic loads and stores of the same words
        __syncwarp();
        if (r == 1u && k == P.fault_k) a2a_fault(P, seq, gwarp, nwarps, c.lane);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        __threadfence_system();  // every store of this CTA has reached its receiver
        atomicMax(&bs->rep[k][r].t_end, (unsigned long long)gtimer());
      }
      if (!grid_barrier(c, bs, b++, nullptr, &P.dom, true)) return;
      a2a_check(c, P, as, k, r, bytes, gwarp, nwarps);
    }
  }
}

int alltoall_launch(const AllToAllParams& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  return grid_launch(alltoall_kernel, p, grid, cooperative, stream);
}

}  // namespace cdp
