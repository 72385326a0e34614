// allreduce_path.cuh — the read-and-add side of the all-reduce kernels, shared by allreduce_kernel (one-shot,
// allreduce_kernels.cu) and allreduce_twoshot_kernel (allreduce_twoshot_kernels.cu): every warp walks 8 KiB output
// units, streams unit u of all P.n inputs (TMA ring or ld.global.v4) and adds them in registers (64-bit, wrapping).
// Two things are parameters: the walk (which units a warp sums) and the store policy (where a summed unit goes).
// Also the word check and clear of allreduce_ll_kernel's output after the last rep of a size (ar_check,
// allreduce_ll_kernels.cu), and the word check and clear of an output after every rep (ar_check_clear), shared by the
// one-shot, the two-shot, allreduce_ring_kernel (allreduce_ring_kernels.cu) and allreduce_nvls_kernel.  And the pieces
// the all-reduce kernels share around those: the store of a unit to several ranks (put_ranks, the two-shot's and the
// push's store policies), the pair store (stg_pair, also the one-shot's and the ring's), the armed delay (delay_us, the
// LL's and the ring's) and the fenced close of a phase (close_fenced, the two-shot's and the push's).
//
// A store policy S has one member, called once per unit by every lane with the unit's sums in acc:
//   template <uint32_t kLaneBytes> static void S::put(const Ctx&, const Params& P, uint64_t u, uint32_t len,
//                                                      uint64_t fw, uint64_t (&acc)[kArWords], Sum& a)
// It stores the len bytes of unit u, lane vector i at ar_vec_off<kLaneBytes>(lane, i), and leaves acc all zero.  fw is
// the word index of the armed fault (~0: none).
//
// Internal linkage, as datapath.cuh: each unit that includes this header compiles its own copy.
#pragma once
#include <stdint.h>

#include "allreduce.h"
#include "datapath.cuh"

namespace cdp {
namespace {
constexpr int kArWords = 2 * kLdstVecs;  // uint64 accumulators per lane: a warp holds one 8 KiB output unit

// Byte offset in a unit of the lane's 16-byte vector i when each access moves kLaneBytes contiguous bytes: the layout
// job_read_ldst loads in, and for kLaneBytes = 16 also the one job_read_tma reads a stage in.
template <uint32_t kLaneBytes>
__device__ __forceinline__ uint32_t ar_vec_off(int lane, int i) {
  constexpr int kV = kLaneBytes / 16;
  return kLaneBytes * (uint32_t)lane + 32u * kLaneBytes * (uint32_t)(i / kV) + 16u * (uint32_t)(i % kV);
}

__device__ __forceinline__ void ar_add(uint64_t (&acc)[kArWords], int i, const uint4& v) {
  acc[2 * i] += pack64(v.x, v.y);
  acc[2 * i + 1] += pack64(v.z, v.w);
}

// Two 64-bit words to global memory at p with one st.global.v4.
__device__ __forceinline__ void stg_pair(uint8_t* p, uint64_t w0, uint64_t w1) {
  stg_v4(reinterpret_cast<uint4*>(p),
         make_uint4((uint32_t)w0, (uint32_t)(w0 >> 32), (uint32_t)w1, (uint32_t)(w1 >> 32)));
}

// A store policy's body for a unit that goes to several ranks: the summed unit u (len bytes, lane vector i at
// ar_vec_off<kLaneBytes>(lane, i)) goes to P.dst[t0], P.dst[t0 + 1], ..., P.dst[P.n - 1], and acc is cleared.  The
// armed fault (fw, an output word index; ~0 when none) acts on the stores to P.dst[P.fault_dst] only: the word leaves
// xored with 1, or (kDrop, for parameters with a fault_drop, and P.fault_drop) nothing of its unit goes there.  The
// xor is written out here and in the ring's ring_unit rather than in a helper of its own: as a separate inline
// function it compiled to a branch around every vector's store instead of predicated instructions, and this form
// compiles to the same SASS as the store policies it replaced.
template <uint32_t kLaneBytes, bool kDrop, typename Params>
__device__ __forceinline__ void put_ranks(const Ctx& c, const Params& P, uint32_t t0, uint64_t u, uint32_t len,
                                          uint64_t fw, uint64_t (&acc)[kArWords]) {
  const uint32_t hit_dst = fw / (kUnitBytes / 8) == u ? P.fault_dst : ~0u;  // rare: this unit holds the armed word
  const uint32_t fb = (uint32_t)(fw % (kUnitBytes / 8)) * 8u;
  for (uint32_t t = t0; t < P.n; ++t) {
    if constexpr (kDrop) {
      if (t == hit_dst && P.fault_drop) continue;
    }
    uint8_t* base = P.dst[t] + u * kUnitBytes;
#pragma unroll
    for (int i = 0; i < kArWords / 2; ++i) {
      const uint32_t off = ar_vec_off<kLaneBytes>(c.lane, i);
      if (off >= len) continue;
      uint64_t w0 = acc[2 * i], w1 = acc[2 * i + 1];
      if (t == hit_dst && off == (fb & ~15u)) {
        if (fb & 8u) w1 ^= 1ull;
        else w0 ^= 1ull;
      }
      stg_pair(base + off, w0, w1);
    }
  }
#pragma unroll
  for (int i = 0; i < kArWords; ++i) acc[i] = 0ull;
}

// The armed delay of the LL and ring kernels: spins until `us` microseconds have passed (below timeout_ms / 2, which
// the host checks).
__device__ __forceinline__ void delay_us(uint64_t us) {
  const uint64_t until = gtimer() + us * 1000u;
  while (gtimer() < until) {
  }
}

// Closes a phase whose stores go to peers (the two-shot and the push): after a CTA barrier, thread 0 issues one
// fence.sys, so every store of the CTA has reached its peer before the fenced domain barrier b signals; its release
// is stamped into *stamp (unless null).  Returns false in every thread once the launch is aborted.
__device__ __forceinline__ bool close_fenced(const Ctx& c, BwScratch* bs, uint32_t b, unsigned long long* stamp,
                                             const DomainLines* dom) {
  __syncthreads();
  if (threadIdx.x == 0) __threadfence_system();
  return grid_barrier(c, bs, b, stamp, dom, true);
}

// TMA read side: the warp walks (unit, input) pairs, the n inputs of a unit in a row, through its kStages-deep ring of
// bulk loads, one load per pair.  Each stage is added into the accumulators and then refilled with the next pair, so
// the ring runs on across unit boundaries.  Aborted: stops issuing and drains what is in flight.
template <typename Store, typename Params>
__device__ void ar_units_tma(Ctx& c, const Params& P, uint64_t bytes, Walk<false> walk, uint64_t fw, Sum& a) {
  const uint32_t n = P.n;
  Walk<false> iw = walk;  // the issue side: up to kStages pairs ahead of the consume side, over the same pairs
  uint64_t iu = 0;
  bool imore = iw.take(c, iu);
  uint32_t isrc = 0, in_flight = 0;
  if (c.lane == 0) fence_proxy_async_global();  // data may have been written through the generic proxy
#pragma unroll
  for (int s = 0; s < kStages; ++s) {
    if (!imore) break;
    if (c.lane == 0) issue_load(c, P.src[isrc], bytes, iu, s);
    ++in_flight;
    if (++isrc == n) {
      isrc = 0;
      imore = iw.take(c, iu);
    }
  }
  uint64_t acc[kArWords];
#pragma unroll
  for (int i = 0; i < kArWords; ++i) acc[i] = 0ull;
  int s = 0;
  uint32_t csrc = 0;
  uint64_t u = 0;
  bool more = walk.take(c, u);
  while (more) {
    if (!mbar_wait(c, s)) {
      for (; in_flight > 0; --in_flight) {
        mbar_drain(c, s);
        s = (s + 1 == kStages) ? 0 : s + 1;
      }
      return;
    }
    --in_flight;
    const uint32_t len = unit_len(bytes, u);
    const uint32_t sbase = c.stage_smem + s * kUnitBytes;
    if (len == kUnitBytes) {
#pragma unroll
      for (int i = 0; i < kArWords / 2; ++i) ar_add(acc, i, lds_v4(sbase + ar_vec_off<16>(c.lane, i)));
    } else {
#pragma unroll
      for (int i = 0; i < kArWords / 2; ++i)
        if (ar_vec_off<16>(c.lane, i) < len) ar_add(acc, i, lds_v4(sbase + ar_vec_off<16>(c.lane, i)));
    }
    __syncwarp();
    if (imore) {
      if (c.lane == 0) {
        fence_proxy_async_smem();
        issue_load(c, P.src[isrc], bytes, iu, s);
      }
      ++in_flight;
      if (++isrc == n) {
        isrc = 0;
        imore = iw.take(c, iu);
      }
    }
    s = (s + 1 == kStages) ? 0 : s + 1;
    if (++csrc == n) {
      Store::template put<16>(c, P, u, len, fw, acc, a);
      csrc = 0;
      more = walk.take(c, u);
    }
  }
}

// ld/st read side: for each unit, the n inputs one after another, kLdstVecs 16-byte loads in flight per lane each.
template <uint32_t kLaneBytes, typename Store, typename Params>
__device__ void ar_units_ldst(const Ctx& c, const Params& P, uint64_t bytes, Walk<false> walk, uint64_t fw, Sum& a) {
  uint64_t acc[kArWords];
#pragma unroll
  for (int i = 0; i < kArWords; ++i) acc[i] = 0ull;
  for (uint64_t u; walk.take(c, u);) {
    const uint32_t len = unit_len(bytes, u);
    for (uint32_t t = 0; t < P.n; ++t) {
      const uint8_t* base = P.src[t] + u * kUnitBytes;
      uint4 v[kLdstVecs];
      if (len == kUnitBytes) {
#pragma unroll
        for (int i = 0; i < (int)kLdstVecs; ++i)
          v[i] = ldg_stream_v4(reinterpret_cast<const uint4*>(base + ar_vec_off<kLaneBytes>(c.lane, i)));
      } else {
#pragma unroll
        for (int i = 0; i < (int)kLdstVecs; ++i) {
          v[i] = make_uint4(0u, 0u, 0u, 0u);
          const uint32_t off = ar_vec_off<kLaneBytes>(c.lane, i);
          if (off < len) v[i] = ldg_stream_v4(reinterpret_cast<const uint4*>(base + off));
        }
      }
#pragma unroll
      for (int i = 0; i < (int)kLdstVecs; ++i) ar_add(acc, i, v[i]);
    }
    Store::template put<kLaneBytes>(c, P, u, len, fw, acc, a);
  }
}

// The read side on the data path picked at run time (ProbeParams::path): 0 TMA bulk copies, 1 16-byte ld/st, 2 32-byte
// ld/st.
template <typename Store, typename Params>
__device__ __forceinline__ void ar_units(Ctx& c, const Params& P, uint64_t bytes, Walk<false> walk, uint64_t fw,
                                         Sum& a) {
  if (P.path == 2u) ar_units_ldst<32, Store>(c, P, bytes, walk, fw, a);
  else if (P.path == 1u) ar_units_ldst<16, Store>(c, P, bytes, walk, fw, a);
  else ar_units_tma<Store>(c, P, bytes, walk, fw, a);
}

// The end of a word check, by every lane with its own count of bad words and lowest bad word's byte offset: one atomic
// pair per warp with a bad word into the counters of size k.
__device__ __forceinline__ void ar_check_flush(const Ctx& c, ArScratch* as, uint32_t k, uint64_t bad, uint64_t first) {
  bad = warp_sum64(bad);
  first = warp_min64(first);
  if (c.lane == 0 && bad != 0) {
    atomicAdd(&as->bad_words[k], (unsigned long long)bad);
    atomicMax(&as->first_bad_n[k], (unsigned long long)~first);
  }
}

// The untimed word check and clear of the output the last rep of size k stored at P.out (allreduce_ll_kernel): each
// lane compares every 32nd word of its warp's share with allreduce_word, reading at L2 (other SMs stored them), and
// overwrites it with 0, so a word that the next size or call does not store reads as 0 rather than as this size's
// sum.  One atomic pair per warp with a bad word.
template <typename Params>
__device__ void ar_check(const Ctx& c, const Params& P, ArScratch* as, uint32_t k, uint64_t bytes, uint32_t gwarp,
                         uint32_t nwarps) {
  unsigned long long* out = reinterpret_cast<unsigned long long*>(P.out);
  const uint64_t words = bytes / 8;
  uint64_t bad = 0, first = ~0ull;
  for (uint64_t w = (uint64_t)gwarp * 32u + (uint32_t)c.lane; w < words; w += (uint64_t)nwarps * 32u) {
    if (__ldcg(out + w) != allreduce_word(P.seed, P.n, w)) {
      ++bad;
      first = min(first, w * 8u);
    }
    out[w] = 0ull;
  }
  __threadfence();  // the clearing stores are performed before the next size's opening barrier
  ar_check_flush(c, as, k, bad, first);
}

// The untimed check of rep r of size k of an output (allreduce_kernel's in the rank's scratch,
// allreduce_twoshot_kernel's gather area, allreduce_ring_kernel's ring area): every word of it is read at L2 (peers and
// other SMs stored it), compared with allreduce_word, folded into the rep's (S, X) by its place in the output, and then
// overwritten with 0, so a unit that is not delivered in a later rep reads as 0s rather than as this rep's sums.  One
// atomic pair per warp with a bad word, over every rep of the size.
template <typename Params>
__device__ void ar_check_clear(const Ctx& c, const Params& P, uint4* const out, ArScratch* as, uint64_t* red,
                               uint32_t k, uint32_t r, uint64_t bytes, uint32_t gwarp, uint32_t nwarps) {
  Sum a{0ull, 0ull, 0ull};
  uint64_t bad = 0, first = ~0ull;
  Walk<false> walk = strided(bytes, gwarp, nwarps);
  for (uint64_t u; walk.take(c, u);) {
    uint4* const p = out + u * (kUnitBytes / 16);
    const uint32_t nvec = unit_len(bytes, u) / 16;
    const uint64_t w_base = u * (kUnitBytes / 8);
    uint64_t ux = 0;
#pragma unroll 4
    for (uint32_t v = c.lane; v < nvec; v += 32) {
      const uint4 q = __ldcg(p + v);
      const uint64_t w0 = pack64(q.x, q.y), w1 = pack64(q.z, q.w), k0 = w_base + 2 * v;
      if (w0 != allreduce_word(P.seed, P.n, k0)) {
        ++bad;
        first = min(first, 8 * k0);
      }
      if (w1 != allreduce_word(P.seed, P.n, k0 + 1)) {
        ++bad;
        first = min(first, 8 * k0 + 8);
      }
      add_pair(a, ux, w0, w1);
      stg_v4(p + v, make_uint4(0u, 0u, 0u, 0u));
    }
    fold_unit(a, ux, u);
  }
  __threadfence();  // the clearing stores are performed before the next opening barrier signals the peers
  ar_check_flush(c, as, k, bad, first);
  Acc* const acc = &as->rep.rep[k][r];
  cta_reduce<1>(c, red, &a, &acc);
}
}  // namespace
}  // namespace cdp
