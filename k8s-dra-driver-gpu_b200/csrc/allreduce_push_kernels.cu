// allreduce_push_kernels.cu — sm_90a kernel of cdprobe_allreduce_push's push all-reduce, in which every byte moves as a
// write: every rank reduces each 8 KiB unit of its input straight into the push area of the unit's owner (the two-shot's
// chunks), with cp.reduce.async.bulk .add.u64 on the TMA path or red.relaxed.sys.global.add.u64 per word on the ld/st
// paths; after a fenced domain barrier each owner pushes its finished chunk to every peer with st.global.v4 (the
// one-shot's read side, allreduce_path.cuh, through ToPeers); a fenced domain barrier closes the rep, and every rank
// checks and clears its own area (allreduce_push_kernel, with allreduce_path.cuh's ar_check_clear).
//
// probe_kernels.cu is untouched: the probe kernel's code generation does not depend on this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "allreduce_path.cuh"
#include "allreduce_push.h"

namespace cdp {
namespace {
// 1-D TMA bulk reduction: the `bytes` at src_smem are added, as 64-bit words mod 2^64, into global memory at dst (local
// HBM or a peer's, through its mapping) by the memory system that owns dst.  Completion by bulk_group, as bulk_store.
// dst, src_smem and bytes are multiples of 16: the ladder's sizes are multiples of 128 (bytes_per_pair is a whole
// number of 128-byte slices), so every unit_len is too.
__device__ __forceinline__ void bulk_reduce_add_u64(void* dst, uint32_t src_smem, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.u64 [%0], [%1], %2;" ::"l"(dst), "r"(src_smem),
               "r"(bytes)
               : "memory");
}
// One 64-bit word added at p by the memory system that owns p, atomic at system scope.
__device__ __forceinline__ void red_add_sys(uint64_t* p, uint64_t v) {
  asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t lds_u64(uint32_t addr) {
  uint64_t v;
  asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void sts_u64(uint32_t addr, uint64_t v) {
  asm volatile("st.shared.u64 [%0], %1;" ::"r"(addr), "l"(v) : "memory");
}

// Where unit u of a size of `units` units goes in the reduce-scatter: its owner's push area, through this rank's
// mapping.
__device__ __forceinline__ uint8_t* owner_unit(const PushParams& P, uint64_t units, uint64_t u) {
  const uint32_t o = twoshot_owner(units, P.n, u);
  return P.dst[(o + P.n - P.rank) % P.n] + u * kUnitBytes;
}

// The reduce-scatter on the TMA path, by one warp over the units of `walk`: lane 0 bulk-loads each source unit into
// the next stage of the warp's kStages ring and reduces it from there into its owner's area, one bulk group per unit;
// a stage is refilled once the reduction issued kStages units earlier has read it.  The armed fault acts on unit fu
// (~0: none): mode 0 adds 1 to word fb of the stage (a generic store, made visible to the async proxy), mode 1 skips
// the reduction, mode 2 issues it twice.  Ends with every reduction of the warp performed (wait_group 0) and a
// fence.proxy.async.global.  Returns false once the launch is aborted.
__device__ bool reduce_tma(Ctx& c, const PushParams& P, uint64_t bytes, Walk<false> walk, uint64_t fu, uint32_t fb,
                           uint32_t mode) {
  const uint64_t units = units_of(bytes);
  bool ok = true;
  int s = 0;
  if (c.lane == 0) fence_proxy_async_global();  // the last check's clearing stores were generic
  uint32_t it = 0;
  for (uint64_t u; walk.take(c, u); ++it) {
    const uint32_t len = unit_len(bytes, u);
    const uint32_t sbase = c.stage_smem + s * kUnitBytes;
    if (c.lane == 0) {
      if (it >= (uint32_t)kStages) bulk_wait_read<kStages - 1>();  // the reduction that used stage s has read it
      issue_load(c, P.src, bytes, u, s);
    }
    if (!mbar_wait(c, s)) {
      mbar_drain(c, s);
      ok = false;
      break;
    }
    if (c.lane == 0) {
      uint8_t* const dst = owner_unit(P, units, u);
      const bool hit = u == fu;
      if (hit && mode == 0u) {
        sts_u64(sbase + fb, lds_u64(sbase + fb) + 1ull);
        fence_proxy_async_smem();
      }
      if (!(hit && mode == 1u)) bulk_reduce_add_u64(dst, sbase, len);
      if (hit && mode == 2u) bulk_reduce_add_u64(dst, sbase, len);
      bulk_commit();
    }
    s = (s + 1 == kStages) ? 0 : s + 1;
  }
  if (c.lane == 0) {
    bulk_wait_all();             // the reductions are performed, not only read out of shared memory
    fence_proxy_async_global();  // and ordered before this thread's later generic-proxy operations
  }
  __syncwarp();
  return ok;
}

// The reduce-scatter on the ld/st paths, by one warp: each lane loads its 16-byte vectors of a unit in the layout
// job_read_ldst uses and adds every 8-byte word into the owner's area with its own red.relaxed.sys.global.add.u64
// (there is no vector red for u64, so the two paths differ only in that layout).  The fault as in reduce_tma; fb is
// the armed word's byte offset in its unit.
template <uint32_t kLaneBytes>
__device__ void reduce_ldst(const Ctx& c, const PushParams& P, uint64_t bytes, Walk<false> walk, uint64_t fu,
                            uint32_t fb, uint32_t mode) {
  const uint64_t units = units_of(bytes);
  for (uint64_t u; walk.take(c, u);) {
    const uint32_t len = unit_len(bytes, u);
    const bool hit = u == fu;
    if (hit && mode == 1u) continue;
    const uint8_t* const base = P.src + u * kUnitBytes;
    uint8_t* const dst = owner_unit(P, units, u);
    uint4 v[kLdstVecs];
#pragma unroll
    for (int i = 0; i < (int)kLdstVecs; ++i) {
      v[i] = make_uint4(0u, 0u, 0u, 0u);
      const uint32_t off = ar_vec_off<kLaneBytes>(c.lane, i);
      if (off < len) v[i] = ldg_stream_v4(reinterpret_cast<const uint4*>(base + off));
    }
    for (uint32_t twice = hit && mode == 2u ? 2u : 1u; twice > 0; --twice) {
#pragma unroll
      for (int i = 0; i < (int)kLdstVecs; ++i) {
        const uint32_t off = ar_vec_off<kLaneBytes>(c.lane, i);
        if (off >= len) continue;
        uint64_t w0 = pack64(v[i].x, v[i].y), w1 = pack64(v[i].z, v[i].w);
        if (hit && mode == 0u && off == (fb & ~15u)) {
          if (fb & 8u) w1 += 1ull;
          else w0 += 1ull;
        }
        red_add_sys(reinterpret_cast<uint64_t*>(dst + off), w0);
        red_add_sys(reinterpret_cast<uint64_t*>(dst + off + 8), w1);
      }
    }
  }
}

// The all-gather's view of the parameters for ar_units: one input, this rank's own push area, whose chunk of finished
// units it reads back, and the peers' areas it pushes them to (ToPeers).
struct PeerView {
  const uint8_t* src[1];  // this rank's own push area
  uint32_t n;             // inputs: 1
  uint32_t path;          // the read side, ProbeParams::path
  const PushParams* P;    // the peers' areas: P->dst[1 .. P->n - 1]
};

// The all-gather's store policy (allreduce_path.cuh): a finished unit goes to every peer's push area, r + 1, r + 2, ...
// (mod n); this rank's own copy is already in place.  The armed mode-3 fault (fw, an output word index; ~0 when none)
// leaves the word xored with 1 on its way to dst[fault_dst] only.  Nothing is folded into (S, X); the word check reads
// the output back.
struct ToPeers {
  template <uint32_t kLaneBytes>
  __device__ __forceinline__ static void put(const Ctx& c, const PeerView& V, uint64_t u, uint32_t len, uint64_t fw,
                                             uint64_t (&acc)[kArWords], Sum&) {
    put_ranks<kLaneBytes, false>(c, *V.P, 1u, u, len, fw, acc);
  }
};
}  // namespace

// One rank of cdprobe_allreduce_push: for every size of the ladder, one warm-up and P.reps timed reps.  A rep opens with
// a domain barrier whose leader fences first (the previous check's clearing stores precede every peer's reductions),
// and whose release is stamped into t_rel[k][r].  Every warp then reduces its strided units of this rank's input into
// their owners' areas (reduce_tma, reduce_ldst).  Once every reduction of the CTA is performed, a CTA barrier, one
// fence.sys per CTA and a fenced domain barrier leave this rank's own chunk complete in its area; the rank reads that
// chunk back and pushes it to every peer (ar_units with ToPeers).  A CTA barrier, one fence.sys per CTA and a fenced
// domain barrier close the rep: its release, stamped into rep[k][r].t_end, is when this rank's output is complete.
// The word check and clear follow, untimed (DESIGN §5l).  State lives in the rank's scratch buffer; outside it, only
// the push areas and the barrier lines are written.
__global__ void __launch_bounds__(kThreads, 1) allreduce_push_kernel(const __grid_constant__ PushParams P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  ArScratch* as = P.scratch;
  BwScratch* bs = &as->rep;
  uint64_t* red;
  Ctx c = enter(smem, &bs->abort_flag, P.timeout_ns, &red);

  const uint32_t gwarp = blockIdx.x * kWarpsPerCta + c.warp;
  const uint32_t nwarps = gridDim.x * kWarpsPerCta;
  const PeerView V{{P.dst[0]}, 1u, P.path, &P};
  uint32_t b = 0;
  for (uint32_t k = 0; k < P.n_sizes; ++k) {
    const uint64_t bytes = P.size[k];
    uint64_t lo, hi;
    twoshot_chunk(units_of(bytes), P.n, P.rank, &lo, &hi);
    for (uint32_t r = 0; r <= P.reps; ++r) {
      if (!grid_barrier(c, bs, b++, &bs->t_rel[k][r], &P.dom, true)) return;
      const bool armed = r == 1u && k == P.fault_k;
      const uint64_t fu = armed && P.fault_mode < 3u ? P.fault_word / (kUnitBytes / 8) : ~0ull;
      const uint32_t fb = (uint32_t)(P.fault_word % (kUnitBytes / 8)) * 8u;
      const Walk<false> walk = strided(bytes, gwarp, nwarps);
      if (P.path == 2u) reduce_ldst<32>(c, P, bytes, walk, fu, fb, P.fault_mode);
      else if (P.path == 1u) reduce_ldst<16>(c, P, bytes, walk, fu, fb, P.fault_mode);
      else reduce_tma(c, P, bytes, walk, fu, fb, P.fault_mode);  // aborted: the barrier below sees it
      if (!close_fenced(c, bs, b++, nullptr, &P.dom)) return;  // this rank's chunk is complete in its area
      if (P.n > 1) {
        Sum a{0ull, 0ull, 0ull};
        ar_units<ToPeers>(c, V, bytes, Walk<false>{hi, lo + gwarp, 0ull, nwarps, nullptr},
                          armed && P.fault_mode == 3u ? P.fault_word : ~0ull, a);
      }
      if (!close_fenced(c, bs, b++, &bs->rep[k][r].t_end, &P.dom)) return;
      ar_check_clear(c, P, reinterpret_cast<uint4*>(P.dst[0]), as, red, k, r, bytes, gwarp, nwarps);
    }
  }
}

int allreduce_push_launch(const PushParams& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  return grid_launch(allreduce_push_kernel, p, grid, cooperative, stream);
}

}  // namespace cdp
