// probe_kernels.cu — sm_90a kernels of the ComputeDomain fabric probe.
//
// K1 read probe   : every warp streams 8 KiB units of a peer's source slice
//                   into shared memory with 1-D TMA bulk copies
//                   (cp.async.bulk.shared::cluster.global + mbarrier complete_tx,
//                   3 stages in flight per warp) or with ld.global.v4 loads
//                   (16 or 32 contiguous bytes per lane), and folds them into
//                   the (S, X) checksum.
// K2 write probe  : every warp generates the write pattern into shared memory
//                   and pushes it into the peer's landing slot with TMA bulk
//                   stores (cp.async.bulk.global.shared::cta) or st.global.v4.
// K3 barrier      : grid barrier (atomic arrive / release word) whose last
//                   arriver runs the cross-GPU flag exchange with the ranks the
//                   phase table names (at most four between rounds, nobody between
//                   the write and the read of a round, everybody at open/close):
//                   publish, one fence.sys only if something was published,
//                   pipelined st.relaxed.sys epochs into those peers' Ctrl,
//                   ld.acquire.sys on the local copy.
// K4 verify/local : the read probe pointed at local HBM (landing slots, source
//                   slices at open, the N = 1 loop-back).
// K5 bwcurve      : cdprobe_bwcurve's reads of growing prefixes of one source
//                   slice through the K1 read path, one launch per cell, each
//                   rep between two grid barriers (bwcurve_kernel).
// K6 allreduce    : cdprobe_allreduce's one-shot all-reduce: every warp
//                   streams one output unit of all n ranks' source buffers
//                   (TMA ring or ld.global.v4), adds them in registers and
//                   stores the sum with st.global.v4; each rep opens with a
//                   domain barrier (allreduce_kernel).
// K7 alltoall     : cdprobe_alltoall's one-shot all-to-all: every warp
//                   pushes interleaved units of the rank's blocks into the
//                   receivers' exchange areas through the K2 write path;
//                   each rep sits between two domain barriers and is
//                   followed by the word check of the blocks received
//                   (alltoall_kernel).
//
// One persistent cooperative kernel per GPU runs every phase of a probe
// (wake-up, tournament rounds x {write, read + overlapped verify}) so a run
// costs one launch per GPU; phases are timed with %globaltimer on the issuing
// GPU (SURVEY.md H7).  The phase table comes from schedule.cc.  The single-GPU loop-back table runs as one
// streamed pass without barriers instead (loopback_pass).
//
// The reference has no kernel for this path (SURVEY.md F1/F3); the gate it
// implements is cmd/compute-domain-daemon/main.go:435-459.
#include <cuda_runtime.h>
#include <stdint.h>

#include "allreduce.h"
#include "alltoall.h"
#include "bwcurve.h"
#include "probe_launch.h"
#include "probe_types.h"

namespace cdp {
namespace {

// ------------------------------------------------------------------ PTX ----
__device__ __forceinline__ uint64_t gtimer() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void st_release_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_release_gpu(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
enum Scope { kScopeGpu, kScopeSys };
// Acquire load of a 64-bit word at gpu scope (a word only this GPU's CTAs write) or sys scope (peers write it).
template <Scope S>
__device__ __forceinline__ uint64_t ld_acquire(const void* p) {
  uint64_t v;
  if constexpr (S == kScopeSys) asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  else asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t ld_relaxed_sys(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// 1-D TMA bulk load: global (local HBM or NVLink peer) -> this CTA's shared memory.
__device__ __forceinline__ void bulk_load(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}
// 1-D TMA bulk store: shared memory -> global (local HBM or NVLink peer).
__device__ __forceinline__ void bulk_store(void* dst, uint32_t src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src_smem), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// 128-bit streaming load (coherent at L2; L1 is not polluted). Not .nc: the
// verify job reads data a peer wrote earlier in the same kernel.
__device__ __forceinline__ uint4 ldg_stream_v4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
__device__ __forceinline__ void stg_v4(uint4* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
__device__ __forceinline__ uint4 lds_v4(uint32_t addr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
  return r;
}
__device__ __forceinline__ void sts_v4(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ uint64_t pack64(uint32_t lo, uint32_t hi) { return (uint64_t)lo | ((uint64_t)hi << 32); }

// ------------------------------------------------------------- context -----
struct Ctx {
  unsigned int* abort_word;  // the launch's abort flag: Ctrl::abort_flag, or BwScratch::abort_flag (bwcurve_kernel)
  uint64_t deadline;
  uint32_t stage_smem;   // shared address of this warp's stage 0
  uint32_t bar_smem;     // shared address of this warp's mbarrier 0
  uint32_t parity_bits;  // bit s: parity to wait for on stage s
  int warp, lane;
};

__device__ __forceinline__ bool aborted(const Ctx& c) {
  return *reinterpret_cast<volatile unsigned int*>(c.abort_word) != 0u;
}
// Slow-path check used inside spin loops: watchdog + abort propagation.
__device__ __noinline__ bool check_abort(const Ctx& c) {
  if (aborted(c)) return true;
  if (gtimer() > c.deadline) {
    atomicExch(c.abort_word, 1u);
    return true;
  }
  return false;
}
// Spins until the 64-bit word at p reaches target (acquire loads at scope S), checking abort and the deadline
// every 64 spins.  Returns whether the target was reached; false means the run is aborted.
template <Scope S>
__device__ __forceinline__ bool spin_until(const Ctx& c, const void* p, uint64_t target) {
  uint32_t spins = 0;
  while (ld_acquire<S>(p) < target) {
    if ((++spins & 63u) == 0u && check_abort(c)) return false;
  }
  return true;
}

// Waits for the bulk load armed on `stage`.  Returns false when the run was aborted while waiting —
// the load is then STILL IN FLIGHT towards this CTA's shared memory and the caller must drain it
// (mbar_drain) before the CTA may exit or reuse the stage.
__device__ __forceinline__ bool mbar_wait(Ctx& c, int stage) {
  const uint32_t bar = c.bar_smem + 8u * stage;
  const uint32_t parity = (c.parity_bits >> stage) & 1u;
  uint32_t spins = 0;
  bool ok = true;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 255u) == 0u && check_abort(c)) {
      ok = false;
      break;
    }
  }
  // warp-uniform outcome: a lane that saw the phase complete while another saw the abort must not
  // flip its parity alone (mbar_drain re-waits the same phase; a completed one passes at once)
  if (!__all_sync(0xffffffffu, ok)) return false;
  c.parity_bits ^= (1u << stage);
  return true;
}
// After an abort: wait, without the watchdog, for a load that was already issued.  An abort means a PEER
// missed a barrier; the memory this load targets is mapped and the copy completes in microseconds.  If
// it has not after kDrainNs the fabric itself is gone: trap (sticky error on the context, reported by
// the host as a kernel failure) rather than let a bulk copy land in the shared memory of an exited CTA.
constexpr uint64_t kDrainNs = 200ull * 1000 * 1000;
__device__ __noinline__ void mbar_drain(Ctx& c, int stage) {
  const uint32_t bar = c.bar_smem + 8u * stage;
  const uint32_t parity = (c.parity_bits >> stage) & 1u;
  const uint64_t t_give_up = gtimer() + kDrainNs;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 1023u) == 0u && gtimer() > t_give_up) __trap();
  }
  c.parity_bits ^= (1u << stage);
}

// ---------------------------------------------------------- unit walks -----
// The 8 KiB units one warp works on.  Strided (the phase walk): units gwarp, gwarp + nwarps, ...  Claimed (the
// loop-back pass): runs of kClaimUnits consecutive units taken from a counter shared by every warp of the grid,
// so no warp idles while another still has a backlog.  take() is warp-uniform; once it returns false it keeps
// doing so.  A claimed walk also stops when the run is aborted.
// 2 units (16 KiB) per atomic.  The size sets how far the last write lands after the first warps have moved on
// to reading, and HBM streams slower while reads and writes mix.  On an H100 at a 400 W limit (1 GiB, median of 300
// probes, two runs each) the kernel took 1017.6-1017.9 us with 2, 1023-1024 us with 4, 1033 us with 8 and
// 1038 us with 16; with 1 it varied from 1031 to 1054 us.
constexpr uint32_t kClaimUnits = 2;

template <bool kClaimed>
struct Walk {
  uint64_t n_units, next, end;
  uint32_t stride;
  unsigned long long* claim;

  __device__ __forceinline__ bool take(const Ctx& c, uint64_t& u) {
    if (kClaimed && next == end && next < n_units) {
      unsigned long long b = 0;
      if (c.lane == 0) {
        const bool ab = aborted(c);
        b = atomicAdd(claim, (unsigned long long)kClaimUnits);
        if (ab) b = n_units;
      }
      b = __shfl_sync(0xffffffffu, b, 0);
      next = b < n_units ? b : n_units;
      end = next + kClaimUnits < n_units ? next + kClaimUnits : n_units;
    }
    if (next >= n_units) return false;
    u = next;
    next += kClaimed ? 1u : stride;
    return true;
  }
  static constexpr bool kSpread = false;  // every unit is in one region (BlockWalk spreads units over several)
};
__device__ __forceinline__ uint64_t units_of(uint64_t bytes) { return (bytes + kUnitBytes - 1) / kUnitBytes; }
// Bytes in unit u: kUnitBytes, or what is left of the buffer for its last unit.
__device__ __forceinline__ uint32_t unit_len(uint64_t bytes, uint64_t u) {
  const uint64_t left = bytes - u * kUnitBytes;
  return left < kUnitBytes ? static_cast<uint32_t>(left) : kUnitBytes;
}
__device__ __forceinline__ Walk<false> strided(uint64_t bytes, uint32_t gwarp, uint32_t nwarps) {
  return Walk<false>{units_of(bytes), gwarp, 0ull, nwarps, nullptr};
}
__device__ __forceinline__ Walk<true> claimed(uint64_t bytes, unsigned long long* counter) {
  return Walk<true>{units_of(bytes), 0ull, 0ull, 1u, counter};
}

// ------------------------------------------------------------ checksum -----
struct Sum {
  uint64_t s0, s1;  // two partial sums (ILP), folded at the end
  uint64_t x;       // position-folded xor
};

// Adds two consecutive 64-bit words into the sums and into the xor of the unit they belong to.
__device__ __forceinline__ void add_pair(Sum& a, uint64_t& ux, uint64_t w0, uint64_t w1) {
  a.s0 += w0;
  a.s1 += w1;
  ux ^= w0 ^ w1;
}

// The write pattern one lane generates: word k of a slot is write_word(salt, k) = z ^ (z >> 32) with
// z = (salt + k) * kGolden.  A lane stores kLaneBytes of consecutive words per access, and the 32 lanes of a warp
// store consecutive runs, so after each access a lane moves on by 32 * kLaneBytes / 8 words.
template <uint32_t kLaneBytes>
struct Pattern {
  static constexpr int kV = kLaneBytes / 16;  // 16-byte vectors per access
  uint64_t z;                                 // (salt + k) * kGolden of the lane's next word k
  __device__ __forceinline__ Pattern(uint64_t salt, uint64_t u, int lane)
      : z((salt + u * (kUnitBytes / 8) + 2ull * kV * lane) * kGolden) {}
  // The lane's next access, added into the checksum.
  __device__ __forceinline__ void next(uint4 (&v)[kV], Sum& a, uint64_t& ux) {
#pragma unroll
    for (int h = 0; h < kV; ++h) {
      const uint64_t z0 = z + 2ull * h * kGolden, z1 = z0 + kGolden;
      const uint64_t w0 = z0 ^ (z0 >> 32), w1 = z1 ^ (z1 >> 32);
      add_pair(a, ux, w0, w1);
      v[h] = make_uint4((uint32_t)w0, (uint32_t)(w0 >> 32), (uint32_t)w1, (uint32_t)(w1 >> 32));
    }
    z += 64ull * kV * kGolden;
  }
};

__device__ __forceinline__ void fold_unit(Sum& a, uint64_t unit_xor, uint64_t unit) {
  const uint32_t g = static_cast<uint32_t>(unit / (kGranuleBytes / kUnitBytes));
  a.x ^= rotl64(unit_xor, fold6(g));
}

// ------------------------------------------------------- K1/K4: reading ----
__device__ __forceinline__ void issue_load(const Ctx& c, const uint8_t* base, uint64_t bytes, uint64_t u, int stage) {
  const uint32_t n = unit_len(bytes, u);
  const uint32_t bar = c.bar_smem + 8u * stage;
  mbar_arrive_expect_tx(bar, n);
  bulk_load(c.stage_smem + stage * kUnitBytes, base + u * kUnitBytes, n, bar);
}

// Every read job returns the number of units it folded in.
template <bool kClaimed>
__device__ uint32_t job_read_tma(Ctx& c, const uint8_t* base, uint64_t bytes, Walk<kClaimed> walk, Sum& a) {
  uint64_t q[kStages];     // units in flight, oldest first; the oldest sits on stage s (constant indices only)
  uint32_t in_flight = 0;  // loads issued and not yet waited for (warp-uniform)
  uint32_t it = 0;
  if (c.lane == 0) fence_proxy_async_global();  // data may have been written through the generic proxy
#pragma unroll
  for (int s = 0; s < kStages; ++s) {
    uint64_t u;
    if (walk.take(c, u)) {
      if (c.lane == 0) issue_load(c, base, bytes, u, s);
      q[s] = u;
      ++in_flight;
    }
  }
  int s = 0;
  while (in_flight > 0) {
    const uint64_t u = q[0];
    if (!mbar_wait(c, s)) {
      // aborted: stop issuing, but every load already in flight must land before this CTA can exit
      for (; in_flight > 0; --in_flight) {
        mbar_drain(c, s);
        s = (s + 1 == kStages) ? 0 : s + 1;
      }
      return it;
    }
    --in_flight;
    ++it;
#pragma unroll
    for (int k = 0; k + 1 < kStages; ++k) q[k] = q[k + 1];
    const uint32_t nvec = unit_len(bytes, u) >> 4;
    const uint32_t sbase = c.stage_smem + s * kUnitBytes + c.lane * 16u;
    uint64_t ux = 0;
    if (nvec == kUnitBytes / 16) {
#pragma unroll
      for (int k = 0; k < (int)(kUnitBytes / 16 / 32); ++k) {
        const uint4 v = lds_v4(sbase + k * 512u);
        add_pair(a, ux, pack64(v.x, v.y), pack64(v.z, v.w));
      }
    } else {
      for (uint32_t i = c.lane; i < nvec; i += 32) {
        const uint4 v = lds_v4(c.stage_smem + s * kUnitBytes + i * 16u);
        add_pair(a, ux, pack64(v.x, v.y), pack64(v.z, v.w));
      }
    }
    fold_unit(a, ux, u);
    __syncwarp();
    uint64_t un;
    if (walk.take(c, un)) {
      if (c.lane == 0) {
        fence_proxy_async_smem();
        issue_load(c, base, bytes, un, s);
      }
#pragma unroll
      for (int k = 0; k < kStages; ++k)
        if (k == (int)in_flight) q[k] = un;
      ++in_flight;
    }
    s = (s + 1 == kStages) ? 0 : s + 1;
  }
  return it;
}

// The ld/st data paths: a lane moves kLaneBytes contiguous bytes per access, lane l at kLaneBytes * l +
// 32 * kLaneBytes * k of the unit.  sm_90 has no 256-bit global access, so 32 bytes move as two 16-byte accesses
// issued back to back.  A full unit is kLdstVecs 16-byte loads in flight per lane on either path.
template <uint32_t kLaneBytes, bool kClaimed>
__device__ uint32_t job_read_ldst(Ctx& c, const uint8_t* base, uint64_t bytes, Walk<kClaimed> walk, Sum& a) {
  constexpr int kV = kLaneBytes / 16;  // 16-byte vectors per access; vector i is the (i % kV)-th of access i / kV
  static_assert(kLdstVecs * 16 * 32 == kUnitBytes, "a warp's loads cover one unit");
  uint32_t it = 0;
  for (uint64_t u; walk.take(c, u); ++it) {
    const uint32_t n = unit_len(bytes, u) / kLaneBytes;  // lane accesses in this unit
    const uint4* gp = reinterpret_cast<const uint4*>(base + u * kUnitBytes) + kV * c.lane;
    uint4 v[kLdstVecs];
    if (n == kUnitBytes / kLaneBytes) {
#pragma unroll
      for (int i = 0; i < (int)kLdstVecs; ++i) v[i] = ldg_stream_v4(gp + 32 * kV * (i / kV) + i % kV);
    } else {
#pragma unroll
      for (int i = 0; i < (int)kLdstVecs; ++i) {
        v[i] = make_uint4(0u, 0u, 0u, 0u);
        if (c.lane + (i / kV) * 32u < n) v[i] = ldg_stream_v4(gp + 32 * kV * (i / kV) + i % kV);
      }
    }
    uint64_t ux = 0;
#pragma unroll
    for (int i = 0; i < (int)kLdstVecs; ++i) add_pair(a, ux, pack64(v[i].x, v[i].y), pack64(v[i].z, v[i].w));
    fold_unit(a, ux, u);
  }
  return it;
}

// ---------------------------------------------------------- K2: writing ----
// Every write job returns the number of units it stored.  The walk W names each unit; a walk that spreads its units
// over several regions (kSpread) also names, through place(), the unit's index, region (base) and pattern salt in
// it.  Every region is `bytes` long.
template <typename W>
__device__ uint32_t job_write_tma(Ctx& c, uint8_t* base, uint64_t bytes, W walk, uint64_t salt, Sum& a) {
  uint32_t it = 0;
  int s = 0;
  for (uint64_t u; walk.take(c, u); ++it) {
    if constexpr (W::kSpread) walk.place(u, base, salt);
    if (it >= (uint32_t)kStages) {
      if (c.lane == 0) bulk_wait_read<kStages - 1>();  // the store that used stage s has drained it
    }
    __syncwarp();
    const uint32_t nb = unit_len(bytes, u);
    const uint32_t sbase = c.stage_smem + s * kUnitBytes;
    Pattern<16> pat(salt, u, c.lane);
    uint64_t ux = 0;
    for (uint32_t i = c.lane; i < nb >> 4; i += 32) {
      uint4 v[1];
      pat.next(v, a, ux);
      sts_v4(sbase + i * 16u, v[0]);
    }
    fold_unit(a, ux, u);
    fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the async proxy
    __syncwarp();
    if (c.lane == 0) {
      bulk_store(base + u * kUnitBytes, sbase, nb);
      bulk_commit();
    }
    s = (s + 1 == kStages) ? 0 : s + 1;
  }
  if (c.lane == 0) bulk_wait_all();  // stores complete (not just smem drained)
  __syncwarp();
  return it;
}

// Stores the write pattern to the addresses job_read_ldst loads from.
template <uint32_t kLaneBytes, typename W>
__device__ uint32_t job_write_ldst(Ctx& c, uint8_t* base, uint64_t bytes, W walk, uint64_t salt, Sum& a) {
  constexpr int kV = Pattern<kLaneBytes>::kV;
  uint32_t it = 0;
  for (uint64_t u; walk.take(c, u); ++it) {
    if constexpr (W::kSpread) walk.place(u, base, salt);
    const uint32_t n = unit_len(bytes, u) / kLaneBytes;
    uint4* gp = reinterpret_cast<uint4*>(base + u * kUnitBytes);
    Pattern<kLaneBytes> pat(salt, u, c.lane);
    uint64_t ux = 0;
#pragma unroll 4
    for (uint32_t i = c.lane; i < n; i += 32) {
      uint4 v[kV];
      pat.next(v, a, ux);
#pragma unroll
      for (int h = 0; h < kV; ++h) stg_v4(gp + kV * i + h, v[h]);
    }
    fold_unit(a, ux, u);
  }
  return it;
}

// The data path picked at run time (ProbeParams::path): 0 TMA bulk copies, 1 16-byte ld/st, 2 32-byte ld/st.
template <bool kClaimed>
__device__ __forceinline__ uint32_t read_units(Ctx& c, uint32_t path, const uint8_t* base, uint64_t bytes,
                                               Walk<kClaimed> walk, Sum& a) {
  if (path == 2u) return job_read_ldst<32>(c, base, bytes, walk, a);
  if (path == 1u) return job_read_ldst<16>(c, base, bytes, walk, a);
  return job_read_tma(c, base, bytes, walk, a);
}
template <typename W>
__device__ __forceinline__ uint32_t write_units(Ctx& c, uint32_t path, uint8_t* base, uint64_t bytes, W walk,
                                                uint64_t salt, Sum& a) {
  if (path == 2u) return job_write_ldst<32>(c, base, bytes, walk, salt, a);
  if (path == 1u) return job_write_ldst<16>(c, base, bytes, walk, salt, a);
  return job_write_tma(c, base, bytes, walk, salt, a);
}

// ---------------------------------------------------------- K3: barrier ----
// Leader-only publications once every local CTA has finished a phase.
//  * a write job: (S, X, run_seq) of what was stored, into the owner's Ctrl, so that the owner can verify the
//    landing slot — must be visible before the flag that tells the owner "phase done";
//  * verify jobs: the verdict goes back to the writer.  Writers read it only when they assemble their result row,
//    after the last barrier of the run, so ALL verdicts are published by the last barrier's leader in one go (one
//    thread, one fence: no cross-thread ordering argument needed).
__device__ bool publish_writes(const ProbeParams& P, Ctrl* ctrl, int ph) {
  bool any = false;
#pragma unroll
  for (int jb = 0; jb < 2; ++jb) {
    const Job job = P.phase[ph].job[jb];
    if (job.kind != kJobWrite) continue;
    const volatile Acc* acc = &ctrl->acc[ph][jb];
    Ctrl* pc = reinterpret_cast<Ctrl*>(P.base_peer[job.peer]);
    st_relaxed_sys(&pc->wr[job.slot].sum, acc->sum);
    st_relaxed_sys(&pc->wr[job.slot].xr, acc->xr);
    st_relaxed_sys(&pc->wr[job.slot].seq, P.run_seq);
    any = true;
  }
  return any;
}
__device__ void publish_verdicts(const ProbeParams& P, Ctrl* ctrl) {
  for (uint32_t ph = 0; ph < P.n_phases; ++ph) {
#pragma unroll
    for (int jb = 0; jb < 2; ++jb) {
      const Job job = P.phase[ph].job[jb];
      if (job.kind != kJobVerify) continue;
      const volatile Acc* acc = &ctrl->acc[ph][jb];
      const uint64_t wsum = ld_relaxed_sys(&ctrl->wr[job.slot].sum);
      const uint64_t wxr = ld_relaxed_sys(&ctrl->wr[job.slot].xr);
      const uint64_t wseq = ld_relaxed_sys(&ctrl->wr[job.slot].seq);
      uint64_t code = kVerdictNotWritten;
      if (wseq == P.run_seq) code = (wsum == acc->sum && wxr == acc->xr) ? kVerdictOk : kVerdictMismatch;
      uint8_t* wb = P.base_peer[job.writer];
      if (wb != nullptr) st_relaxed_sys(&reinterpret_cast<Ctrl*>(wb)->verdict[P.rank], P.run_seq * 4ull + code);
    }
  }
}

// ------------------------------------------------------ test-only fault injection ----
// cdprobe_corrupt_landing arms ctrl->fault in the issuer's Ctrl.  The fault is applied by one thread after the write
// into the armed target's slot has completed and before anything that lets a verifier read the slot, so to the
// verifier it is a fault in transit; the writer's published (S, X) is untouched.  Every store stays inside the slot
// (the host checks word[e] < bytes_per_pair / 8).
__device__ __forceinline__ bool fault_armed(const ProbeParams& P, const Ctrl* ctrl, uint32_t target) {
  return ctrl->fault.n != 0u && ctrl->fault.target == target && P.base_peer[target] != nullptr;
}
__device__ __forceinline__ void xor_landing(const LandingFault* f, uint8_t* slot) {
  fence_proxy_async_global();  // the slot may hold TMA bulk stores
  const uint32_t n = f->n;
  for (uint32_t e = 0; e < n && e < kMaxLandingFaults; ++e) {
    uint64_t* w = reinterpret_cast<uint64_t*>(slot) + f->word[e];
    st_relaxed_sys(w, ld_relaxed_sys(w) ^ f->mask[e]);
  }
}
// Phase walk: phase ph has a write job into the armed target (either job slot, as in publish_writes).  Called by the
// barrier leader before its publications, signals and release, which the target's verify waits for.
__device__ __noinline__ void fault_phase_write(const ProbeParams& P, Ctrl* ctrl, int ph) {
#pragma unroll
  for (int jb = 0; jb < 2; ++jb) {
    const Job job = P.phase[ph].job[jb];
    if (job.kind != kJobWrite || !fault_armed(P, ctrl, (uint32_t)job.peer)) continue;
    xor_landing(&ctrl->fault, P.base_peer[job.peer] + P.land_off + (uint64_t)job.slot * P.bpp);
    __threadfence_system();
  }
}

__device__ __forceinline__ void signal_ranks(const ProbeParams& P, uint32_t mask, uint64_t target) {
  for (uint32_t j = 0; j < P.n_ranks; ++j) {
    if (j == P.rank || !((mask >> j) & 1u)) continue;
    st_relaxed_sys(&reinterpret_cast<Ctrl*>(P.base_peer[j])->flags[P.rank].v, target);
  }
}

// Barrier b: b == 0 opens the run, barrier b >= 1 closes phase b - 1.
//   sync = ranks to exchange flags with (signal, then wait): the ranks whose traffic touches the same NVLink ports
//          as this rank's in the phases either side of the barrier (schedule.cc: current partner, next partner and
//          their partners; every rank at open and close).  Symmetric: whoever is waited for also signals.
//   post = ranks that are only signalled, AFTER this rank's own CTAs have been released: the write -> read step
//          inside a round — nobody waits there; the verify job that needs the partner's data polls for it itself.
// A system-scope fence precedes the flag stores only when this rank published something the receiver acts on at
// this barrier (write checksums; the verdicts at the last barrier): reads leave nothing in flight, and each CTA
// already fenced its own remote stores before it arrived.
__device__ void barrier(const ProbeParams& P, Ctx& c, Ctrl* ctrl, int b, uint32_t sync, uint32_t post, bool last) {
  __syncthreads();
  if (threadIdx.x == 0) {
    // the deadline is checked at every arrival, not only inside long waits: a run whose waits all stay short
    // would otherwise finish past timeout_ms without the watchdog ever firing
    const bool ab = check_abort(c);
    if (!ab) {
      const unsigned long long target = P.seq_base + (unsigned long long)b + 1ull;
      // This CTA's accumulator atomics precede the arrive.  Remote stores of a write job were already
      // fenced at system scope by this thread (see the job epilogue), so gpu scope is enough here.
      __threadfence();
      const unsigned int prev = atomicAdd(&ctrl->grid_arrive, 1u);
      if (prev == gridDim.x - 1) {
        // last arriver: every local CTA is done with the phase
        *reinterpret_cast<volatile unsigned int*>(&ctrl->grid_arrive) = 0u;
        __threadfence();
        const uint64_t t_arr = gtimer();
        if (b >= 1 && ctrl->fault.n != 0u) fault_phase_write(P, ctrl, b - 1);
        bool published = false, wrote_done = false;
        if (sync) {
          if (b >= 1) {
            published = publish_writes(P, ctrl, b - 1);
            wrote_done = true;
          }
          if (last) {
            publish_verdicts(P, ctrl);
            published = true;
          }
          if (published) __threadfence_system();  // one fence, then relaxed flag stores that pipeline over NVLink
          signal_ranks(P, sync, target);
          bool timed_out = false;
          for (uint32_t j = 0; j < P.n_ranks && !timed_out; ++j) {
            if (j == P.rank || !((sync >> j) & 1u)) continue;
            timed_out = !spin_until<kScopeSys>(c, &ctrl->flags[j].v, target);
          }
        } else if (last) {
          publish_verdicts(P, ctrl);  // single-rank domains: the verdict word is local
          __threadfence_system();
        }
        const uint64_t t_rel = gtimer();
        ctrl->t_arr[b] = t_arr;
        ctrl->t_rel[b] = t_rel;
        st_release_gpu(&ctrl->grid_release, target);
        // off the critical path: the local CTAs are already running the next phase
        if (post && !aborted(c)) {
          if (b >= 1 && !wrote_done) publish_writes(P, ctrl, b - 1);
          __threadfence_system();
          signal_ranks(P, post, target);
        } else if (b >= 1 && !wrote_done && !aborted(c)) {
          if (publish_writes(P, ctrl, b - 1)) __threadfence_system();  // loop-back write: the owner is this GPU
        }
      } else {
        spin_until<kScopeGpu>(c, &ctrl->grid_release, target);
      }
    }
  }
  __syncthreads();
}

__device__ __forceinline__ uint64_t warp_sum64(uint64_t v) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
  return v;
}
__device__ __forceinline__ uint64_t warp_xor64(uint64_t v) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v ^= __shfl_xor_sync(0xffffffffu, v, m);
  return v;
}
// CTA reduction of the checksums of kJobs jobs, called by every thread: thread 0 adds the CTA's totals into acc[j],
// one atomicAdd and one atomicXor per job.  The warps' partials take the first 2 * kJobs * kWarpsPerCta slots of
// red; what a warp stores into later slots before the call, thread 0 may read after it.
template <int kJobs>
__device__ __forceinline__ void cta_reduce(const Ctx& c, uint64_t* red, const Sum* a, Acc* const* acc) {
#pragma unroll
  for (int j = 0; j < kJobs; ++j) {
    const uint64_t ws = warp_sum64(a[j].s0 + a[j].s1);
    const uint64_t wx = warp_xor64(a[j].x);
    if (c.lane == 0) {
      red[(c.warp * kJobs + j) * 2] = ws;
      red[(c.warp * kJobs + j) * 2 + 1] = wx;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int j = 0; j < kJobs; ++j) {
      uint64_t ts = 0, tx = 0;
#pragma unroll
      for (int w = 0; w < kWarpsPerCta; ++w) {
        ts += red[(w * kJobs + j) * 2];
        tx ^= red[(w * kJobs + j) * 2 + 1];
      }
      atomicAdd(&acc[j]->sum, (unsigned long long)ts);
      atomicXor(&acc[j]->xr, (unsigned long long)tx);
    }
  }
}

// The result row, written into pinned host memory by one whole CTA (every thread calls this), then the
// accumulators are cleared for the next run.  Phase p ran from t_rel[p] to t_arr[p + 1].
__device__ void write_row(const ProbeParams& P, const Ctx& c, Ctrl* ctrl, uint64_t t_enter) {
  ResultRow* row = P.row;
  const bool ab = aborted(c);
  const uint32_t t = threadIdx.x;
  if (t < P.n_phases) {
    PhaseOut o;
    o.t_start = *reinterpret_cast<volatile uint64_t*>(&ctrl->t_rel[t]);
    o.t_arrive = *reinterpret_cast<volatile uint64_t*>(&ctrl->t_arr[t + 1]);
#pragma unroll
    for (int jb = 0; jb < 2; ++jb) {
      const Job job = P.phase[t].job[jb];
      const volatile Acc* acc = &ctrl->acc[t][jb];
      o.t_end[jb] = acc->t_end;
      o.sum[jb] = acc->sum;
      o.xr[jb] = acc->xr;
      o.exp_sum[jb] = 0;
      o.exp_xr[jb] = 0;
      o.verdict[jb] = 0;
      o.code[jb] = job.kind == kJobNone ? kCodeSkipped : (ab ? kCodeAborted : kCodeOk);
      if (!ab) {
        if (job.kind == kJobRead) {
          const Ctrl* pc = reinterpret_cast<const Ctrl*>(P.base_peer[job.peer]);
          const uint32_t slice = P.full_mode ? 0u : job.slot;
          o.exp_sum[jb] = ld_relaxed_sys(&pc->src_sum[slice]);
          o.exp_xr[jb] = ld_relaxed_sys(&pc->src_xor[slice]);
        } else if (job.kind == kJobVerify) {
          o.exp_sum[jb] = ld_relaxed_sys(&ctrl->wr[job.slot].sum);
          o.exp_xr[jb] = ld_relaxed_sys(&ctrl->wr[job.slot].xr);
          o.verdict[jb] = ld_relaxed_sys(&ctrl->wr[job.slot].seq);
        } else if (job.kind == kJobWrite) {
          o.verdict[jb] = ld_relaxed_sys(&ctrl->verdict[job.peer]);
        }
      }
    }
    row->ph[t] = o;
  }
  __syncthreads();
  // reset the accumulators for the next run
  if (t < P.n_phases) {
#pragma unroll
    for (int jb = 0; jb < 2; ++jb) {
      Acc* acc = &ctrl->acc[t][jb];
      acc->sum = 0ull;
      acc->xr = 0ull;
      acc->t_end = 0ull;
    }
  }
  // The row lives in pinned host memory.  One release at system scope by thread 0 publishes it: the other
  // threads' stores are ordered before it through the CTA barrier (cumulativity), so no per-thread
  // fence.sys — each one is a round trip over PCIe.
  __syncthreads();
  if (t == 0) {
    row->t_first = *reinterpret_cast<volatile uint64_t*>(&ctrl->t_rel[0]);
    row->t_last = *reinterpret_cast<volatile uint64_t*>(&ctrl->t_arr[P.n_phases]);
    row->aborted = ab ? 1u : 0u;
    row->n_phases = P.n_phases;
    row->t_enter = t_enter;
    row->t_exit = gtimer();
    st_release_sys(const_cast<uint64_t*>(&row->done), P.run_seq);
  }
}

// ------------------------------------------------- N = 1: one streamed pass ----
// The loop-back phase table (schedule.cc) is [write diag] [read diag || verify diag] and only the verify depends
// on the write.  So instead of walking it with barriers in between, every warp claims write units until none are
// left, then source-read units, then verify units (Walk<true>).  The phase table still names the jobs, the slot
// and the salt, and the row keeps its two phases.
__device__ __forceinline__ bool is_loopback(const ProbeParams& P) {
  if (P.peer_mask != 0u || P.n_phases != 2u) return false;
  const Job& w = P.phase[0].job[0];
  const Job& r = P.phase[1].job[0];
  const Job& v = P.phase[1].job[1];
  const int8_t me = (int8_t)P.rank;
  return w.kind == kJobWrite && P.phase[0].job[1].kind == kJobNone && r.kind == kJobRead && v.kind == kJobVerify &&
         w.peer == me && r.peer == me && v.peer == me && v.writer == P.rank && v.slot == w.slot && v.salt == 0;
}

// Ordering of the verify after the write (the grid barrier's job in the phase walk):
//   writer warp:   its stores complete (bulk: cp.async.bulk.wait_group 0 by the issuing lane; ld/st: every lane's
//                  st.global) -> __syncwarp -> lane 0: fence.proxy.async.global, __threadfence, atomicAdd of the
//                  units it stored onto lb.written (a gpu-scope release)
//   verifier warp: lane 0 spins on ld.acquire.gpu of lb.written until it reaches the slot's unit count ->
//                  __syncwarp -> loads (the bulk path issues fence.proxy.async.global before its first load).
// Counting units rather than warps means no warp waits for a CTA that has not started: the units are all claimed
// by CTAs that are running.  An armed landing fault counts as one more unit: the writer warp whose atomicAdd
// completes the slot's count applies it between two __threadfence and then adds 1, and the verifiers wait for that.
// The CTA that finishes last (lb.done) publishes the write checksum and the verdict,
// writes the row and zeroes the counters for the next run.
__device__ void loopback_pass(const ProbeParams& P, Ctx& c, Ctrl* ctrl, uint64_t* red, uint64_t t_enter) {
  constexpr int kRed = 6 + 5;  // per warp: (sum, xor) x 3 jobs (cta_reduce), end time x 3 jobs, first issue x 2 jobs
  static_assert(kWarpsPerCta * (kStages + kRed) * 8 <= kSmemBytes - kWarpsPerCta * kStages * kUnitBytes,
                "mbarriers + reduction slots fit the tail of the dynamic shared memory");
  __shared__ bool s_last;
  __shared__ uint64_t s_t_enter;
  LoopBack* lb = &ctrl->lb;
  const Job wj = P.phase[0].job[0];
  uint8_t* self = P.base_peer[P.rank];
  uint8_t* slot = self + P.land_off + (uint64_t)wj.slot * P.bpp;
  const uint8_t* src = self + P.src_off + (P.full_mode ? 0ull : (uint64_t)P.phase[1].job[0].slot * P.bpp);
  const uint64_t n_units = units_of(P.bpp);
  if (threadIdx.x == 0) atomicMax(&lb->t_enter_n, ~t_enter);

  Sum a[3] = {};                    // write, source read, verify
  uint64_t t_end[3] = {0ull, 0ull, 0ull};  // per job: when this warp's last unit was done (0: it did none)
  uint64_t t_first[2];              // when this warp started the write and the source read

  t_first[0] = gtimer();
  const uint32_t n_wr = write_units(c, P.path, slot, P.bpp, claimed(P.bpp, &lb->claim[0].v), wj.salt, a[0]);
  __syncwarp();
  if (n_wr) {
    if (c.lane == 0) {
      fence_proxy_async_global();
      __threadfence();
      const unsigned long long before = atomicAdd(&lb->written.v, (unsigned long long)n_wr);
      if (before + n_wr == n_units && fault_armed(P, ctrl, P.rank)) {
        // the whole slot is stored: an armed landing fault goes in now and counts as one more unit, so the
        // verifiers, which wait for n_units + 1, read it (acquire of every writer's release, then release again)
        __threadfence();
        xor_landing(&ctrl->fault, slot);
        __threadfence();
        atomicAdd(&lb->written.v, 1ull);
      }
    }
    t_end[0] = gtimer();
  }

  t_first[1] = gtimer();
  if (read_units(c, P.path, src, P.bpp, claimed(P.bpp, &lb->claim[1].v), a[1])) t_end[1] = gtimer();

  bool go = true;
  // deadline checked at the transition too, as at a barrier arrival
  if (c.lane == 0)
    go = !check_abort(c) &&
         spin_until<kScopeGpu>(c, &lb->written.v, n_units + (fault_armed(P, ctrl, P.rank) ? 1u : 0u));
  go = __shfl_sync(0xffffffffu, go, 0);
  if (go && read_units(c, P.path, slot, P.bpp, claimed(P.bpp, &lb->claim[2].v), a[2])) t_end[2] = gtimer();

  // CTA reduce -> one set of atomics per CTA; the times take the slots after the checksums'
  uint64_t* red_t = red + 6 * kWarpsPerCta;
  if (c.lane == 0) {
#pragma unroll
    for (int j = 0; j < 3; ++j) red_t[c.warp * 5 + j] = t_end[j];
    red_t[c.warp * 5 + 3] = t_first[0];
    red_t[c.warp * 5 + 4] = t_first[1];
  }
  Acc* const acc[3] = {&ctrl->acc[0][0], &ctrl->acc[1][0], &ctrl->acc[1][1]};
  cta_reduce<3>(c, red, a, acc);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      uint64_t te = 0, tf = ~0ull;
#pragma unroll
      for (int w = 0; w < kWarpsPerCta; ++w) {
        te = max(te, red_t[w * 5 + j]);
        if (j < 2) tf = min(tf, red_t[w * 5 + 3 + j]);
      }
      if (te) atomicMax(&acc[j]->t_end, (unsigned long long)te);
      if (j < 2) atomicMax(&lb->t_first_n[j], ~tf);
    }
    __threadfence();
    const bool last = atomicAdd(&lb->done.v, 1ull) == gridDim.x - 1;
    if (last) {
      // every CTA is done: its accumulator atomics precede its arrival on lb.done
      __threadfence();
      const volatile LoopBack* vlb = lb;
      ctrl->t_rel[0] = ~vlb->t_first_n[0];
      ctrl->t_rel[1] = ~vlb->t_first_n[1];
      ctrl->t_arr[1] = *reinterpret_cast<volatile unsigned long long*>(&ctrl->acc[0][0].t_end);
      ctrl->t_arr[2] = gtimer();
      s_t_enter = ~vlb->t_enter_n;
      if (!aborted(c)) {
        publish_writes(P, ctrl, 0);  // the owner of the slot is this GPU
        publish_verdicts(P, ctrl);
      }
      __threadfence();
    }
    s_last = last;
  }
  __syncthreads();
  if (!s_last) return;
  write_row(P, c, ctrl, s_t_enter);
  if (threadIdx.x == 0) {
    for (int j = 0; j < 3; ++j) lb->claim[j].v = 0ull;
    lb->written.v = 0ull;
    lb->done.v = 0ull;
    lb->t_first_n[0] = lb->t_first_n[1] = 0ull;
    lb->t_enter_n = 0ull;
  }
}

}  // namespace

// ------------------------------------------------- the persistent kernel ----
__global__ void __launch_bounds__(kThreads, 1) cdprobe_kernel(const __grid_constant__ ProbeParams P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kWarpsPerCta * kStages * kUnitBytes);
  uint64_t* red = bars + kWarpsPerCta * kStages;  // CTA reduction slots: 2 per warp, 11 in the loop-back pass
  __shared__ uint64_t s_deadline;

  Ctx c;
  Ctrl* const ctrl = reinterpret_cast<Ctrl*>(P.base_peer[P.rank]);
  c.abort_word = &ctrl->abort_flag;
  c.warp = threadIdx.x >> 5;
  c.lane = threadIdx.x & 31;
  c.stage_smem = smem_u32(smem) + c.warp * kStages * kUnitBytes;
  c.bar_smem = smem_u32(bars) + c.warp * kStages * 8u;
  c.parity_bits = 0u;
  __shared__ uint64_t s_enter;
  if (threadIdx.x == 0) {
    s_enter = gtimer();
    s_deadline = s_enter + P.timeout_ns;
  }
  if (c.lane == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) mbar_init(c.bar_smem + 8u * s, 1u);
    fence_mbar_init();
  }
  __syncthreads();
  c.deadline = s_deadline;

  if (is_loopback(P)) {
    loopback_pass(P, c, ctrl, red, s_enter);
    return;
  }

  barrier(P, c, ctrl, 0, P.peer_mask, 0u, false);

  for (uint32_t ph = 0; ph < P.n_phases; ++ph) {
    const Phase& phd = P.phase[ph];
#pragma unroll
    for (int jb = 0; jb < 2; ++jb) {
      const Job job = phd.job[jb];
      if (job.kind == kJobNone) continue;
      if (blockIdx.x < job.cta0 || blockIdx.x >= (uint32_t)job.cta0 + job.nctas) continue;
      Sum a{0ull, 0ull, 0ull};
      if (!aborted(c)) {
        const uint32_t gwarp = (blockIdx.x - job.cta0) * kWarpsPerCta + c.warp;
        const uint32_t nwarps = (uint32_t)job.nctas * kWarpsPerCta;
        uint8_t* pb = P.base_peer[job.peer];
        if (job.kind == kJobWarm) {
          // untimed link wake-up: stream a prefix of the partner's slice (result ignored)
          const uint8_t* src = pb + P.src_off + (P.full_mode ? 0ull : (uint64_t)job.slot * P.bpp);
          const uint64_t nb = job.salt < P.bpp ? job.salt : P.bpp;
          if (nb) read_units(c, P.path, src, nb, strided(nb, gwarp, nwarps), a);
        } else if (job.kind == kJobRead) {
          const uint8_t* src = pb + P.src_off + (P.full_mode ? 0ull : (uint64_t)job.slot * P.bpp);
          read_units(c, P.path, src, P.bpp, strided(P.bpp, gwarp, nwarps), a);
        } else if (job.kind == kJobVerify) {
          // the slot's writer signals when its write phase is over (and its checksums are published); where the
          // schedule put no wait between that phase and this one (post_mask), this job does the waiting
          bool go = true;
          if (job.salt != 0 && job.writer != P.rank && P.base_peer[job.writer] != nullptr) {
            if (threadIdx.x == 0) spin_until<kScopeSys>(c, &ctrl->flags[job.writer].v, P.seq_base + job.salt + 1ull);
            __syncthreads();
            go = !aborted(c);
          }
          if (go) {
            const uint8_t* src = pb + P.land_off + (uint64_t)job.slot * P.bpp;
            read_units(c, P.path, src, P.bpp, strided(P.bpp, gwarp, nwarps), a);
          }
        } else {
          uint8_t* dst = pb + P.land_off + (uint64_t)job.slot * P.bpp;
          write_units(c, P.path, dst, P.bpp, strided(P.bpp, gwarp, nwarps), job.salt, a);
        }
      }
      // CTA reduce -> one atomic per CTA into the phase accumulator
      Acc* const acc = &ctrl->acc[ph][jb];
      cta_reduce<1>(c, red, &a, &acc);
      if (threadIdx.x == 0) {
        if (job.kind == kJobWrite) __threadfence_system();  // stores have reached the peer
        atomicMax(&acc->t_end, (unsigned long long)gtimer());
      }
    }
    barrier(P, c, ctrl, (int)ph + 1, phd.sync_mask & P.peer_mask, phd.post_mask & P.peer_mask, ph + 1 == P.n_phases);
  }

  // ---- output: CTA 0 writes the result row ----------------------------------
  if (blockIdx.x == 0) write_row(P, c, ctrl, s_enter);
}

// ------------------------------------------------------- source pattern ----
__global__ void __launch_bounds__(256) cdprobe_fill_src_kernel(uint4* dst, uint64_t nvec, uint64_t seed, uint32_t rank) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    const uint64_t w0 = src_word(seed, rank, 2 * v), w1 = src_word(seed, rank, 2 * v + 1);
    dst[v] = make_uint4((uint32_t)w0, (uint32_t)(w0 >> 32), (uint32_t)w1, (uint32_t)(w1 >> 32));
  }
}

// ------------------------------------------- K5: bandwidth versus size ----
namespace {
// The entry of bwcurve_kernel and allreduce_kernel, in the probe kernel's shared-memory layout: the warp's stages and
// mbarriers (initialised here), the launch's abort word and the deadline timeout_ns from now.  *red gets the CTA
// reduction slots.  cdprobe_kernel has its own copy, which also stamps its entry time.
__device__ __forceinline__ Ctx enter(uint8_t* smem, unsigned int* abort_word, uint64_t timeout_ns, uint64_t** red) {
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kWarpsPerCta * kStages * kUnitBytes);
  *red = bars + kWarpsPerCta * kStages;
  __shared__ uint64_t s_deadline;
  Ctx c;
  c.abort_word = abort_word;
  c.warp = threadIdx.x >> 5;
  c.lane = threadIdx.x & 31;
  c.stage_smem = smem_u32(smem) + c.warp * kStages * kUnitBytes;
  c.bar_smem = smem_u32(bars) + c.warp * kStages * 8u;
  c.parity_bits = 0u;
  if (threadIdx.x == 0) s_deadline = gtimer() + timeout_ns;
  if (c.lane == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) mbar_init(c.bar_smem + 8u * s, 1u);
    fence_mbar_init();
  }
  __syncthreads();
  c.deadline = s_deadline;
  return c;
}

// Grid barrier b of a bwcurve_kernel, allreduce_kernel or alltoall_kernel launch, called by every thread.  Arrivals
// count on one word that only rises, so barrier b is complete at (b + 1) x gridDim.x arrivals; the CTA that completes it
// stamps *t_rel (unless null) and releases b + 1.  Given peer lines (dom), it is a domain barrier: before the stamp,
// that CTA stores (call_seq << 16) | (b + 1) into the lines dom names (st.relaxed.sys) and waits until every line it
// waits on holds at least that (ld.acquire.sys).  `fence`: a fence.sys precedes those stores, for a barrier that
// publishes this rank's stores to its peers; the all-reduce's inputs are written at open and its output is local, so
// its barriers need none.  Returns false in every thread once the launch is aborted (the deadline is checked at every
// arrival, as in barrier()).
__device__ bool grid_barrier(const Ctx& c, BwScratch* bs, uint32_t b, unsigned long long* t_rel,
                             const DomainLines* dom, bool fence) {
  __shared__ bool s_go;
  __syncthreads();
  if (threadIdx.x == 0) {
    bool go = !check_abort(c);
    if (go) {
      const unsigned int prev = atomicAdd(&bs->arrive, 1u);
      if (prev == (b + 1u) * gridDim.x - 1u) {
        if (dom != nullptr) {
          const uint64_t v = (dom->call_seq << kArBarrierBits) | (b + 1ull);
          if (fence) __threadfence_system();
          if (dom->self != nullptr) st_relaxed_sys(dom->self, v);
          for (uint32_t j = 0; j < (uint32_t)kMaxRanks; ++j)
            if (dom->sig_out[j] != nullptr) st_relaxed_sys(dom->sig_out[j], v);
          for (uint32_t j = 0; j < (uint32_t)kMaxRanks && go; ++j)
            if (dom->sig_in[j] != nullptr) go = spin_until<kScopeSys>(c, dom->sig_in[j], v);
        }
        if (go) {
          if (t_rel != nullptr) *t_rel = gtimer();
          st_release_gpu(&bs->release, b + 1ull);
        }
      } else {
        go = spin_until<kScopeGpu>(c, &bs->release, b + 1ull);
      }
    }
    s_go = go;
  }
  __syncthreads();
  return s_go;
}
}  // namespace

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

// The per-granule (sum, xor) of a region whose word k is word(k), from the pattern definition: one warp per 16 KiB
// granule.  Instantiated for bwcurve's source slices (SrcRegionWord) and the all-reduce output (AllReduceWord).
template <typename Word>
__global__ void __launch_bounds__(256) granules_kernel(uint64_t* gsum, uint64_t* gxor, Word word, uint64_t n_granules) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t nwarps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  for (uint64_t g = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < n_granules; g += nwarps) {
    uint64_t s = 0, x = 0;
    for (uint32_t k = lane; k < kGranuleWords; k += 32) {
      const uint64_t w = word(g * kGranuleWords + k);
      s += w;
      x ^= w;
    }
    s = warp_sum64(s);
    x = warp_xor64(x);
    if (lane == 0) {
      gsum[g] = s;
      gxor[g] = x;
    }
  }
}

// ------------------------------------------- K6: one-shot all-reduce ----
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

// TMA read side: the warp walks (unit, input) pairs, the n inputs of a unit in a row, through its kStages-deep ring of
// bulk loads, one load per pair.  Each stage is added into the accumulators and then refilled with the next pair, so
// the ring runs on across unit boundaries.  Aborted: stops issuing and drains what is in flight.
__device__ void ar_units_tma(Ctx& c, const AllReduceParams& P, uint64_t bytes, Walk<false> walk, uint64_t fw, Sum& a) {
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
      ar_store<16>(c, P.out, u, len, fw, acc, a);
      csrc = 0;
      more = walk.take(c, u);
    }
  }
}

// ld/st read side: for each unit, the n inputs one after another, kLdstVecs 16-byte loads in flight per lane each.
template <uint32_t kLaneBytes>
__device__ void ar_units_ldst(const Ctx& c, const AllReduceParams& P, uint64_t bytes, Walk<false> walk, uint64_t fw,
                              Sum& a) {
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
    ar_store<kLaneBytes>(c, P.out, u, len, fw, acc, a);
  }
}

__device__ __forceinline__ uint64_t warp_min64(uint64_t v) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v = min(v, (uint64_t)__shfl_xor_sync(0xffffffffu, v, m));
  return v;
}

// The untimed word check of the output the last rep of size k stored: each lane compares every 32nd word of its
// warp's share with allreduce_word, reading at L2 (other SMs stored them).  One atomic pair per warp with a bad word.
__device__ void ar_check(const Ctx& c, const AllReduceParams& P, ArScratch* as, uint32_t k, uint64_t bytes,
                         uint32_t gwarp, uint32_t nwarps) {
  const unsigned long long* out = reinterpret_cast<const unsigned long long*>(P.out);
  const uint64_t words = bytes / 8;
  uint64_t bad = 0, first = ~0ull;
  for (uint64_t w = (uint64_t)gwarp * 32u + (uint32_t)c.lane; w < words; w += (uint64_t)nwarps * 32u) {
    if (__ldcg(out + w) != allreduce_word(P.seed, P.n, w)) {
      ++bad;
      first = min(first, w * 8u);
    }
  }
  bad = warp_sum64(bad);
  first = warp_min64(first);
  if (c.lane == 0 && bad != 0) {
    atomicAdd(&as->bad_words[k], (unsigned long long)bad);
    atomicMax(&as->first_bad_n[k], (unsigned long long)~first);
  }
}
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
      if (P.path == 2u) ar_units_ldst<32>(c, P, bytes, walk, fw, a);
      else if (P.path == 1u) ar_units_ldst<16>(c, P, bytes, walk, fw, a);
      else ar_units_tma(c, P, bytes, walk, fw, a);
      __threadfence();  // this warp's stores are performed before the CTA's completion stamp
      Acc* const acc = &bs->rep[k][r];
      cta_reduce<1>(c, red, &a, &acc);
      if (threadIdx.x == 0) atomicMax(&acc->t_end, (unsigned long long)gtimer());
    }
    if (!grid_barrier(c, bs, b++, nullptr, nullptr, false)) return;
    ar_check(c, P, as, k, bytes, gwarp, nwarps);
  }
}

// ------------------------------------------------ K7: one-shot all-to-all ----
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

// ----------------------------------------------------------- launchers -----
namespace {
// Launches a persistent kernel (cdprobe_kernel, bwcurve_kernel or allreduce_kernel) on `stream` of the current device:
// `grid` CTAs of kThreads threads and kSmemBytes of dynamic shared memory, cooperative or not.  Returns a cudaError_t.
template <typename Params>
int grid_launch(void (*kernel)(Params), const Params& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  void* args[] = {const_cast<Params*>(&p)};
  const void* f = reinterpret_cast<const void*>(kernel);
  return (int)(cooperative ? cudaLaunchCooperativeKernel(f, dim3(grid), dim3(kThreads), args, kSmemBytes, stream)
                           : cudaLaunchKernel(f, dim3(grid), dim3(kThreads), args, kSmemBytes, stream));
}
}  // namespace

int probe_kernel_prepare(int* max_ctas_per_sm) {
  cudaError_t e = cudaFuncSetAttribute(cdprobe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
  if (e != cudaSuccess) return (int)e;
  int nb = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, cdprobe_kernel, kThreads, kSmemBytes);
  if (e != cudaSuccess) return (int)e;
  if (max_ctas_per_sm) *max_ctas_per_sm = nb;
  return 0;
}

int probe_kernel_launch(const ProbeParams* p, unsigned grid, bool cooperative, cudaStream_t stream) {
  return grid_launch(cdprobe_kernel, *p, grid, cooperative, stream);
}

int probe_fill_launch(void* dst, uint64_t bytes, uint64_t seed, uint32_t rank, unsigned grid, cudaStream_t stream) {
  cdprobe_fill_src_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<uint4*>(dst), bytes / 16, seed, rank);
  return (int)cudaGetLastError();
}

int bwcurve_launch(const BwCurveParams& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  const cudaError_t e =
      cudaFuncSetAttribute(bwcurve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
  return e != cudaSuccess ? (int)e : grid_launch(bwcurve_kernel, p, grid, cooperative, stream);
}

int allreduce_launch(const AllReduceParams& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  const cudaError_t e =
      cudaFuncSetAttribute(allreduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
  return e != cudaSuccess ? (int)e : grid_launch(allreduce_kernel, p, grid, cooperative, stream);
}

int alltoall_launch(const AllToAllParams& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  const cudaError_t e =
      cudaFuncSetAttribute(alltoall_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
  return e != cudaSuccess ? (int)e : grid_launch(alltoall_kernel, p, grid, cooperative, stream);
}

template <typename Word>
int granules_launch(uint64_t* gsum, uint64_t* gxor, const Word& word, uint64_t n_granules, unsigned grid,
                    cudaStream_t stream) {
  if (n_granules == 0) return (int)cudaSuccess;
  const uint64_t need = (n_granules + 7) / 8;  // eight warps per block
  granules_kernel<<<need < grid ? (unsigned)need : grid, 256, 0, stream>>>(gsum, gxor, word, n_granules);
  return (int)cudaGetLastError();
}
template int granules_launch(uint64_t*, uint64_t*, const SrcRegionWord&, uint64_t, unsigned, cudaStream_t);
template int granules_launch(uint64_t*, uint64_t*, const AllReduceWord&, uint64_t, unsigned, cudaStream_t);

}  // namespace cdp
