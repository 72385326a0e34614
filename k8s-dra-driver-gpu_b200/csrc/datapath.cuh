// datapath.cuh — the sm_90a device code that more than one persistent kernel uses: cdprobe_kernel (probe_kernels.cu),
// bwcurve_kernel (bwcurve_kernels.cu), allreduce_kernel (allreduce_kernels.cu) and alltoall_kernel
// (alltoall_kernels.cu).
//
//   * the PTX wrappers, the launch context (Ctx) with its abort and deadline checks, and the spin-waits;
//   * the unit walks, the (S, X) checksum and the write pattern;
//   * the data path: the K1/K4 read jobs and the K2 write jobs (probe_kernels.cu names K1-K4) on TMA bulk copies or
//     16- / 32-byte ld/st, picked at run time by read_units / write_units;
//   * the CTA reduction of the checksums;
//   * for the grid measurements: their kernel entry (enter), their grid / domain barrier (grid_barrier) and the
//     granule-sum kernel (granules_kernel, instantiated by the unit of the measurement that uses it);
//   * the launcher of the persistent kernels (grid_launch).
//
// Everything but the granule-sum templates has internal linkage, so every translation unit that includes this header
// compiles its own copy, as with timed_rep.cuh: a kernel's code generation depends on this header and on its own file,
// not on the other kernels.  Each granules_launch instantiation lives in exactly one unit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "bwcurve.h"
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

// ------------------------------------------------------ CTA reduction ----
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
__device__ __forceinline__ uint64_t warp_min64(uint64_t v) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v = min(v, (uint64_t)__shfl_xor_sync(0xffffffffu, v, m));
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

// ----------------------------------------------- the grid measurements ----
// The entry of bwcurve_kernel, allreduce_kernel and alltoall_kernel, in the probe kernel's shared-memory layout: the
// warp's stages and mbarriers (initialised here), the launch's abort word and the deadline timeout_ns from now.  *red
// gets the CTA reduction slots.  cdprobe_kernel has its own copy, which also stamps its entry time.
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
// arrival, as in probe_kernels.cu's barrier()).
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

// The per-granule (sum, xor) of a region whose word k is word(k), from the pattern definition: one warp per 16 KiB
// granule.  Instantiated for bwcurve's source slices (SrcRegionWord, in bwcurve_kernels.cu) and the all-reduce output
// (AllReduceWord, in allreduce_kernels.cu).
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

template <typename Word>
int granules_launch(uint64_t* gsum, uint64_t* gxor, const Word& word, uint64_t n_granules, unsigned grid,
                    cudaStream_t stream) {
  if (n_granules == 0) return (int)cudaSuccess;
  const uint64_t need = (n_granules + 7) / 8;  // eight warps per block
  granules_kernel<<<need < grid ? (unsigned)need : grid, 256, 0, stream>>>(gsum, gxor, word, n_granules);
  return (int)cudaGetLastError();
}

// ----------------------------------------------------------- launcher -----
namespace {
// Launches a persistent kernel (cdprobe_kernel, bwcurve_kernel, alltoall_kernel or one of the six all-reduce kernels)
// on `stream` of the current device: `grid` CTAs of kThreads threads and kSmemBytes of dynamic shared memory,
// cooperative or not.  Sets the kernel's dynamic shared-memory limit to kSmemBytes first, on every launch; for
// cdprobe_kernel, whose launcher has already set it before its occupancy check, that is one redundant driver call.
// Returns a cudaError_t.
template <typename Params>
int grid_launch(void (*kernel)(Params), const Params& p, unsigned grid, bool cooperative, cudaStream_t stream) {
  const void* f = reinterpret_cast<const void*>(kernel);
  const cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
  if (e != cudaSuccess) return (int)e;
  void* args[] = {const_cast<Params*>(&p)};
  return (int)(cooperative ? cudaLaunchCooperativeKernel(f, dim3(grid), dim3(kThreads), args, kSmemBytes, stream)
                           : cudaLaunchKernel(f, dim3(grid), dim3(kThreads), args, kSmemBytes, stream));
}
}  // namespace

}  // namespace cdp
