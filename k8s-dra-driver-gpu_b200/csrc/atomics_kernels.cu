// atomics_kernels.cu — sm_90a kernels of cdprobe_atomics: system-scope 64-bit atomics on a peer's word, timed with
// %globaltimer on the issuing GPU.
//
// One 32-thread block per cell, on the issuer's stream.  In the two chain kinds lane 0 works and the other lanes exit;
// in CONTENDED all 32 lanes run fetch-add chains on the same word.  Every atomic is atom.relaxed.sys.global
// (ATOMG.E.*.64.STRONG.SYS): the owner's L2 performs it and returns the old value to the issuer.
//
// Each rep opens with lane 0's atom.exch of its start value (probe_types.h, atomics_start); the opening timer read
// comes after that exch has returned, and the closing one after the last returned value has been used.  An add whose
// operand is a constant does not wait for the add before it (nvcc unrolls such a loop into several ATOMGs in flight
// per lane), so every op's operand is computed from the previous op's return: 1 + (r >> 63), which is 1 because no
// value the word holds has bit 63 set.  A CAS compares with the previous return + 1, so its chain is dependent by
// construction.  After the timed region lane 0 reads the word back with ld.relaxed.sys.  The device deadline
// (timeout_ms from kernel entry) is checked every 64 ops.
//
// probe_kernels.cu is untouched: the probe kernel's code generation does not depend on this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cdprobe.h"
#include "atomics.h"

namespace cdp {
namespace {

constexpr unsigned kFullMask = 0xFFFFFFFFu;

__device__ __forceinline__ uint64_t atom_exch(unsigned long long* p, uint64_t v) {
  uint64_t r;
  asm volatile("atom.relaxed.sys.global.exch.b64 %0, [%1], %2;" : "=l"(r) : "l"(p), "l"(v) : "memory");
  return r;
}
__device__ __forceinline__ uint64_t atom_add(unsigned long long* p, uint64_t v) {
  uint64_t r;
  asm volatile("atom.relaxed.sys.global.add.u64 %0, [%1], %2;" : "=l"(r) : "l"(p), "l"(v) : "memory");
  return r;
}
__device__ __forceinline__ uint64_t atom_cas(unsigned long long* p, uint64_t cmp, uint64_t v) {
  uint64_t r;
  asm volatile("atom.relaxed.sys.global.cas.b64 %0, [%1], %2, %3;" : "=l"(r) : "l"(p), "l"(cmp), "l"(v) : "memory");
  return r;
}
__device__ __forceinline__ uint64_t ld_relaxed_sys(const unsigned long long* p) {
  uint64_t v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// FETCH_ADD and CAS: one lane, `ops` dependent atomics per rep; op k must return start + k.
template <bool kCas>
__global__ void __launch_bounds__(32) atomics_chain_kernel(const __grid_constant__ AtomicsParams p, TimedRep* out) {
  if (threadIdx.x != 0) return;
  unsigned long long* const w = p.cell[blockIdx.x].word;
  TimedRep* o = out + (size_t)blockIdx.x * kRepSlots;
  const uint64_t deadline = globaltimer() + p.timeout_ns;
  for (uint32_t r = 0; r <= p.reps; ++r) {
    const uint64_t start = atomics_start(p.call_seq, kCas ? CDPROBE_ATOMIC_CAS : CDPROBE_ATOMIC_FETCH_ADD, r);
    const uint64_t extra = blockIdx.x == p.fault_cell && r == 1 ? 1u : 0u;  // the armed fault: op 0 steps by 2
    // The shuffle consumes the exch's return before the timer read, so the read cannot issue before the exch is back
    // (the asm operand of globaltimer_after alone orders the two only in the front end: ptxas may hoist the read).
    const uint64_t prev = __shfl_sync(1u, atom_exch(w, start), 0);
    const uint64_t t0 = globaltimer_after(prev);
    // op 0 waits for the exch through its operand (prev >> 63 is 0)
    uint64_t x = kCas ? atom_cas(w, start | (prev >> 63), start + 1 + extra) : atom_add(w, 1 + extra + (prev >> 63));
    uint64_t digest = x;
    bool bad = x != start;
    int32_t status = 0;
    for (uint32_t k = 1; k < p.ops; ++k) {
      if (kCas) {
        const uint64_t v = x + 1;
        x = atom_cas(w, v, v + 1);
      } else {
        x = atom_add(w, 1 + (x >> 63));
      }
      digest ^= x;
      bad |= x != start + k;
      if ((k & 63u) == 63u && globaltimer() > deadline) {
        status = CDPROBE_ERR_TIMEOUT;
        break;
      }
    }
    const uint64_t t1 = globaltimer_after(x);
    if (status == 0 && (bad || ld_relaxed_sys(w) != start + p.ops)) status = CDPROBE_ERR_INTEGRITY;
    o[r].ns = t1 - t0;
    o[r].digest = digest;
    o[r].status = status;
    if (status == CDPROBE_ERR_TIMEOUT) return;
  }
}

__device__ __forceinline__ uint64_t warp_sum(uint64_t v) {
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(kFullMask, v, d);
  return v;
}
__device__ __forceinline__ uint64_t warp_xor(uint64_t v) {
  for (int d = 16; d > 0; d >>= 1) v ^= __shfl_xor_sync(kFullMask, v, d);
  return v;
}

// CONTENDED: 32 lanes, `ops` dependent fetch-adds each on the same word.  The returns over the warp must be exactly
// start .. start + 32 * ops - 1; their sum is checked here, their xor by the host.
__global__ void __launch_bounds__(32) atomics_contended_kernel(const __grid_constant__ AtomicsParams p, TimedRep* out) {
  const uint32_t lane = threadIdx.x;
  unsigned long long* const w = p.cell[blockIdx.x].word;
  TimedRep* o = out + (size_t)blockIdx.x * kRepSlots;
  const uint64_t deadline = globaltimer() + p.timeout_ns;
  const uint64_t total = 32ull * p.ops;
  for (uint32_t r = 0; r <= p.reps; ++r) {
    const uint64_t start = atomics_start(p.call_seq, CDPROBE_ATOMIC_CONTENDED, r);
    const uint64_t extra = lane == 0 && blockIdx.x == p.fault_cell && r == 1 ? 1u : 0u;
    uint64_t prev = 0;
    if (lane == 0) prev = atom_exch(w, start);
    // every lane's first add waits for the exch through its operand, and the timer read after the shuffle does too
    prev = __shfl_sync(kFullMask, prev, 0);
    __syncwarp();
    const uint64_t t0 = globaltimer_after(prev);
    uint64_t x = atom_add(w, 1 + extra + (prev >> 63));
    uint64_t sum = x, digest = x;
    bool timed_out = false;
    for (uint32_t k = 1; k < p.ops; ++k) {
      x = atom_add(w, 1 + (x >> 63));
      sum += x;
      digest ^= x;
      if ((k & 63u) == 63u && __any_sync(kFullMask, globaltimer() > deadline)) {  // warp-uniform break
        timed_out = true;
        break;
      }
    }
    sum = warp_sum(sum);
    digest = warp_xor(digest);
    const uint64_t t1 = globaltimer_after(sum);
    __syncwarp();
    if (lane == 0) {
      int32_t status = 0;
      if (timed_out) status = CDPROBE_ERR_TIMEOUT;
      else if (sum != atomics_rep_sum(start, total) || ld_relaxed_sys(w) != start + total) status = CDPROBE_ERR_INTEGRITY;
      o[r].ns = t1 - t0;
      o[r].digest = digest;
      o[r].status = status;
    }
    if (timed_out) return;
  }
}

}  // namespace

int atomics_launch(const AtomicsParams& p, uint32_t kind, TimedRep* out, cudaStream_t stream) {
  if (p.n_cells == 0) return (int)cudaSuccess;
  if (kind == CDPROBE_ATOMIC_FETCH_ADD) atomics_chain_kernel<false><<<p.n_cells, 32, 0, stream>>>(p, out);
  else if (kind == CDPROBE_ATOMIC_CAS) atomics_chain_kernel<true><<<p.n_cells, 32, 0, stream>>>(p, out);
  else atomics_contended_kernel<<<p.n_cells, 32, 0, stream>>>(p, out);
  return (int)cudaGetLastError();
}

}  // namespace cdp
