// pingpong_kernels.cu — sm_90a kernel of cdprobe_pingpong: the K3 barrier's cross-GPU signal, timed as a round trip
// with %globaltimer on the initiating GPU.
//
// One 32-thread block per local rank; lane 0 works and the other lanes exit.  The block walks the tournament's rounds;
// in each round it runs two legs with its partner, the lower rank initiating first.  In a leg the initiator stores a
// word into its line in the partner's memory and polls its own copy of the partner's line for the echo; the responder
// polls its local copy for the ping and stores the echo (received + 1) into its line in the initiator's memory.
// Between the legs, leg 0's initiator stores a hand-over word once it has read the last echo, and leg 1's initiator
// waits for it before its first ping (untimed, outside the digest).
// These are the barrier's own operations (probe_kernels.cu, signal_ranks; datapath.cuh, spin_until): every store is
// st.relaxed.sys (STG.E.64.STRONG.SYS), every poll ld.acquire.sys, and the fenced variant puts the barrier's
// system-scope fence (__threadfence_system, as after publish_writes / publish_verdicts) before each store.
//
// Every wait is for a word >= the expected one, followed by an equality check; words rise strictly (probe_types.h,
// pingpong_word), so no stale word satisfies a wait and a larger one fails the check at once.  The device deadline
// (timeout_ms from kernel entry) is checked every 64 spins of a poll; past it, the kernel marks the cells it has not
// finished initiating CDPROBE_ERR_TIMEOUT and exits.
//
// probe_kernels.cu is untouched: the probe kernel's code generation does not depend on this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cdprobe.h"
#include "pingpong.h"

namespace cdp {
namespace {

__device__ __forceinline__ uint64_t ld_acquire_sys(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// Spins until the word at p is >= want; v gets the word that ended the wait.  False: the deadline passed.
__device__ __forceinline__ bool poll(const uint64_t* p, uint64_t want, uint64_t deadline, uint64_t& v) {
  uint32_t spins = 0;
  while ((v = ld_acquire_sys(p)) < want) {
    if ((++spins & 63u) == 0u && globaltimer() > deadline) return false;
  }
  return true;
}

template <bool kFenced>
__device__ __forceinline__ void signal(uint64_t* p, uint64_t w) {
  if (kFenced) __threadfence_system();
  st_relaxed_sys(p, w);
}

// The initiator's side of one leg: the warm-up rep, then p.reps timed reps of p.trips round trips.
template <bool kFenced>
__device__ bool initiate(const PingPongParams& p, const PingPongRound& R, uint32_t r, uint32_t leg, uint64_t deadline,
                         TimedRep* o) {
  for (uint32_t rep = 0; rep <= p.reps; ++rep) {
    const uint64_t base = pingpong_word(p.call_seq, r, leg, rep, 0, 0);
    uint64_t digest = 0, v = 0;
    int32_t status = 0;
    const uint64_t t0 = globaltimer();
    for (uint32_t trip = 0; trip < p.trips; ++trip) {
      const uint64_t ping = base + 2ull * trip;
      signal<kFenced>(R.remote, ping);
      if (!poll(R.local, ping + 1, deadline, v)) {
        status = CDPROBE_ERR_TIMEOUT;
        break;
      }
      digest ^= v;
      if (v != ping + 1) status = CDPROBE_ERR_INTEGRITY;
    }
    const uint64_t t1 = globaltimer_after(v);
    o[rep].ns = t1 - t0;
    o[rep].digest = digest;
    o[rep].status = status;
    if (status == CDPROBE_ERR_TIMEOUT) return false;
  }
  return true;
}

// The responder's side of one leg: echo every ping as received + 1, so a wrong ping becomes a wrong echo.
template <bool kFenced>
__device__ bool respond(const PingPongParams& p, const PingPongRound& R, uint32_t r, uint32_t leg, uint64_t deadline) {
  for (uint32_t rep = 0; rep <= p.reps; ++rep) {
    const uint64_t base = pingpong_word(p.call_seq, r, leg, rep, 0, 0);
    for (uint32_t trip = 0; trip < p.trips; ++trip) {
      const uint64_t ping = base + 2ull * trip;
      uint64_t v;
      if (!poll(R.local, ping, deadline, v)) return false;
      uint64_t echo = v + 1;
      if (r == p.fault_round && rep == 1 && trip == p.fault_trip) echo = ping + 3;  // the echo of trip + 1
      signal<kFenced>(R.remote, echo);
    }
  }
  return true;
}

template <bool kFenced>
__global__ void __launch_bounds__(32) pingpong_kernel(const __grid_constant__ PingPongParams p, TimedRep* out) {
  if (threadIdx.x != 0) return;
  const uint64_t deadline = globaltimer() + p.timeout_ns;
  for (uint32_t r = 0; r < p.n_rounds; ++r) {
    const PingPongRound& R = p.round[r];
    if (R.remote == nullptr) continue;
    TimedRep* o = out + (size_t)r * kRepSlots;
    // Leg 1's first ping goes into the line that carried leg 0's echoes, so it must not be stored before leg 0's
    // last echo has been read: leg 0's initiator hands the pair over with this word, which leg 1's initiator awaits.
    // Its echo bit is 0, so it lies above every leg-0 ping and below every leg-1 echo of its sender.
    const uint64_t handover = pingpong_word(p.call_seq, r, 1, 0, 0, 0);
    bool ok = true, initiated = false;
    for (uint32_t leg = 0; leg < 2 && ok; ++leg) {
      if ((leg == 0) == (R.first != 0)) {
        bool handover_bad = false;
        if (leg == 1) {
          uint64_t v;
          if (!poll(R.local, handover, deadline, v)) {
            ok = false;
            break;
          }
          handover_bad = v != handover;
        }
        ok = initiate<kFenced>(p, R, r, leg, deadline, o);
        initiated = true;
        if (ok && handover_bad) o[0].status = CDPROBE_ERR_INTEGRITY;
        if (ok && leg == 0) signal<kFenced>(R.remote, handover);
      } else {
        ok = respond<kFenced>(p, R, r, leg, deadline);
      }
    }
    if (ok) continue;
    // timed out: every cell this rank has not initiated yet is marked, and the kernel exits
    for (uint32_t q = initiated ? r + 1 : r; q < p.n_rounds; ++q) {
      if (p.round[q].remote == nullptr) continue;
      TimedRep& first = out[(size_t)q * kRepSlots];
      first.ns = 0;
      first.digest = 0;
      first.status = CDPROBE_ERR_TIMEOUT;
    }
    return;
  }
}

}  // namespace

int pingpong_launch(const PingPongParams& p, bool fenced, TimedRep* out, cudaStream_t stream) {
  if (fenced) pingpong_kernel<true><<<1, 32, 0, stream>>>(p, out);
  else pingpong_kernel<false><<<1, 32, 0, stream>>>(p, out);
  return (int)cudaGetLastError();
}

}  // namespace cdp
