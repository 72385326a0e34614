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
//
// The data path of K1, K2 and K4 lives in datapath.cuh, which the persistent kernels of the on-demand measurements
// include too.
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

#include "datapath.cuh"
#include "probe_launch.h"
#include "probe_types.h"

namespace cdp {
namespace {

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

// ----------------------------------------------------------- launchers -----
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

}  // namespace cdp
