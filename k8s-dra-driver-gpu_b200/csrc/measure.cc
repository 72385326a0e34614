// measure.cc — the on-demand measurements behind the C ABI: cdprobe_diagnose, cdprobe_latency, cdprobe_pingpong,
// cdprobe_atomics, cdprobe_bwcurve and cdprobe_allreduce.  Each runs on the local ranks' own streams, between probe
// runs, and has its results on the host before it returns.
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "allreduce.h"
#include "atomics.h"
#include "bwcurve.h"
#include "diagnose.h"
#include "handle.h"
#include "latency.h"
#include "pingpong.h"

namespace cdp {

// Grows local rank L's scratch to at least `bytes`, on its device (the caller has selected it); the old buffer is freed
// first.  The measurements share it: each runs on L's one stream, copies its results out before it returns, and reads
// back only what its own kernels wrote in the same call.  diag_launch clears its DiagOut and the compare pass writes
// every granule count; a rep table is read up to its first TIMEOUT slot, and the kernels write one for every cell they
// leave unfinished.
static int ensure_scratch(LocalRank& L, size_t bytes) {
  if (L.scratch_bytes >= bytes) return CDPROBE_OK;
  if (L.scratch) cudaFree(L.scratch);
  L.scratch = nullptr;
  L.scratch_bytes = 0;
  CDP_RT(cudaMalloc(&L.scratch, bytes));
  L.scratch_bytes = bytes;
  return CDPROBE_OK;
}

// Grows every local rank's scratch to hold its rep tables before any kernel is launched.  cudaFree synchronizes the
// device, and local ranks may share one: a pingpong kernel launched for an earlier rank would wait on this rank's.
static int ensure_rep_tables(cdprobe* h) {
  for (uint32_t li = 0; li < h->n_local; ++li) {
    CDP_RT(cudaSetDevice(h->lr[li].ordinal));
    const int rc = ensure_scratch(h->lr[li], sizeof(TimedRep) * kMaxRanks * kRepSlots);
    if (rc != CDPROBE_OK) return rc;
  }
  return CDPROBE_OK;
}

// Copies the first `bytes` of local rank L's scratch (its rep tables) to `got` once its kernel is done.
static int fetch_reps(cdprobe* h, LocalRank& L, size_t bytes, void* got, const char* what) {
  cudaError_t e = cudaSetDevice(L.ordinal);
  if (e == cudaSuccess) e = cudaMemcpyAsync(got, L.scratch, bytes, cudaMemcpyDeviceToHost, L.stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(L.stream);
  if (e != cudaSuccess) {
    h->sticky = true;  // a failed kernel leaves the context unusable
    return fail_cuda(what, e);
  }
  return CDPROBE_OK;
}

// Fills cell idx of a cdprobe_latency_t, cdprobe_pingpong_t or cdprobe_atomics_t from its rep table: the warm-up rep,
// then `reps` timed reps of `per_rep` hops, round trips or atomics each.  The digest covers every rep that ran; a CDPROBE_ERR_TIMEOUT rep ends the
// cell, which then has no times.  Any other non-zero rep status is kept, and a digest other than `want` makes the cell
// CDPROBE_ERR_INTEGRITY.  The latency kernel writes only 0 or CDPROBE_ERR_TIMEOUT, so for latency this is the rule
// "stop at the first non-zero status".
template <typename Out>
static void summarize(const TimedRep* rep, uint32_t reps, uint32_t per_rep, uint64_t want, uint32_t idx, Out* out) {
  uint64_t digest = 0;
  int32_t s = 0;
  float ns[kMaxTimedReps];
  for (uint32_t k = 0; k <= reps; ++k) {
    digest ^= rep[k].digest;
    if (rep[k].status == CDPROBE_ERR_TIMEOUT) {
      s = CDPROBE_ERR_TIMEOUT;
      break;
    }
    if (rep[k].status != 0) s = rep[k].status;
    if (k > 0) ns[k - 1] = (float)((double)rep[k].ns / per_rep);
  }
  out->measured[idx] = 1;
  out->digest[idx] = digest;
  if (s != CDPROBE_ERR_TIMEOUT) {
    std::sort(ns, ns + reps);
    out->ns_min[idx] = ns[0];
    out->ns_median[idx] = ns[reps / 2];
    out->ns_max[idx] = ns[reps - 1];
    if (digest != want) s = CDPROBE_ERR_INTEGRITY;
  }
  out->status[idx] = s;
}

// Fills entry idx of a cdprobe_bwcurve_t (a cell) or a cdprobe_allreduce_t (a row) from the records bwcurve_kernel or
// allreduce_kernel left in `s`: per size, ns of the timed reps and the (S, X) of the last one, every rep's (S, X)
// compared with want[k] (bad_sizes), and the model-free summary of the medians.  An entry whose kernel was aborted at
// the deadline has no times.
template <typename Out>
static void bw_summarize(const BwScratch& s, const uint64_t (*want)[2], const uint64_t* size, uint32_t n_sizes,
                         uint32_t reps, uint32_t idx, Out* out) {
  out->measured[idx] = 1;
  if (s.abort_flag != 0) {
    out->status[idx] = CDPROBE_ERR_TIMEOUT;
    return;
  }
  uint32_t bad = 0;
  double rate[kBwMaxSizes], peak = 0.0;
  for (uint32_t k = 0; k < n_sizes; ++k) {
    float ns[kMaxTimedReps];
    for (uint32_t r = 0; r <= reps; ++r) {
      const Acc& a = s.rep[k][r];
      if (a.sum != want[k][0] || a.xr != want[k][1]) bad |= 1u << k;
      if (r > 0) ns[r - 1] = (float)(a.t_end - s.t_rel[k][r]);
    }
    std::sort(ns, ns + reps);
    out->ns_min[idx][k] = ns[0];
    out->ns_median[idx][k] = ns[reps / 2];
    out->ns_max[idx][k] = ns[reps - 1];
    out->sum[idx][k] = s.rep[k][reps].sum;
    out->xr[idx][k] = s.rep[k][reps].xr;
    rate[k] = ns[reps / 2] > 0.f ? (double)size[k] / (double)ns[reps / 2] : 0.0;
    peak = std::max(peak, rate[k]);
  }
  out->t0_ns[idx] = out->ns_median[idx][0];
  out->peak_gbps[idx] = (float)peak;
  for (uint32_t k = 0; k < n_sizes; ++k) {
    if (rate[k] >= peak / 2) {
      out->half_bytes[idx] = size[k];
      break;
    }
  }
  out->bad_sizes[idx] = bad;
  out->status[idx] = bad ? CDPROBE_ERR_INTEGRITY : 0;
}

}  // namespace cdp

extern "C" {

static_assert(CDPROBE_DIAG_FLIP == cdp::kDiagFlip && CDPROBE_DIAG_ZERO == cdp::kDiagZero &&
                  CDPROBE_DIAG_DISPLACED == cdp::kDiagDisplaced && CDPROBE_DIAG_STALE == cdp::kDiagStale &&
                  CDPROBE_DIAG_FOREIGN == cdp::kDiagForeign && CDPROBE_DIAG_SAMPLES == cdp::kDiagSamples,
              "diagnosis classes");
static_assert(sizeof(cdp::DiagSample) == sizeof(cdprobe_diag_sample_t) &&
                  offsetof(cdp::DiagSample, run_seq) == offsetof(cdprobe_diag_sample_t, run_seq) &&
                  offsetof(cdp::DiagSample, rank) == offsetof(cdprobe_diag_sample_t, rank),
              "the kernel writes samples in the ABI layout");

int cdprobe_diagnose(cdprobe_t* h, uint32_t op, uint32_t issuer, uint32_t target, uint32_t reader, cdprobe_diag_t* out) {
  cdp::g_last_error.clear();
  if (h == nullptr || out == nullptr) return CDPROBE_ERR_ARG;
  // like cdprobe_run: the caller may read *out whatever the return code
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  out->op = op;
  out->issuer = issuer;
  out->target = target;
  out->reader = reader;
  out->first_bad = UINT64_MAX;
  const cdp::Plan& pl = h->plan;
  if (op != CDPROBE_OP_READ && op != CDPROBE_OP_WRITE) {
    cdp::set_err("op must be CDPROBE_OP_READ or CDPROBE_OP_WRITE");
    return CDPROBE_ERR_ARG;
  }
  if (issuer >= h->n_total || target >= h->n_total || reader >= h->n_total) {
    cdp::set_err("rank out of range");
    return CDPROBE_ERR_ARG;
  }
  if (issuer == target && !pl.diag) {
    cdp::set_err("cell (i, i) exists only with a loop-back slot (n == 1 or CDPROBE_FLAG_LOCAL_DIAG)");
    return CDPROBE_ERR_ARG;
  }
  if (reader < h->first || reader >= h->first + h->n_local) {
    cdp::set_err("reader is not a rank of this process");
    return CDPROBE_ERR_ARG;
  }
  if (const int rc = cdp::require_usable(h); rc != CDPROBE_OK) return rc;
  if (h->last_run_seq == 0) {
    cdp::set_err("no cdprobe_run yet: there is no pattern to compare with");
    return CDPROBE_ERR_STATE;
  }
  cdp::LocalRank& L = h->lr[reader - h->first];
  if (cdp::cell_status(h, reader - h->first, target) != 0) {  // never read through a mapping that is down
    cdp::set_err("reader does not map the target");
    return CDPROBE_ERR_STATE;
  }
  const uint64_t run_seq = h->last_run_seq;
  out->run_seq = run_seq;
  out->region_offset = cdp::cell_offset(pl, op, issuer, target);
  out->bytes = pl.bpp;

  const cdp::DiagSpec s =
      op == CDPROBE_OP_WRITE
          ? cdp::diag_write_spec(h->seed, h->n_total, issuer, target, run_seq, pl.bpp / 8)
          : cdp::diag_read_spec(h->seed, h->n_total, target, (uint64_t)cdp::cell_slice(pl, issuer, target) * (pl.bpp / 8),
                                pl.bpp / 8, pl.src_bytes / 8);

  CDP_RT(cudaSetDevice(L.ordinal));
  if (const int rc = cdp::ensure_scratch(L, cdp::diag_scratch_bytes(pl.bpp)); rc != CDPROBE_OK) return rc;
  const uint8_t* region = reinterpret_cast<const uint8_t*>(L.va[target]) + out->region_offset;
  cdp::DiagOut d;
  float ms = 0.f;
  cudaError_t e = cudaEventRecord(L.ev0, L.stream);
  if (e == cudaSuccess) e = (cudaError_t)cdp::diag_launch(region, s, L.scratch, L.sm_count, L.stream);
  if (e == cudaSuccess) e = cudaEventRecord(L.ev1, L.stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&d, L.scratch, sizeof(d), cudaMemcpyDeviceToHost, L.stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(L.stream);
  if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, L.ev0, L.ev1);
  if (e != cudaSuccess) {
    h->sticky = true;  // a failed kernel leaves the context unusable
    return cdp::fail_cuda("cdprobe_diagnose", e);
  }
  out->ms = ms;
  out->bad_words = d.bad_words;
  out->bad_granules = d.bad_granules;
  out->zero_words = d.kind_count[cdp::kDiagZero];
  if (d.bad_words) {
    out->first_bad = ~d.first_bad_n;
    out->last_bad = d.last_bad;
  }
  for (int k = 0; k < cdp::kDiagKinds; ++k) out->kind_count[k] = d.kind_count[k];
  for (int b = 0; b < 64; ++b) out->bit_flips[b] = d.bit_flips[b];
  out->n_samples = d.bad_words < (uint64_t)CDPROBE_DIAG_SAMPLES ? (uint32_t)d.bad_words : (uint32_t)CDPROBE_DIAG_SAMPLES;
  memcpy(out->sample, d.sample, sizeof(out->sample[0]) * out->n_samples);
  return CDPROBE_OK;
}

int cdprobe_latency(cdprobe_t* h, uint32_t hops, uint32_t reps, cdprobe_latency_t* out) {
  cdp::g_last_error.clear();
  if (out == nullptr) return CDPROBE_ERR_ARG;
  // like cdprobe_run: the caller may read *out whatever the return code
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  out->hops = hops != 0 ? hops : cdp::kLatencyDefaultHops;
  out->reps = reps != 0 ? reps : cdp::kLatencyDefaultReps;
  if (h == nullptr) return CDPROBE_ERR_ARG;
  const double t_begin = cdp::now_ms();
  const cdp::Plan& pl = h->plan;
  out->n = h->n_total;
  out->region_bytes = pl.bpp;
  if (out->hops > cdp::kLatencyMaxHops || out->reps > cdp::kMaxTimedReps) {
    cdp::set_err("hops must be at most 1 << 20 and reps at most 64");
    return CDPROBE_ERR_ARG;
  }
  if (const int rc = cdp::require_usable(h); rc != CDPROBE_OK) return rc;
  hops = out->hops;
  reps = out->reps;
  const uint64_t lines = pl.bpp / (cdp::kLineWords * 8);
  if (const int rc = cdp::ensure_rep_tables(h); rc != CDPROBE_OK) return rc;

  // 1. every local issuer's chases, all launched before any is waited for
  cdp::LatencyParams P[cdp::kMaxRanks];
  for (uint32_t li = 0; li < h->n_local; ++li) {
    cdp::LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    out->row_mask |= 1u << g;
    cdp::LatencyParams& p = P[li];
    memset(&p, 0, sizeof(p));
    p.seed = h->seed;
    p.timeout_ns = (uint64_t)h->cfg.timeout_ms * 1000000ull;
    p.hops = hops;
    p.reps = reps;
    for (uint32_t j = 0; j < h->n_total; ++j) {
      if (j == g && !pl.diag) continue;  // no loop-back slice to chase
      const int32_t s = cdp::cell_status(h, li, j);
      if (s != 0) {  // never read through a mapping that is down
        out->status[g * CDPROBE_MAX_GPUS + j] = s;
        continue;
      }
      cdp::LatencyCell& c = p.cell[p.n_cells++];
      c.region = reinterpret_cast<const uint8_t*>(L.va[j]) + cdp::cell_offset(pl, CDPROBE_OP_READ, g, j);
      c.lines = lines;
      c.issuer = g;
      c.target = j;
    }
    if (p.n_cells == 0) continue;
    CDP_RT(cudaSetDevice(L.ordinal));
    const cudaError_t e = (cudaError_t)cdp::latency_launch(p, static_cast<cdp::TimedRep*>(L.scratch), L.stream);
    if (e != cudaSuccess) {
      h->sticky = true;
      return cdp::fail_cuda("launch latency_kernel", e);
    }
  }

  // 2. while they run: the digest each chase gives over an intact region
  uint64_t want[cdp::kMaxRanks][cdp::kMaxRanks] = {};
  for (uint32_t li = 0; li < h->n_local; ++li) {
    for (uint32_t k = 0; k < P[li].n_cells; ++k) {
      const cdp::LatencyCell& c = P[li].cell[k];
      const uint64_t first = (uint64_t)cdp::cell_slice(pl, c.issuer, c.target) * (pl.bpp / 8);
      for (uint32_t r = 0; r <= reps; ++r)
        want[li][k] ^= cdp::latency_rep_digest(h->seed, c.issuer, c.target, first, lines, r, hops);
    }
  }

  // 3. collect: ns per hop of the timed reps, the digest of all of them
  std::vector<cdp::TimedRep> got((size_t)cdp::kMaxRanks * cdp::kRepSlots);
  for (uint32_t li = 0; li < h->n_local; ++li) {
    const cdp::LatencyParams& p = P[li];
    if (p.n_cells == 0) continue;
    const size_t bytes = sizeof(cdp::TimedRep) * p.n_cells * cdp::kRepSlots;
    if (const int rc = cdp::fetch_reps(h, h->lr[li], bytes, got.data(), "cdprobe_latency"); rc != CDPROBE_OK) return rc;
    for (uint32_t k = 0; k < p.n_cells; ++k)
      cdp::summarize(got.data() + (size_t)k * cdp::kRepSlots, reps, hops, want[li][k],
                     p.cell[k].issuer * CDPROBE_MAX_GPUS + p.cell[k].target, out);
  }
  out->ms = cdp::now_ms() - t_begin;
  return CDPROBE_OK;
}

// What each process contributes at the start of cdprobe_pingpong, so that every process refuses or runs the same call
// over the same pair set (cdprobe_unmap_peer changes only the local view).
struct PingPongAgree {
  uint64_t call_seq;
  uint32_t trips, reps, fenced, ok;
  int32_t status[cdp::kMaxRanks][cdp::kMaxRanks];  // [local rank][rank]: mapping status, unmapped cells folded in
};

int cdprobe_pingpong(cdprobe_t* h, uint32_t trips, uint32_t reps, uint32_t fenced, cdprobe_pingpong_t* out) {
  cdp::g_last_error.clear();
  if (out == nullptr) return CDPROBE_ERR_ARG;
  // like cdprobe_run: the caller may read *out whatever the return code
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  out->trips = trips != 0 ? trips : cdp::kPingPongDefaultTrips;
  out->reps = reps != 0 ? reps : cdp::kPingPongDefaultReps;
  out->fenced = fenced;
  if (h == nullptr) return CDPROBE_ERR_ARG;
  const double t_begin = cdp::now_ms();
  const cdp::Plan& pl = h->plan;
  const uint32_t n = h->n_total;
  out->n = n;
  trips = out->trips;
  reps = out->reps;
  if (const int rc = cdp::require_usable(h); rc != CDPROBE_OK) return rc;
  // 1. the arguments; in a multi-process domain the verdict is shared below, so every process refuses together
  std::string bad;
  if (trips > cdp::kPingPongMaxTrips || reps > cdp::kMaxTimedReps || fenced > 1)
    bad = "trips must be at most 1 << 16, reps at most 64 and fenced 0 or 1";
  uint32_t f_init = cdp::kPingPongNoFault, f_target = cdp::kPingPongNoFault, f_trip = cdp::kPingPongNoFault;
  if (h->pp_fault != 0) {
    const uint64_t fi = h->pp_fault >> 32, ft = (h->pp_fault >> 16) & 0xffffu, trip = h->pp_fault & 0xffffu;
    if (fi == 0 || ft == 0 || fi > n || ft > n || fi == ft) {
      bad = "the armed pingpong fault names no off-diagonal cell";
    } else if (trip + 1 >= trips || (reps == 1 && trip + 2 == trips)) {
      // the initiator runs one trip ahead until the responder catches up; that must happen inside the leg
      bad = "the armed pingpong fault's trip must be below trips - 1, and below trips - 2 when reps is 1";
    } else {
      f_init = (uint32_t)fi - 1;
      f_target = (uint32_t)ft - 1;
      f_trip = (uint32_t)trip;
    }
  }
  PingPongAgree mine;
  memset(&mine, 0, sizeof(mine));
  mine.call_seq = h->pp_calls + 1;
  mine.trips = trips;
  mine.reps = reps;
  mine.fenced = fenced;
  mine.ok = bad.empty() ? 1u : 0u;
  int32_t st[cdp::kMaxRanks][cdp::kMaxRanks];
  memcpy(st, h->status, sizeof(st));
  for (uint32_t li = 0; li < h->n_local; ++li) {
    const cdp::LocalRank& L = h->lr[li];
    for (uint32_t j = 0; j < n; ++j) st[L.grank][j] = mine.status[li][j] = cdp::cell_status(h, li, j);
  }
  if (h->cfg.world_size > 1) {
    std::vector<PingPongAgree> all(h->cfg.world_size);
    std::string err;
    if (h->rdv.allgather(&mine, sizeof(mine), all.data(), &err) != 0) {
      cdp::set_err(err);
      return CDPROBE_ERR_RENDEZVOUS;
    }
    for (uint32_t r = 0; r < h->cfg.world_size; ++r) {
      const PingPongAgree& o = all[r];
      if (!o.ok && bad.empty()) bad = "another process called cdprobe_pingpong with invalid arguments";
      if ((o.call_seq != mine.call_seq || o.trips != trips || o.reps != reps || o.fenced != fenced) && bad.empty())
        bad = "cdprobe_pingpong is collective: every process must call it with the same arguments";
      for (uint32_t li = 0; li < h->n_local; ++li) memcpy(st[r * h->n_local + li], o.status[li], sizeof(st[0]));
    }
  }
  if (!bad.empty()) {
    cdp::set_err(bad);
    return CDPROBE_ERR_ARG;
  }
  h->pp_calls = mine.call_seq;
  out->call_seq = h->pp_calls;
  for (uint32_t li = 0; li < h->n_local; ++li) out->row_mask |= 1u << h->lr[li].grank;
  if (n == 1) {
    out->ms = cdp::now_ms() - t_begin;
    return CDPROBE_OK;
  }
  if (h->cfg.world_size > 1) {  // every process has agreed before any kernel polls a peer
    std::string err;
    if (h->rdv.barrier(&err) != 0) {
      cdp::set_err(err);
      return CDPROBE_ERR_RENDEZVOUS;
    }
  }
  if (const int rc = cdp::ensure_rep_tables(h); rc != CDPROBE_OK) return rc;
  // a pair is exchanged only when both directions are mapped; the status of its cells is the pair's mapping status
  auto pair_status = [&](uint32_t i, uint32_t j) { return st[i][j] != 0 ? st[i][j] : st[j][i]; };

  // 2. one block per local rank, every one launched before any is waited for
  cdp::PingPongParams P[cdp::kMaxRanks];
  bool launched[cdp::kMaxRanks] = {};
  for (uint32_t li = 0; li < h->n_local; ++li) {
    cdp::LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    cdp::PingPongParams& p = P[li];
    memset(&p, 0, sizeof(p));
    p.call_seq = h->pp_calls;
    p.timeout_ns = (uint64_t)h->cfg.timeout_ms * 1000000ull;
    p.n_rounds = pl.rounds;
    p.trips = trips;
    p.reps = reps;
    p.fault_round = cdp::kPingPongNoFault;
    p.fault_trip = f_trip;
    for (uint32_t j = 0; j < n; ++j)
      if (j != g) out->status[g * CDPROBE_MAX_GPUS + j] = pair_status(g, j);
    uint32_t active = 0;
    for (uint32_t r = 0; r < pl.rounds; ++r) {
      const int q = pl.partner[r][g];
      if (q < 0 || pair_status(g, (uint32_t)q) != 0) continue;
      cdp::PingPongRound& R = p.round[r];
      R.remote = reinterpret_cast<uint64_t*>(L.va[q] + cdp::kPingOff + (uint64_t)g * sizeof(cdp::FlagLine));
      R.local = reinterpret_cast<const uint64_t*>(L.va[g] + cdp::kPingOff + (uint64_t)q * sizeof(cdp::FlagLine));
      R.partner = (uint32_t)q;
      R.first = g < (uint32_t)q ? 1u : 0u;
      if (g == f_target && (uint32_t)q == f_init) p.fault_round = r;
      ++active;
    }
    if (active == 0) continue;
    CDP_RT(cudaSetDevice(L.ordinal));
    const cudaError_t e =
        (cudaError_t)cdp::pingpong_launch(p, fenced != 0, static_cast<cdp::TimedRep*>(L.scratch), L.stream);
    if (e != cudaSuccess) {
      h->sticky = true;
      return cdp::fail_cuda("launch pingpong_kernel", e);
    }
    launched[li] = true;
  }

  // 3. while they run: the digest of a clean leg for every cell a local rank initiates
  uint64_t want[cdp::kMaxRanks][cdp::kMaxRanks] = {};  // [local rank][round]
  for (uint32_t li = 0; li < h->n_local; ++li) {
    for (uint32_t r = 0; r < pl.rounds; ++r) {
      const cdp::PingPongRound& R = P[li].round[r];
      if (R.remote == nullptr) continue;
      const uint32_t leg = R.first ? 0u : 1u;
      for (uint32_t rep = 0; rep <= reps; ++rep) want[li][r] ^= cdp::pingpong_rep_digest(h->pp_calls, r, leg, rep, trips);
    }
  }

  // 4. collect: ns per round trip of the timed reps, the digest of all of them
  std::vector<cdp::TimedRep> got((size_t)cdp::kMaxRanks * cdp::kRepSlots);
  for (uint32_t li = 0; li < h->n_local; ++li) {
    if (!launched[li]) continue;
    const cdp::PingPongParams& p = P[li];
    const size_t bytes = sizeof(cdp::TimedRep) * p.n_rounds * cdp::kRepSlots;
    if (const int rc = cdp::fetch_reps(h, h->lr[li], bytes, got.data(), "cdprobe_pingpong"); rc != CDPROBE_OK) return rc;
    for (uint32_t r = 0; r < p.n_rounds; ++r) {
      const cdp::PingPongRound& R = p.round[r];
      if (R.remote == nullptr) continue;
      cdp::summarize(got.data() + (size_t)r * cdp::kRepSlots, reps, trips, want[li][r],
                     h->lr[li].grank * CDPROBE_MAX_GPUS + R.partner, out);
    }
  }
  out->ms = cdp::now_ms() - t_begin;
  return CDPROBE_OK;
}

int cdprobe_atomics(cdprobe_t* h, uint32_t kind, uint32_t ops, uint32_t reps, cdprobe_atomics_t* out) {
  cdp::g_last_error.clear();
  if (out == nullptr) return CDPROBE_ERR_ARG;
  // like cdprobe_run: the caller may read *out whatever the return code
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  out->kind = kind;
  out->ops = ops != 0 ? ops : cdp::kAtomicsDefaultOps;
  out->reps = reps != 0 ? reps : cdp::kAtomicsDefaultReps;
  out->lanes = kind == CDPROBE_ATOMIC_CONTENDED ? 32u : 1u;
  if (h == nullptr) return CDPROBE_ERR_ARG;
  const double t_begin = cdp::now_ms();
  const cdp::Plan& pl = h->plan;
  const uint32_t n = h->n_total;
  out->n = n;
  if (kind > CDPROBE_ATOMIC_CONTENDED || out->ops > cdp::kAtomicsMaxOps || out->reps > cdp::kMaxTimedReps) {
    cdp::set_err("kind must be a CDPROBE_ATOMIC_*, ops at most 1 << 16 and reps at most 64");
    return CDPROBE_ERR_ARG;
  }
  uint32_t f_issuer = cdp::kMaxRanks, f_target = cdp::kMaxRanks;
  if (h->at_fault != 0) {
    const uint64_t fi = h->at_fault >> 16, ft = h->at_fault & 0xffffu;
    if (fi == 0 || ft == 0 || fi > n || ft > n || (fi == ft && !pl.diag)) {
      cdp::set_err("the armed atomics fault names no cell of this domain");
      return CDPROBE_ERR_ARG;
    }
    f_issuer = (uint32_t)fi - 1;
    f_target = (uint32_t)ft - 1;
  }
  if (const int rc = cdp::require_usable(h); rc != CDPROBE_OK) return rc;
  ops = out->ops;
  reps = out->reps;
  const uint64_t total = (uint64_t)out->lanes * ops;  // increments per rep
  if (const int rc = cdp::ensure_rep_tables(h); rc != CDPROBE_OK) return rc;
  out->call_seq = ++h->at_calls;

  // 1. every local issuer's cells, all launched before any is waited for; no kernel waits on another rank
  cdp::AtomicsParams P[cdp::kMaxRanks];
  for (uint32_t li = 0; li < h->n_local; ++li) {
    cdp::LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    out->row_mask |= 1u << g;
    cdp::AtomicsParams& p = P[li];
    memset(&p, 0, sizeof(p));
    p.call_seq = h->at_calls;
    p.timeout_ns = (uint64_t)h->cfg.timeout_ms * 1000000ull;
    p.ops = ops;
    p.reps = reps;
    p.fault_cell = cdp::kAtomicsNoFault;
    for (uint32_t j = 0; j < n; ++j) {
      const uint32_t idx = g * CDPROBE_MAX_GPUS + j;
      // native atomics: a device is atomic with itself; a peer in another process has a device this one cannot see
      const cdp::LocalRank* peer = j >= h->first && j < h->first + h->n_local ? &h->lr[j - h->first] : nullptr;
      int native = 1;
      if (peer == nullptr) {
        native = 2;
      } else if (peer->ordinal != L.ordinal) {
        CDP_RT(cudaDeviceGetP2PAttribute(&native, cudaDevP2PAttrNativeAtomicSupported, L.ordinal, peer->ordinal));
        native = native != 0 ? 1 : 0;
      }
      out->native[idx] = (uint8_t)native;
      if (j == g && !pl.diag) continue;  // no loop-back slot
      const int32_t s = cdp::cell_status(h, li, j);
      if (s != 0) {  // never touch a mapping that is down
        out->status[idx] = s;
        continue;
      }
      if (native == 0) {
        out->status[idx] = CDPROBE_ERR_UNSUPPORTED;
        continue;
      }
      if (g == f_issuer && j == f_target) p.fault_cell = p.n_cells;
      cdp::AtomicsCell& c = p.cell[p.n_cells++];
      c.word = reinterpret_cast<unsigned long long*>(L.va[j] + cdp::kAtomOff + (uint64_t)g * sizeof(cdp::AtomLine));
      c.issuer = g;
      c.target = j;
    }
    if (p.n_cells == 0) continue;
    CDP_RT(cudaSetDevice(L.ordinal));
    const cudaError_t e = (cudaError_t)cdp::atomics_launch(p, kind, static_cast<cdp::TimedRep*>(L.scratch), L.stream);
    if (e != cudaSuccess) {
      h->sticky = true;
      return cdp::fail_cuda("launch atomics kernel", e);
    }
  }

  // 2. while they run: the digest of clean reps, the same for every cell
  uint64_t want = 0;
  for (uint32_t r = 0; r <= reps; ++r) want ^= cdp::atomics_rep_digest(cdp::atomics_start(h->at_calls, kind, r), total);

  // 3. collect: ns per atomic of the timed reps, the digest of all of them
  std::vector<cdp::TimedRep> got((size_t)cdp::kMaxRanks * cdp::kRepSlots);
  for (uint32_t li = 0; li < h->n_local; ++li) {
    const cdp::AtomicsParams& p = P[li];
    if (p.n_cells == 0) continue;
    const size_t bytes = sizeof(cdp::TimedRep) * p.n_cells * cdp::kRepSlots;
    if (const int rc = cdp::fetch_reps(h, h->lr[li], bytes, got.data(), "cdprobe_atomics"); rc != CDPROBE_OK) return rc;
    for (uint32_t k = 0; k < p.n_cells; ++k)
      cdp::summarize(got.data() + (size_t)k * cdp::kRepSlots, reps, (uint32_t)total, want,
                     p.cell[k].issuer * CDPROBE_MAX_GPUS + p.cell[k].target, out);
  }
  out->ms = cdp::now_ms() - t_begin;
  return CDPROBE_OK;
}

// What each process contributes at the start of cdprobe_bwcurve, so that every process refuses or runs the same call.
// Every cell is one-sided and the rounds come from the plan, which all processes share, so nothing else must agree.
struct BwCurveAgree {
  uint64_t call_seq;
  uint32_t reps, ok;
};

int cdprobe_bwcurve(cdprobe_t* h, uint32_t reps, cdprobe_bwcurve_t* out) {
  cdp::g_last_error.clear();
  if (out == nullptr) return CDPROBE_ERR_ARG;
  // like cdprobe_run: the caller may read *out whatever the return code
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  out->reps = reps != 0 ? reps : cdp::kBwDefaultReps;
  if (h == nullptr) return CDPROBE_ERR_ARG;
  const double t_begin = cdp::now_ms();
  const cdp::Plan& pl = h->plan;
  const uint32_t n = h->n_total;
  out->n = n;
  out->path = h->path;
  reps = out->reps;
  if (const int rc = cdp::require_usable(h); rc != CDPROBE_OK) return rc;
  // 1. the arguments; in a multi-process domain the verdict is shared below, so every process refuses together
  std::string bad;
  uint64_t size[cdp::kBwMaxSizes];
  const uint32_t n_sizes = cdp::bwcurve_ladder(pl.bpp, size);
  if (reps > cdp::kMaxTimedReps) bad = "reps must be at most 64";
  else if (n_sizes == 0) bad = "bytes_per_pair must be at most 32 GiB";
  BwCurveAgree mine = {h->bw_calls + 1, reps, bad.empty() ? 1u : 0u};
  if (h->cfg.world_size > 1) {
    std::vector<BwCurveAgree> all(h->cfg.world_size);
    std::string err;
    if (h->rdv.allgather(&mine, sizeof(mine), all.data(), &err) != 0) {
      cdp::set_err(err);
      return CDPROBE_ERR_RENDEZVOUS;
    }
    for (const BwCurveAgree& o : all) {
      if (!o.ok && bad.empty()) bad = "another process called cdprobe_bwcurve with invalid arguments";
      if ((o.call_seq != mine.call_seq || o.reps != reps) && bad.empty())
        bad = "cdprobe_bwcurve is collective: every process must call it with the same arguments";
    }
  }
  if (!bad.empty()) {
    cdp::set_err(bad);
    return CDPROBE_ERR_ARG;
  }
  h->bw_calls = mine.call_seq;
  out->call_seq = h->bw_calls;
  out->n_sizes = n_sizes;
  memcpy(out->size, size, sizeof(size[0]) * n_sizes);
  for (uint32_t li = 0; li < h->n_local; ++li) out->row_mask |= 1u << h->lr[li].grank;

  // 2. scratch for the rep records and one cell's granule table, grown on every local rank before any kernel runs
  const uint64_t granules = pl.bpp / cdp::kGranuleBytes;
  const size_t table_off = (sizeof(cdp::BwScratch) + 255) / 256 * 256;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    CDP_RT(cudaSetDevice(h->lr[li].ordinal));
    if (const int rc = cdp::ensure_scratch(h->lr[li], table_off + 16 * granules); rc != CDPROBE_OK) return rc;
  }

  // 3. the (S, X) each size of each cell that runs must read, from the pattern definition: the per-granule sums of the
  //    slice on the issuer's GPU, folded into every prefix on the host
  bool runs[cdp::kMaxRanks][cdp::kMaxRanks] = {};
  std::vector<uint64_t> want((size_t)cdp::kMaxRanks * cdp::kMaxRanks * cdp::kBwMaxSizes * 2);
  auto want_of = [&](uint32_t li, uint32_t j) {
    return reinterpret_cast<uint64_t(*)[2]>(want.data() + ((size_t)li * cdp::kMaxRanks + j) * cdp::kBwMaxSizes * 2);
  };
  std::vector<uint64_t> table(2 * granules);
  for (uint32_t li = 0; li < h->n_local; ++li) {
    cdp::LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    for (uint32_t j = 0; j < n; ++j) {
      if (j == g && !pl.diag) continue;  // no loop-back slice
      const int32_t s = cdp::cell_status(h, li, j);
      if (s != 0) {  // never read through a mapping that is down
        out->status[g * CDPROBE_MAX_GPUS + j] = s;
        continue;
      }
      runs[li][j] = true;
      const uint64_t first = (uint64_t)cdp::cell_slice(pl, g, j) * (pl.bpp / 8);
      uint64_t* gsum = reinterpret_cast<uint64_t*>(static_cast<uint8_t*>(L.scratch) + table_off);
      cudaError_t e = (cudaError_t)cdp::bwcurve_granules_launch(gsum, gsum + granules, h->seed, j, first, granules,
                                                                 (unsigned)L.sm_count * 8u, L.stream);
      if (e == cudaSuccess && granules)
        e = cudaMemcpyAsync(table.data(), gsum, 16 * granules, cudaMemcpyDeviceToHost, L.stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(L.stream);
      if (e != cudaSuccess) {
        h->sticky = true;
        return cdp::fail_cuda("cdprobe_bwcurve: granule checksums", e);
      }
      uint64_t(*w)[2] = want_of(li, j);
      for (uint32_t k = 0; k < n_sizes; ++k)
        cdp::bwcurve_prefix_checksum(table.data(), table.data() + granules, h->seed, j, first, size[k] / 8, &w[k][0],
                                     &w[k][1]);
    }
  }

  // 4. the rounds: the tournament's, then the loop-back; every local kernel of a round is launched before any is
  //    waited for, and no process starts a round before every process has finished the one before
  const bool coop_ok = !(h->cfg.flags & CDPROBE_FLAG_NO_COOPERATIVE);
  std::vector<cdp::BwScratch> got(1);
  const uint32_t n_rounds = pl.rounds + (pl.diag ? 1u : 0u);
  for (uint32_t r = 0; r < n_rounds; ++r) {
    if (h->cfg.world_size > 1) {
      std::string err;
      if (h->rdv.barrier(&err) != 0) {
        cdp::set_err(err);
        return CDPROBE_ERR_RENDEZVOUS;
      }
    }
    int32_t target[cdp::kMaxRanks];
    for (uint32_t li = 0; li < h->n_local; ++li) {
      cdp::LocalRank& L = h->lr[li];
      const int q = r < pl.rounds ? pl.partner[r][L.grank] : (int)L.grank;
      target[li] = q >= 0 && runs[li][q] ? q : -1;
      if (target[li] < 0) continue;
      cdp::BwCurveParams p;
      memset(&p, 0, sizeof(p));
      p.region = reinterpret_cast<const uint8_t*>(L.va[q]) + cdp::cell_offset(pl, CDPROBE_OP_READ, L.grank, (uint32_t)q);
      p.scratch = static_cast<cdp::BwScratch*>(L.scratch);
      memcpy(p.size, size, sizeof(size));
      p.timeout_ns = (uint64_t)h->cfg.timeout_ms * 1000000ull;
      p.n_sizes = n_sizes;
      p.reps = reps;
      p.path = h->path;
      CDP_RT(cudaSetDevice(L.ordinal));
      cudaError_t e = cudaMemsetAsync(L.scratch, 0, sizeof(cdp::BwScratch), L.stream);
      if (e == cudaSuccess) e = (cudaError_t)cdp::bwcurve_launch(p, L.ctas, L.coop && coop_ok, L.stream);
      if (e != cudaSuccess) {
        h->sticky = true;
        return cdp::fail_cuda("launch bwcurve_kernel", e);
      }
    }
    for (uint32_t li = 0; li < h->n_local; ++li) {
      if (target[li] < 0) continue;
      cdp::LocalRank& L = h->lr[li];
      if (const int rc = cdp::fetch_reps(h, L, sizeof(cdp::BwScratch), got.data(), "cdprobe_bwcurve"); rc != CDPROBE_OK)
        return rc;
      cdp::bw_summarize(got[0], want_of(li, (uint32_t)target[li]), size, n_sizes, reps,
                        L.grank * CDPROBE_MAX_GPUS + (uint32_t)target[li], out);
    }
  }
  out->ms = cdp::now_ms() - t_begin;
  return CDPROBE_OK;
}

// What each process contributes at the start of cdprobe_allreduce, so that every process refuses, skips or runs the
// same call.  The mapping verdict must agree too: a process that ran while another skipped would wait at the first
// domain barrier until its watchdog fired.
struct AllReduceAgree {
  uint64_t call_seq;
  uint32_t reps, ok;
  uint32_t down_cell;    // issuer * kMaxRanks + target of this process's first cell whose mapping is down (kNoCell: none)
  int32_t down_status;   // that cell's mapping status
};
static constexpr uint32_t kNoCell = ~0u;

int cdprobe_allreduce(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out) {
  cdp::g_last_error.clear();
  if (out == nullptr) return CDPROBE_ERR_ARG;
  // like cdprobe_run: the caller may read *out whatever the return code
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  out->reps = reps != 0 ? reps : cdp::kArDefaultReps;
  if (h == nullptr) return CDPROBE_ERR_ARG;
  const double t_begin = cdp::now_ms();
  const cdp::Plan& pl = h->plan;
  const uint32_t n = h->n_total;
  out->n = n;
  out->path = h->path;
  reps = out->reps;
  if (const int rc = cdp::require_usable(h); rc != CDPROBE_OK) return rc;
  // 1. the arguments, the armed fault and the mapping verdict; in a multi-process domain all three are shared below,
  //    so every process refuses, skips or runs together
  std::string bad;
  uint64_t size[cdp::kBwMaxSizes];
  const uint32_t n_sizes = cdp::bwcurve_ladder(pl.bpp, size);
  if (reps > cdp::kMaxTimedReps) bad = "reps must be at most 64";
  else if (n_sizes == 0) bad = "bytes_per_pair must be at most 32 GiB";
  uint32_t f_rank = cdp::kArNoFault, f_k = cdp::kArNoFault;
  uint64_t f_word = 0;
  if (h->ar_fault != 0 && bad.empty()) {
    const uint64_t fr = h->ar_fault >> 32, fk = (h->ar_fault >> 24) & 0xffu;
    f_word = h->ar_fault & 0xffffffu;
    if (fr == 0 || fr > n || fk == 0 || fk > n_sizes || f_word >= size[fk - 1] / 8) {
      bad = "the armed all-reduce fault names no rank, size or output word of this call";
    } else {
      f_rank = (uint32_t)fr - 1;
      f_k = (uint32_t)fk - 1;
    }
  }
  AllReduceAgree mine;
  memset(&mine, 0, sizeof(mine));
  mine.call_seq = h->ar_calls + 1;
  mine.reps = reps;
  mine.ok = bad.empty() ? 1u : 0u;
  mine.down_cell = kNoCell;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    for (uint32_t j = 0; j < n; ++j) {
      const int32_t s = cdp::cell_status(h, li, j);
      const uint32_t cell = h->lr[li].grank * cdp::kMaxRanks + j;
      if (s != 0 && cell < mine.down_cell) {
        mine.down_cell = cell;
        mine.down_status = s;
      }
    }
  }
  AllReduceAgree down = mine;
  if (h->cfg.world_size > 1) {
    std::vector<AllReduceAgree> all(h->cfg.world_size);
    std::string err;
    if (h->rdv.allgather(&mine, sizeof(mine), all.data(), &err) != 0) {
      cdp::set_err(err);
      return CDPROBE_ERR_RENDEZVOUS;
    }
    for (const AllReduceAgree& o : all) {
      if (!o.ok && bad.empty()) bad = "another process called cdprobe_allreduce with invalid arguments";
      if ((o.call_seq != mine.call_seq || o.reps != reps) && bad.empty())
        bad = "cdprobe_allreduce is collective: every process must call it with the same arguments";
      if (o.down_cell < down.down_cell) down = o;
    }
  }
  if (!bad.empty()) {
    cdp::set_err(bad);
    return CDPROBE_ERR_ARG;
  }
  h->ar_calls = mine.call_seq;
  out->call_seq = h->ar_calls;
  out->n_sizes = n_sizes;
  memcpy(out->size, size, sizeof(size[0]) * n_sizes);
  for (uint32_t li = 0; li < h->n_local; ++li) out->row_mask |= 1u << h->lr[li].grank;
  if (down.down_cell != kNoCell) {  // some rank cannot read some input: nothing runs, in any process
    for (uint32_t li = 0; li < h->n_local; ++li) out->status[h->lr[li].grank] = down.down_status;
    out->ms = cdp::now_ms() - t_begin;
    return CDPROBE_OK;
  }

  // 2. scratch for the records, the output and the granule table, grown on every local rank before any kernel runs
  const uint64_t granules = pl.bpp / cdp::kGranuleBytes;
  const size_t table_off = cdp::kArOutOff + (pl.bpp + 255) / 256 * 256;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    CDP_RT(cudaSetDevice(h->lr[li].ordinal));
    if (const int rc = cdp::ensure_scratch(h->lr[li], table_off + 16 * granules); rc != CDPROBE_OK) return rc;
  }

  // 3. the (S, X) every prefix of the output must have, from the pattern definition: the per-granule sums of the
  //    summed words on the first local rank's GPU, folded into every prefix on the host
  uint64_t want[cdp::kBwMaxSizes][2] = {};
  {
    cdp::LocalRank& L = h->lr[0];
    std::vector<uint64_t> table(2 * granules);
    uint64_t* gsum = reinterpret_cast<uint64_t*>(static_cast<uint8_t*>(L.scratch) + table_off);
    CDP_RT(cudaSetDevice(L.ordinal));
    cudaError_t e = (cudaError_t)cdp::allreduce_granules_launch(gsum, gsum + granules, h->seed, n, granules,
                                                                 (unsigned)L.sm_count * 8u, L.stream);
    if (e == cudaSuccess && granules)
      e = cudaMemcpyAsync(table.data(), gsum, 16 * granules, cudaMemcpyDeviceToHost, L.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(L.stream);
    if (e != cudaSuccess) {
      h->sticky = true;
      return cdp::fail_cuda("cdprobe_allreduce: granule checksums", e);
    }
    for (uint32_t k = 0; k < n_sizes; ++k)
      cdp::allreduce_prefix_checksum(table.data(), table.data() + granules, h->seed, n, size[k] / 8, &want[k][0],
                                     &want[k][1]);
  }

  // 4. no process launches before every process is ready, so that no kernel waits at the first domain barrier for a
  //    process still setting up; then every local kernel is launched before any is waited for
  if (h->cfg.world_size > 1) {
    std::string err;
    if (h->rdv.barrier(&err) != 0) {
      cdp::set_err(err);
      return CDPROBE_ERR_RENDEZVOUS;
    }
  }
  const bool coop_ok = !(h->cfg.flags & CDPROBE_FLAG_NO_COOPERATIVE);
  for (uint32_t li = 0; li < h->n_local; ++li) {
    cdp::LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    cdp::AllReduceParams p;
    memset(&p, 0, sizeof(p));
    for (uint32_t t = 0; t < n; ++t) p.src[t] = reinterpret_cast<const uint8_t*>(L.va[(g + t) % n]) + pl.src_off;
    for (uint32_t j = 0; j < n; ++j)
      if (j != g) p.sig_out[j] = reinterpret_cast<uint64_t*>(L.va[j] + cdp::kArOff + (uint64_t)g * sizeof(cdp::FlagLine));
    p.sig_in = reinterpret_cast<const cdp::FlagLine*>(L.va[g] + cdp::kArOff);
    p.scratch = static_cast<cdp::ArScratch*>(L.scratch);
    p.out = static_cast<uint8_t*>(L.scratch) + cdp::kArOutOff;
    memcpy(p.size, size, sizeof(size));
    p.seed = h->seed;
    p.call_seq = h->ar_calls;
    p.timeout_ns = (uint64_t)h->cfg.timeout_ms * 1000000ull;
    p.fault_k = g == f_rank ? f_k : cdp::kArNoFault;
    p.fault_word = f_word;
    p.rank = g;
    p.n = n;
    p.n_sizes = n_sizes;
    p.reps = reps;
    p.path = h->path;
    CDP_RT(cudaSetDevice(L.ordinal));
    cudaError_t e = cudaMemsetAsync(L.scratch, 0, sizeof(cdp::ArScratch), L.stream);
    if (e == cudaSuccess) e = (cudaError_t)cdp::allreduce_launch(p, L.ctas, L.coop && coop_ok, L.stream);
    if (e != cudaSuccess) {
      h->sticky = true;
      return cdp::fail_cuda("launch allreduce_kernel", e);
    }
  }

  // 5. collect: per row, the times and checksums of every size, then the word checks
  std::vector<cdp::ArScratch> got(1);
  for (uint32_t li = 0; li < h->n_local; ++li) {
    cdp::LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    if (const int rc = cdp::fetch_reps(h, L, sizeof(cdp::ArScratch), got.data(), "cdprobe_allreduce"); rc != CDPROBE_OK)
      return rc;
    const cdp::ArScratch& s = got[0];
    cdp::bw_summarize(s.rep, want, size, n_sizes, reps, g, out);
    if (out->status[g] == CDPROBE_ERR_TIMEOUT) continue;
    for (uint32_t k = 0; k < n_sizes; ++k) {
      out->bad_words[g][k] = s.bad_words[k];
      out->first_bad[g][k] = s.bad_words[k] != 0 ? ~s.first_bad_n[k] : UINT64_MAX;
      if (s.bad_words[k] != 0) {
        out->bad_sizes[g] |= 1u << k;
        out->status[g] = CDPROBE_ERR_INTEGRITY;
      }
    }
  }
  out->ms = cdp::now_ms() - t_begin;
  return CDPROBE_OK;
}

}  // extern "C"
