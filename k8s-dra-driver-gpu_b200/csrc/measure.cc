// measure.cc — the on-demand measurements behind the C ABI: cdprobe_diagnose, cdprobe_latency, cdprobe_pingpong,
// cdprobe_atomics, cdprobe_bwcurve, cdprobe_allreduce, cdprobe_allreduce_twoshot, cdprobe_allreduce_ll,
// cdprobe_allreduce_ring, cdprobe_allreduce_push, cdprobe_allreduce_nvls, cdprobe_alltoall, cdprobe_memcpy and
// cdprobe_ce_alltoall.  Each
// runs on the local ranks' own streams, between probe runs, and has its results on the host before it returns.
#include <string.h>
#include <unistd.h>

#include <stddef.h>

#include <algorithm>
#include <array>
#include <memory>
#include <string>
#include <vector>

#include "allreduce.h"
#include "allreduce_ll.h"
#include "allreduce_nvls.h"
#include "allreduce_push.h"
#include "allreduce_ring.h"
#include "allreduce_twoshot.h"
#include "alltoall.h"
#include "atomics.h"
#include "bwcurve.h"
#include "diagnose.h"
#include "handle.h"
#include "latency.h"
#include "pingpong.h"

namespace cdp {

// Grows local rank L's scratch to at least `bytes`, on its device (the caller has selected it); the old buffer is freed
// first, and the new one is not zeroed.  The measurements share it: each runs on L's one stream, copies its results
// out before it returns, and reads back only what its own kernels wrote in the same call.  diag_launch clears its
// DiagOut and the compare pass writes every granule count; a rep table is read up to its first TIMEOUT slot, and the
// kernels write one for every cell they leave unfinished; launch_ladder clears a ladder kernel's records; the one-shot
// and LL all-reduces zero their output at the start of every call, and their word checks clear each word they read.
static int ensure_scratch(LocalRank& L, size_t bytes) {
  if (L.scratch_bytes >= bytes) return CDPROBE_OK;
  if (L.scratch) cudaFree(L.scratch);
  L.scratch = nullptr;
  L.scratch_bytes = 0;
  CDP_RT(cudaMalloc(&L.scratch, bytes));
  L.scratch_bytes = bytes;
  return CDPROBE_OK;
}

// Grows every local rank's scratch to at least `bytes` before any kernel is launched.  cudaFree synchronizes the
// device, and local ranks may share one: a kernel launched for an earlier rank would wait on this rank's.
static int ensure_scratch_all(cdprobe* h, size_t bytes) {
  for (uint32_t li = 0; li < h->n_local; ++li) {
    CDP_RT(cudaSetDevice(h->lr[li].ordinal));
    if (const int rc = ensure_scratch(h->lr[li], bytes); rc != CDPROBE_OK) return rc;
  }
  return CDPROBE_OK;
}
constexpr size_t kRepTableBytes = sizeof(TimedRep) * kMaxRanks * kRepSlots;  // latency, pingpong, atomics

// A launch, a copy or a kernel failed: the context is unusable, and so is the handle.
static int fail_sticky(cdprobe* h, const char* what, cudaError_t e) {
  h->sticky = true;
  return fail_cuda(what, e);
}

// Copies count T's from the head of local rank L's scratch (its rep tables, or the records a ladder kernel left) to
// `got` once its kernel is done.
template <typename T>
static int fetch_reps(cdprobe* h, LocalRank& L, T* got, size_t count, const char* what) {
  cudaError_t e = cudaSetDevice(L.ordinal);
  if (e == cudaSuccess) e = cudaMemcpyAsync(got, L.scratch, sizeof(T) * count, cudaMemcpyDeviceToHost, L.stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(L.stream);
  return e != cudaSuccess ? fail_sticky(h, what, e) : CDPROBE_OK;
}

// Clears the last error and *out and stamps the ABI version, as cdprobe_run does: the caller may read *out whatever
// the return code.  False when out is null.
template <typename Out>
static bool begin_output(Out* out) {
  g_last_error.clear();
  if (out == nullptr) return false;
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  return true;
}

// What each process contributes at the start of a collective measurement (cdprobe_pingpong, cdprobe_bwcurve,
// cdprobe_allreduce, cdprobe_alltoall), so that every process refuses, skips or runs the same call: the call number it
// is about to make, the arguments every process must pass alike (unused ones 0), whether its own were valid, its local
// ranks' smallest grid, whether its shared area must be zeroed before use, and its local ranks' rows of mapping status,
// [local rank][rank] with unmapped cells folded in (cdprobe_unmap_peer changes only the local view).
struct Agreement {
  uint64_t call_seq;
  std::array<uint32_t, 3> args;
  uint32_t ok;
  uint32_t ctas, zero;
  int32_t rows[kMaxRanks][kMaxRanks];
};

// What each process adds for cdprobe_allreduce_nvls, in a second exchange that only that call makes: whether its driver
// and every local device can take part in a multicast object (multicast_here), and its local ranks' device UUIDs.
struct NvlsFacts {
  uint32_t mc;
  char uuid[kMaxRanks][48];
};

// Whether this process can put every local rank into a multicast object: the driver has the multicast entry points,
// and every local device reports CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED (a MIG instance, or one simulated, never
// does).  A query that fails counts as no.
static bool multicast_here(cdprobe* h) {
  if (!h->drv.load_multicast()) return false;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    CUdevice dev;
    int on = 0;
    if (h->lr[li].mig || h->drv.DeviceGet(&dev, h->lr[li].ordinal) != CUDA_SUCCESS ||
        h->drv.DeviceGetAttribute(&on, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) != CUDA_SUCCESS || on == 0)
      return false;
  }
  return true;
}

// The handshake of collective measurement `fn`: every process contributes its Agreement (ok: its own verdict `bad` on
// its arguments is empty; zero: *zero, when given).  The first error wins: this process's own arguments, then another
// process's, then a call number or arguments that differ.  Returns CDPROBE_ERR_RENDEZVOUS when the exchange fails and
// CDPROBE_ERR_ARG on a refusal, with the message set.  Otherwise st, when given, gets the domain's matrix of mapping
// status, [rank][rank], which every process derives alike; grid, when given, the domain's smallest grid; and *zero
// whether any process must zero its area.  native: a measurement that needs remote atomics, so a live cell between two
// devices this process sees and that CUDA reports without cudaDevP2PAttrNativeAtomicSupported is folded into the rows
// as CDPROBE_ERR_UNSUPPORTED (a peer in another process counts as native, as in cdprobe_atomics).  nvls, when given,
// gets whether the domain can form one multicast object, from a second exchange (NvlsFacts): every process can put its
// ranks in (multicast_here), and no two ranks of the domain share a device, by UUID; a team holds each device once.
static int agree(cdprobe* h, const char* fn, std::string bad, uint64_t call_seq, const std::array<uint32_t, 3>& args,
                 int32_t (*st)[kMaxRanks], uint32_t* grid = nullptr, bool* zero = nullptr, bool native = false,
                 bool* nvls = nullptr) {
  Agreement mine = {call_seq, args, bad.empty() ? 1u : 0u, UINT32_MAX, zero != nullptr && *zero ? 1u : 0u, {}};
  for (uint32_t li = 0; li < h->n_local; ++li) {
    mine.ctas = std::min(mine.ctas, h->lr[li].ctas);
    for (uint32_t j = 0; j < h->n_total; ++j) {
      mine.rows[li][j] = cell_status(h, li, j);
      const bool local = j >= h->first && j < h->first + h->n_local;
      if (!native || mine.rows[li][j] != 0 || !local || h->lr[j - h->first].ordinal == h->lr[li].ordinal) continue;
      // a query that fails counts as no native atomics: returning here would leave the other processes at the allgather
      int ok = 0;
      if (cudaDeviceGetP2PAttribute(&ok, cudaDevP2PAttrNativeAtomicSupported, h->lr[li].ordinal,
                                    h->lr[j - h->first].ordinal) != cudaSuccess || ok == 0)
        mine.rows[li][j] = CDPROBE_ERR_UNSUPPORTED;
    }
  }
  std::vector<Agreement> all(h->cfg.world_size, mine);
  if (h->cfg.world_size > 1) {
    std::string err;
    if (h->rdv.allgather(&mine, sizeof(mine), all.data(), &err) != 0) {
      set_err(err);
      return CDPROBE_ERR_RENDEZVOUS;
    }
  }
  for (const Agreement& o : all) {
    if (!o.ok && bad.empty()) bad = std::string("another process called ") + fn + " with invalid arguments";
    if ((o.call_seq != mine.call_seq || o.args != mine.args) && bad.empty())
      bad = std::string(fn) + " is collective: every process must call it with the same arguments";
  }
  if (!bad.empty()) {
    set_err(bad);
    return CDPROBE_ERR_ARG;
  }
  if (st != nullptr) {
    memset(st, 0, sizeof(int32_t) * kMaxRanks * kMaxRanks);
    for (uint32_t r = 0; r < all.size(); ++r)
      for (uint32_t li = 0; li < h->n_local; ++li) memcpy(st[r * h->n_local + li], all[r].rows[li], sizeof(st[0]));
  }
  if (grid != nullptr) *grid = UINT32_MAX;
  for (const Agreement& o : all) {
    if (grid != nullptr) *grid = std::min(*grid, o.ctas);
    if (zero != nullptr) *zero |= o.zero != 0;
  }
  if (nvls == nullptr) return CDPROBE_OK;
  // every process has got here: the arguments agree everywhere
  NvlsFacts facts;
  memset(&facts, 0, sizeof(facts));
  facts.mc = multicast_here(h) ? 1u : 0u;
  for (uint32_t li = 0; li < h->n_local; ++li) memcpy(facts.uuid[li], h->lr[li].uuid, sizeof(facts.uuid[li]));
  std::vector<NvlsFacts> each(h->cfg.world_size, facts);
  if (h->cfg.world_size > 1) {
    std::string err;
    if (h->rdv.allgather(&facts, sizeof(facts), each.data(), &err) != 0) {
      set_err(err);
      return CDPROBE_ERR_RENDEZVOUS;
    }
  }
  *nvls = true;
  for (uint32_t p = 0; p < each.size(); ++p) {
    *nvls &= each[p].mc != 0;
    for (uint32_t li = 0; li < h->n_local; ++li)
      for (uint32_t q = 0; q <= p; ++q)
        for (uint32_t lj = 0; lj < (q == p ? li : h->n_local); ++lj)
          *nvls &= strncmp(each[p].uuid[li], each[q].uuid[lj], sizeof(each[p].uuid[li])) != 0;
  }
  return CDPROBE_OK;
}

// The cell rule of the one-sided measurements (latency, atomics, bwcurve): whether local rank li's cell to rank j runs.
// Cell (g, g) exists only with a loop-back slice; a cell whose mapping is down gets that status in status[] and is
// never read or written through.
static bool live_cell(const cdprobe* h, uint32_t li, uint32_t j, int32_t* status) {
  const uint32_t g = h->lr[li].grank;
  if (j == g && !h->plan.diag) return false;
  const int32_t s = cell_status(h, li, j);
  if (s != 0) status[g * CDPROBE_MAX_GPUS + j] = s;
  return s == 0;
}

// Waits until every process of the domain has got here; nothing to wait for in a single process.
static int domain_barrier(cdprobe* h) {
  if (h->cfg.world_size == 1) return CDPROBE_OK;
  std::string err;
  if (h->rdv.barrier(&err) != 0) {
    set_err(err);
    return CDPROBE_ERR_RENDEZVOUS;
  }
  return CDPROBE_OK;
}

// want[k], the (S, X) of the first size[k] bytes of the region whose word k is word(k), for every size: the
// per-granule sums of its whole bpp granules, computed from the pattern definition on local rank L's GPU into its
// scratch at table_off (grown by the caller), then folded into every prefix on the host.
template <typename Word>
static int expected_sums(cdprobe* h, LocalRank& L, size_t table_off, const Word& word, const uint64_t* size,
                         uint32_t n_sizes, uint64_t (*want)[2], const char* what) {
  const uint64_t granules = h->plan.bpp / kGranuleBytes;
  std::vector<uint64_t> table(2 * granules);
  uint64_t* gsum = reinterpret_cast<uint64_t*>(static_cast<uint8_t*>(L.scratch) + table_off);
  CDP_RT(cudaSetDevice(L.ordinal));
  cudaError_t e = (cudaError_t)granules_launch(gsum, gsum + granules, word, granules, (unsigned)L.sm_count * 8u,
                                               L.stream);
  if (e == cudaSuccess && granules)
    e = cudaMemcpyAsync(table.data(), gsum, 16 * granules, cudaMemcpyDeviceToHost, L.stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(L.stream);
  if (e != cudaSuccess) return fail_sticky(h, what, e);
  for (uint32_t k = 0; k < n_sizes; ++k)
    prefix_checksum(table.data(), table.data() + granules, size[k] / 8, word, &want[k][0], &want[k][1]);
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

// The cells one local rank's rep-table kernel measures: slot[k] of its table fills output cell idx[k], whose reps must
// have the digest want[k].  n == 0: no kernel was launched.
struct RepCells {
  uint32_t n = 0;
  uint32_t slot[kMaxRanks], idx[kMaxRanks];
  uint64_t want[kMaxRanks] = {};
  void add(uint32_t s, uint32_t i) {
    slot[n] = s;
    idx[n++] = i;
  }
};

// Collects the rep table of every local rank that launched, once its kernel is done, and summarizes each of its cells:
// ns per hop, round trip or atomic (`per_rep` of them per rep) of the timed reps, and the digest of all of them.
template <typename Out>
static int collect_reps(cdprobe* h, const RepCells* cells, uint32_t reps, uint32_t per_rep, const char* what, Out* out) {
  std::vector<TimedRep> got((size_t)kMaxRanks * kRepSlots);
  for (uint32_t li = 0; li < h->n_local; ++li) {
    const RepCells& c = cells[li];
    if (c.n == 0) continue;
    if (const int rc = fetch_reps(h, h->lr[li], got.data(), (size_t)(c.slot[c.n - 1] + 1) * kRepSlots, what);
        rc != CDPROBE_OK)
      return rc;
    for (uint32_t k = 0; k < c.n; ++k)
      summarize(got.data() + (size_t)c.slot[k] * kRepSlots, reps, per_rep, c.want[k], c.idx[k], out);
  }
  return CDPROBE_OK;
}

// Fills the times of entry idx of a ladder measurement from ns[k][r], ns of timed rep r + 1 of size k: per size, the
// minimum, median and maximum, and the model-free summary of the medians, whose rates are
// scale x size[k] / ns_median[k].  Sorts ns.
template <typename Out>
static void ladder_times(float (*ns)[kMaxTimedReps], const uint64_t* size, uint32_t n_sizes, uint32_t reps,
                         double scale, uint32_t idx, Out* out) {
  double rate[kBwMaxSizes], peak = 0.0;
  for (uint32_t k = 0; k < n_sizes; ++k) {
    std::sort(ns[k], ns[k] + reps);
    out->ns_min[idx][k] = ns[k][0];
    out->ns_median[idx][k] = ns[k][reps / 2];
    out->ns_max[idx][k] = ns[k][reps - 1];
    rate[k] = ns[k][reps / 2] > 0.f ? scale * (double)size[k] / (double)ns[k][reps / 2] : 0.0;
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
  out->status[idx] = 0;
}

// Fills the times of entry idx of a cdprobe_bwcurve_t (a cell), a cdprobe_allreduce_t (a row) or a cdprobe_alltoall_t
// (a row) from the rep records bwcurve_kernel, allreduce_kernel or alltoall_kernel left in `s` (ladder_times).  An
// entry whose kernel was aborted at the deadline has no times and is CDPROBE_ERR_TIMEOUT; returns whether it has times.
template <typename Out>
static bool bw_times(const BwScratch& s, const uint64_t* size, uint32_t n_sizes, uint32_t reps, double scale,
                     uint32_t idx, Out* out) {
  out->measured[idx] = 1;
  if (s.abort_flag != 0) {
    out->status[idx] = CDPROBE_ERR_TIMEOUT;
    return false;
  }
  float ns[kBwMaxSizes][kMaxTimedReps];
  for (uint32_t k = 0; k < n_sizes; ++k)
    for (uint32_t r = 1; r <= reps; ++r) ns[k][r - 1] = (float)(s.rep[k][r].t_end - s.t_rel[k][r]);
  ladder_times(ns, size, n_sizes, reps, scale, idx, out);
  return true;
}

// Fills entry idx of a cdprobe_bwcurve_t (a cell) or a cdprobe_allreduce_t (a row): the times (bw_times), the (S, X) of
// each size's last rep, and every rep's (S, X) compared with want[k] (bad_sizes).
template <typename Out>
static void bw_summarize(const BwScratch& s, const uint64_t (*want)[2], const uint64_t* size, uint32_t n_sizes,
                         uint32_t reps, uint32_t idx, Out* out) {
  if (!bw_times(s, size, n_sizes, reps, 1.0, idx, out)) return;
  uint32_t bad = 0;
  for (uint32_t k = 0; k < n_sizes; ++k) {
    for (uint32_t r = 0; r <= reps; ++r) {
      const Acc& a = s.rep[k][r];
      if (a.sum != want[k][0] || a.xr != want[k][1]) bad |= 1u << k;
    }
    out->sum[idx][k] = s.rep[k][reps].sum;
    out->xr[idx][k] = s.rep[k][reps].xr;
  }
  out->bad_sizes[idx] = bad;
  out->status[idx] = bad ? CDPROBE_ERR_INTEGRITY : 0;
}

// Fills the word checks of entry idx of a cdprobe_allreduce_t (a row) or a cdprobe_alltoall_t (a cell) from its
// kernel's per-size counts; an entry with a bad size gets CDPROBE_ERR_INTEGRITY in *status.
template <typename Out>
static void word_checks(const unsigned long long* bad_words, const unsigned long long* first_bad_n, uint32_t n_sizes,
                        uint32_t idx, int32_t* status, Out* out) {
  for (uint32_t k = 0; k < n_sizes; ++k) {
    out->bad_words[idx][k] = bad_words[k];
    out->first_bad[idx][k] = bad_words[k] != 0 ? ~first_bad_n[k] : UINT64_MAX;
    if (bad_words[k] != 0) out->bad_sizes[idx] |= 1u << k;
  }
  if (out->bad_sizes[idx] != 0) *status = CDPROBE_ERR_INTEGRITY;
}

// A ladder measurement as open_ladder lets it through: when it began, its reps, its size ladder, and the verdict on its
// arguments, empty when they are valid.
struct Ladder {
  double t_begin;
  uint32_t reps, n_sizes;
  uint64_t size[kBwMaxSizes];
  std::string bad;
};

// Where an armed ladder fault acts, from its low 32 bits, (k + 1) << 24 | word: size k and word `word` (for some modes
// a delay instead), and whether the call has that size and that size has that word.  k is valid only when size_ok.
struct FaultSpot {
  uint32_t k;
  uint64_t word;
  bool size_ok, word_ok;
};
static FaultSpot fault_spot(uint64_t v, const Ladder& lad) {
  const uint64_t fk = (v >> 24) & 0xffu, word = v & 0xffffffu;
  const bool size_ok = fk != 0 && fk <= lad.n_sizes;
  return {(uint32_t)fk - 1, word, size_ok, size_ok && word < lad.size[fk - 1] / 8};
}

// out->path of a ladder measurement that runs on the handle's data path (CDPROBE_OPT_PATH).
constexpr uint32_t kHandlePath = UINT32_MAX;

// out->path of a ladder measurement that reports one; cdprobe_memcpy_t and cdprobe_ce_alltoall_t have none (their
// copies use no data path).
template <typename Out>
static void put_path(Out* out, uint32_t path) {
  out->path = path;
}
static void put_path(cdprobe_memcpy_t*, uint32_t) {}
static void put_path(cdprobe_ce_alltoall_t*, uint32_t) {}

// The opening of the ladder measurements (bwcurve, the all-reduces, alltoall, memcpy): *out cleared and stamped with
// reps (0: default_reps); once the handle is known, n and the data path (`path`, or the handle's) before the handle is
// checked; then the size ladder by `rule` (bwcurve_ladder; allreduce_ll: ll_ladder) and the verdict on the arguments.
template <typename Out>
static int open_ladder(cdprobe* h, Out* out, uint32_t reps, uint32_t default_reps, Ladder* lad,
                       uint32_t path = kHandlePath, uint32_t (*rule)(uint64_t, uint64_t*) = bwcurve_ladder) {
  if (!begin_output(out)) return CDPROBE_ERR_ARG;
  out->reps = reps != 0 ? reps : default_reps;
  if (h == nullptr) return CDPROBE_ERR_ARG;
  lad->t_begin = now_ms();
  out->n = h->n_total;
  put_path(out, path == kHandlePath ? h->path : path);
  lad->reps = out->reps;
  if (const int rc = require_usable(h); rc != CDPROBE_OK) return rc;
  lad->n_sizes = rule(h->plan.bpp, lad->size);
  if (lad->reps > kMaxTimedReps) lad->bad = "reps must be at most 64";
  else if (lad->n_sizes == 0) lad->bad = "bytes_per_pair must be at most 32 GiB";
  return CDPROBE_OK;
}

// What a ladder measurement reports once every process has agreed to run it: the ladder and this process's rows.
template <typename Out>
static void put_ladder(const cdprobe* h, const Ladder& lad, Out* out) {
  out->n_sizes = lad.n_sizes;
  memcpy(out->size, lad.size, sizeof(lad.size[0]) * lad.n_sizes);
  for (uint32_t li = 0; li < h->n_local; ++li) out->row_mask |= 1u << h->lr[li].grank;
}

// Launches a ladder kernel on local rank L: the parameters every ladder kernel takes, then its records at the head of
// L's scratch cleared and the launch on L's stream.  A failed launch makes the handle sticky.
template <typename Params>
static int launch_ladder(cdprobe* h, LocalRank& L, Params& p, const Ladder& lad,
                         int (*launch)(const Params&, unsigned, bool, cudaStream_t), const char* what) {
  p.scratch = static_cast<decltype(p.scratch)>(L.scratch);
  memcpy(p.size, lad.size, sizeof(p.size));
  p.timeout_ns = timeout_ns(h);
  p.n_sizes = lad.n_sizes;
  p.reps = lad.reps;
  p.path = h->path;
  CDP_RT(cudaSetDevice(L.ordinal));
  cudaError_t e = cudaMemsetAsync(L.scratch, 0, sizeof(*p.scratch), L.stream);
  if (e == cudaSuccess) e = (cudaError_t)launch(p, L.ctas, launch_cooperatively(h, L), L.stream);
  return e != cudaSuccess ? fail_sticky(h, what, e) : CDPROBE_OK;
}

// [local rank][rank][size]: the (S, X) each size of each cell of bwcurve or memcpy must give.
using CellSums = uint64_t[kMaxRanks][kBwMaxSizes][2];
// *want[li][j] for every cell that runs: expected_sums of the source slice its op moves (memcpy_cell; bwcurve reads the
// slice a pull copies), on the issuer's GPU, with the granule table at table_off of its scratch, grown to hold it.
static int cell_sums(cdprobe* h, const bool (*runs)[kMaxRanks], uint32_t op, size_t table_off, const Ladder& lad,
                     const char* what, std::unique_ptr<CellSums[]>* want) {
  if (const int rc = ensure_scratch_all(h, table_off + 16 * (h->plan.bpp / kGranuleBytes)); rc != CDPROBE_OK) return rc;
  *want = std::make_unique<CellSums[]>(kMaxRanks);
  for (uint32_t li = 0; li < h->n_local; ++li) {
    for (uint32_t j = 0; j < h->n_total; ++j) {
      if (!runs[li][j]) continue;
      const MemcpyCell c = memcpy_cell(h->plan, op, h->lr[li].grank, j);
      const int rc = expected_sums(h, h->lr[li], table_off, SrcRegionWord{h->seed, c.first_word, c.src_rank}, lad.size,
                                   lad.n_sizes, (*want)[li][j], what);
      if (rc != CDPROBE_OK) return rc;
    }
  }
  return CDPROBE_OK;
}

// The rounds of bwcurve and memcpy, the tournament's then the loop-back, each behind a domain barrier: round(target),
// target[li] the rank local rank li's cell of the round reaches, -1 when it has none that runs.
template <typename Round>
static int walk_rounds(cdprobe* h, const bool (*runs)[kMaxRanks], const Round& round) {
  const Plan& pl = h->plan;
  const uint32_t n_rounds = pl.rounds + (pl.diag ? 1u : 0u);
  for (uint32_t r = 0; r < n_rounds; ++r) {
    if (const int rc = domain_barrier(h); rc != CDPROBE_OK) return rc;
    int32_t target[kMaxRanks];
    for (uint32_t li = 0; li < h->n_local; ++li) {
      const uint32_t g = h->lr[li].grank;
      const int q = r < pl.rounds ? pl.partner[r][g] : (int)g;
      target[li] = q >= 0 && runs[li][q] ? q : -1;
    }
    if (const int rc = round(target); rc != CDPROBE_OK) return rc;
  }
  return CDPROBE_OK;
}

// Folds area m's mapping status into the domain's mapping status st ([rank][rank]): a cell whose probe mapping is up
// gets its mapping of m.
static void fold_area_status(const cdprobe* h, const SharedAlloc& m, int32_t (*st)[kMaxRanks]) {
  for (uint32_t s = 0; s < h->n_total; ++s)
    for (uint32_t d = 0; d < h->n_total; ++d)
      if (st[s][d] == 0) st[s][d] = m.status[s][d];
}

// The skip rule of the all-reduces, on the domain's mapping status st ([rank][rank], 0: up): a process that ran while
// another skipped would wait at the first domain barrier until its watchdog fired, so when some rank cannot reach some
// other nothing runs, in any process: every local row gets the status of the domain's first down cell, row-major.
// Returns whether the call skips.
static const int32_t* first_down(int32_t (*st)[kMaxRanks]) {
  const int32_t* down = std::find_if(&st[0][0], &st[0][0] + kMaxRanks * kMaxRanks, [](int32_t s) { return s != 0; });
  return down == &st[0][0] + kMaxRanks * kMaxRanks ? nullptr : down;
}
static bool skip_rows(const cdprobe* h, int32_t (*st)[kMaxRanks], cdprobe_allreduce_t* out) {
  const int32_t* down = first_down(st);
  if (down == nullptr) return false;
  for (uint32_t li = 0; li < h->n_local; ++li) out->status[h->lr[li].grank] = *down;
  return true;
}

// Collects the rows of the all-reduces once their kernels are done: per local row, the times and every rep's (S, X)
// against want (bw_summarize), then the word checks of every size.
static int collect_rows(cdprobe* h, const uint64_t (*want)[2], const Ladder& lad, const char* what,
                        cdprobe_allreduce_t* out) {
  auto got = std::make_unique<ArScratch>();
  for (uint32_t li = 0; li < h->n_local; ++li) {
    LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    if (const int rc = fetch_reps(h, L, got.get(), 1, what); rc != CDPROBE_OK) return rc;
    const ArScratch& s = *got;
    bw_summarize(s.rep, want, lad.size, lad.n_sizes, lad.reps, g, out);
    if (out->status[g] != CDPROBE_ERR_TIMEOUT)
      word_checks(s.bad_words, s.first_bad_n, lad.n_sizes, g, &out->status[g], out);
  }
  return CDPROBE_OK;
}

// The barrier lines of local rank L in the FlagLine array at `off` in the Ctrl granule: it pushes into line L.grank of
// every other rank's array and waits on line j of its own for rank j.
static DomainLines domain_lines(const cdprobe* h, const LocalRank& L, uint64_t off, uint64_t call_seq) {
  DomainLines d;
  memset(&d, 0, sizeof(d));
  const uint32_t g = L.grank;
  const CUdeviceptr* va = h->mem.va[g - h->first];
  for (uint32_t j = 0; j < h->n_total; ++j) {
    if (j == g) continue;
    d.sig_out[j] = reinterpret_cast<uint64_t*>(va[j] + off + (uint64_t)g * sizeof(FlagLine));
    d.sig_in[j] = reinterpret_cast<const uint64_t*>(va[g] + off + (uint64_t)j * sizeof(FlagLine));
  }
  d.call_seq = call_seq;
  return d;
}

// An all-reduce's armed fault once its protocol has accepted it: in timed rep 1 of size k, rank `rank` (kArNoFault:
// none) acts on word `word` towards receiver `recv`, in `mode` (and, for the ring, in `phase`).  What each means is the
// protocol's.
struct ArFault {
  uint32_t rank = kArNoFault, recv = 0, k = kArNoFault, mode = 0;
  uint64_t word = 0;
  uint32_t phase = 0;
};

// One all-reduce protocol, as allreduce_call runs it.
struct ArProtocol {
  const char* fn;                                // the entry point, which names the call in every message
  Measurement meas;                              // its record on the handle: calls that ran, armed fault
  uint32_t (*rule)(uint64_t, uint64_t*);         // its size ladder
  uint32_t path;                                 // out->path: kHandlePath, or its own
  SharedAlloc cdprobe::*area;                    // the shared area peers write, nullptr: none
  uint64_t (*area_bytes)(uint32_t n, uint64_t s_max);  // its size per rank, for the ladder's largest size s_max
  const char* zeroing;                           // the area must start zeroed: names the step in a CUDA failure
  bool out_in_scratch;                           // the output takes s_max bytes of the scratch at kArOutOff
  uint64_t lines;                                // its barrier lines in the Ctrl granule
  // the verdict on fault v, whose size and word are `at`, for this call: nullptr with *f filled, or the refusal
  const char* (*decode)(const cdprobe* h, uint64_t v, const FaultSpot& at, const Ladder& lad, ArFault* f);
  // fills its parameters for local rank L and launches its kernel (launch_ladder)
  int (*launch)(cdprobe* h, LocalRank& L, const DomainLines& dom, const Ladder& lad, const ArFault& f, uint32_t grid);
  bool native = false;                           // it adds into peers' memory: every pair needs native atomics
  bool nvls = false;                             // it runs through the multicast object (h->nvls, ensure_nvls)
};

// The fields every all-reduce's parameters share, for local rank L, in parameters that start zeroed: the domain
// barrier, the seed, the rank, the rank count and the armed fault's size, kArNoFault unless the fault acts in L.
template <typename Params>
static Params ar_params(const cdprobe* h, const LocalRank& L, const DomainLines& dom, const ArFault& f) {
  Params p;
  memset(&p, 0, sizeof(p));
  p.dom = dom;
  p.seed = h->seed;
  p.rank = L.grank;
  p.n = h->n_total;
  p.fault_k = L.grank == f.rank ? f.k : kArNoFault;
  return p;
}

static const char* oneshot_fault(const cdprobe* h, uint64_t v, const FaultSpot& at, const Ladder&, ArFault* f) {
  const uint64_t fr = (v >> 32) & 0xffffu;
  if ((v >> 49) != 0 || fr == 0 || fr > h->n_total || !at.word_ok)
    return "the armed all-reduce fault names no rank, size or output word of this call";
  *f = {(uint32_t)fr - 1, 0, at.k, (uint32_t)(v >> 48), at.word};
  return nullptr;
}

static int oneshot_launch(cdprobe* h, LocalRank& L, const DomainLines& dom, const Ladder& lad, const ArFault& f,
                          uint32_t) {
  const uint32_t g = L.grank, n = h->n_total, li = g - h->first;
  AllReduceParams p = ar_params<AllReduceParams>(h, L, dom, f);
  for (uint32_t t = 0; t < n; ++t)
    p.src[t] = reinterpret_cast<const uint8_t*>(h->mem.va[li][(g + t) % n]) + h->plan.src_off;
  p.out = static_cast<uint8_t*>(L.scratch) + kArOutOff;
  p.fault_word = f.word;
  p.fault_drop = f.mode;
  return launch_ladder(h, L, p, lad, allreduce_launch, "launch allreduce_kernel");
}

// The fault acts in the rank whose chunk holds its word.
static const char* twoshot_fault(const cdprobe* h, uint64_t v, const FaultSpot& at, const Ladder& lad, ArFault* f) {
  const uint32_t n = h->n_total;
  const uint64_t fr = (v >> 32) & 0xffffu;
  if ((v >> 49) != 0 || fr == 0 || fr > n || !at.word_ok)
    return "the armed two-shot all-reduce fault names no receiver, size or output word of this call";
  *f = {kArNoFault, (uint32_t)fr - 1, at.k, (uint32_t)(v >> 48), at.word};
  const uint64_t units = (lad.size[f->k] + kUnitBytes - 1) / kUnitBytes, u = at.word / (kUnitBytes / 8);
  for (uint32_t r = 0; r < n; ++r) {
    uint64_t lo, hi;
    twoshot_chunk(units, n, r, &lo, &hi);
    if (u >= lo && u < hi) f->rank = r;
  }
  return nullptr;
}

static int twoshot_launch(cdprobe* h, LocalRank& L, const DomainLines& dom, const Ladder& lad, const ArFault& f,
                          uint32_t) {
  const uint32_t g = L.grank, n = h->n_total, li = g - h->first;
  TwoShotParams p = ar_params<TwoShotParams>(h, L, dom, f);
  for (uint32_t t = 0; t < n; ++t) {
    p.src[t] = reinterpret_cast<const uint8_t*>(h->mem.va[li][(g + t) % n]) + h->plan.src_off;
    p.dst[t] = reinterpret_cast<uint8_t*>(h->gather.va[li][(g + t) % n]);
  }
  p.fault_word = f.word;
  p.fault_dst = (f.recv + n - g) % n;
  p.fault_drop = f.mode;
  return launch_ladder(h, L, p, lad, allreduce_twoshot_launch, "launch allreduce_twoshot_kernel");
}

// The fault acts in the process that hosts its sender, which for mode 2 is its receiver.
static const char* ll_fault(const cdprobe* h, uint64_t v, const FaultSpot& at, const Ladder&, ArFault* f) {
  const uint32_t n = h->n_total;
  const uint64_t mode = v >> 48, fs = (v >> 40) & 0xffu, fr = (v >> 32) & 0xffu;
  if (mode > 2 || fs == 0 || fs > n || fr == 0 || fr > n || !at.size_ok || (mode != 1 && !at.word_ok) ||
      (mode == 0 && fs == fr) || (mode == 2 && fs != fr) || (mode == 1 && 2 * at.word >= 1000ull * h->cfg.timeout_ms))
    return "the armed LL all-reduce fault names no packet, size or delay of this call";
  *f = {(uint32_t)fs - 1, (uint32_t)fr - 1, at.k, (uint32_t)mode, at.word};
  return nullptr;
}

// Every rank splits the words over the domain's smallest grid, so that each word has the same owner everywhere.
static int ll_launch(cdprobe* h, LocalRank& L, const DomainLines& dom, const Ladder& lad, const ArFault& f,
                     uint32_t grid) {
  const uint32_t g = L.grank, n = h->n_total, li = g - h->first;
  LlParams p = ar_params<LlParams>(h, L, dom, f);
  p.src = reinterpret_cast<const uint8_t*>(h->mem.va[li][g]) + h->plan.src_off;
  for (uint32_t t = 1; t < n; ++t) p.dst[t] = reinterpret_cast<uint8_t*>(h->ll.va[li][(g + t) % n]);
  p.in = reinterpret_cast<const uint8_t*>(h->ll.va[li][g]);
  p.out = static_cast<uint8_t*>(L.scratch) + kArOutOff;
  p.s_max = lad.size[lad.n_sizes - 1];
  p.fault_mode = f.mode;
  p.fault_dst = (f.recv + n - g) % n;
  p.fault_arg = f.word;
  p.ctas = grid;
  return launch_ladder(h, L, p, lad, allreduce_ll_launch, "launch allreduce_ll_kernel");
}

// The fault acts in the process that hosts its sender.  A corrupted or dropped word must lie in a chunk the sender
// pushes in that phase: every chunk but its own in the reduce-scatter, every chunk but its successor's in the
// all-gather.
static const char* ring_fault(const cdprobe* h, uint64_t v, const FaultSpot& at, const Ladder& lad, ArFault* f) {
  const uint32_t n = h->n_total;
  const uint64_t mode = v >> 48, phase = (v >> 40) & 0xffu, fs = (v >> 32) & 0xffu;
  const char* why = "the armed ring all-reduce fault names no pushed word, size or delay of this call";
  if (mode > 2 || phase > 1 || fs == 0 || fs > n || !at.size_ok) return why;
  const uint32_t s = (uint32_t)fs - 1, k = at.k;
  if (mode == 2 && 2 * at.word >= 1000ull * h->cfg.timeout_ms) return why;
  if (mode < 2) {
    if (n == 1 || !at.word_ok) return why;
    const uint64_t units = (lad.size[k] + kUnitBytes - 1) / kUnitBytes, u = at.word / (kUnitBytes / 8);
    uint64_t lo, hi;
    twoshot_chunk(units, n, phase == 0 ? s : (s + 1) % n, &lo, &hi);
    if (u >= lo && u < hi) return why;
  }
  *f = {s, 0, k, (uint32_t)mode, at.word, (uint32_t)phase};
  return nullptr;
}

static int ring_launch(cdprobe* h, LocalRank& L, const DomainLines& dom, const Ladder& lad, const ArFault& f,
                       uint32_t) {
  const uint32_t g = L.grank, n = h->n_total, li = g - h->first;
  RingParams p = ar_params<RingParams>(h, L, dom, f);
  p.src = reinterpret_cast<const uint8_t*>(h->mem.va[li][g]) + h->plan.src_off;
  p.out = reinterpret_cast<uint8_t*>(h->ring.va[li][g]);
  p.next = reinterpret_cast<uint8_t*>(h->ring.va[li][(g + 1) % n]);
  p.s_max = lad.size[lad.n_sizes - 1];
  p.fault_mode = f.mode;
  p.fault_phase = f.phase;
  p.fault_arg = f.word;
  return launch_ladder(h, L, p, lad, allreduce_ring_launch, "launch allreduce_ring_kernel");
}

// Modes 0-2 act in the process that hosts the sender `rank`; mode 3 in the one that hosts the owner of the word's chunk,
// towards receiver `rank`, which must be a peer of that owner.
static const char* push_fault(const cdprobe* h, uint64_t v, const FaultSpot& at, const Ladder& lad, ArFault* f) {
  const uint32_t n = h->n_total;
  const uint64_t mode = v >> 48, fr = (v >> 32) & 0xffffu;
  if (mode > 3) return "the armed push all-reduce fault has a mode above 3";
  if (fr == 0 || fr > n) return "the armed push all-reduce fault names no rank of this domain";
  if (!at.size_ok) return "the armed push all-reduce fault names no size of this call";
  if (!at.word_ok) return "the armed push all-reduce fault names no output word of its size";
  const uint32_t r = (uint32_t)fr - 1, k = at.k;
  if (mode < 3) {
    *f = {r, 0, k, (uint32_t)mode, at.word};
    return nullptr;
  }
  if (n == 1) return "the armed push all-reduce fault's mode 3 has no peer to push to at n == 1";
  const uint32_t owner = twoshot_owner((lad.size[k] + kUnitBytes - 1) / kUnitBytes, n, at.word / (kUnitBytes / 8));
  if (owner == r) return "the armed push all-reduce fault's mode-3 receiver owns the word and is pushed no copy of it";
  *f = {owner, r, k, 3u, at.word};
  return nullptr;
}

static int push_launch(cdprobe* h, LocalRank& L, const DomainLines& dom, const Ladder& lad, const ArFault& f,
                       uint32_t) {
  const uint32_t g = L.grank, n = h->n_total, li = g - h->first;
  PushParams p = ar_params<PushParams>(h, L, dom, f);
  p.src = reinterpret_cast<const uint8_t*>(h->mem.va[li][g]) + h->plan.src_off;
  for (uint32_t t = 0; t < n; ++t) p.dst[t] = reinterpret_cast<uint8_t*>(h->push.va[li][(g + t) % n]);
  p.fault_word = f.word;
  p.fault_mode = f.mode;
  p.fault_dst = (f.recv + n - g) % n;
  return launch_ladder(h, L, p, lad, allreduce_push_launch, "launch allreduce_push_kernel");
}

// The fault acts in the process that hosts the owner of the word's chunk.
static const char* nvls_fault(const cdprobe* h, uint64_t v, const FaultSpot& at, const Ladder& lad, ArFault* f) {
  const uint64_t mode = v >> 48;
  if (mode > 1) return "the armed NVLS all-reduce fault has a mode above 1";
  if (((v >> 32) & 0xffffu) != 0) return "the armed NVLS all-reduce fault sets bits 32 to 47, which name nothing";
  if (!at.size_ok) return "the armed NVLS all-reduce fault names no size of this call";
  if (!at.word_ok) return "the armed NVLS all-reduce fault names no output word of its size";
  const uint64_t units = (lad.size[at.k] + kUnitBytes - 1) / kUnitBytes;
  *f = {twoshot_owner(units, h->n_total, at.word / (kUnitBytes / 8)), 0, at.k, (uint32_t)mode, at.word};
  return nullptr;
}

// The input half is the first s_max bytes of the rank's NVLS area, the output half the next s_max.
static int nvls_launch(cdprobe* h, LocalRank& L, const DomainLines& dom, const Ladder& lad, const ArFault& f,
                       uint32_t) {
  const uint32_t g = L.grank, li = g - h->first;
  const uint64_t s_max = lad.size[lad.n_sizes - 1];
  NvlsParams p = ar_params<NvlsParams>(h, L, dom, f);
  p.mc_in = reinterpret_cast<const uint8_t*>(h->nvls.mc_va[li]);
  p.mc_out = reinterpret_cast<uint8_t*>(h->nvls.mc_va[li] + s_max);
  p.out = reinterpret_cast<uint8_t*>(h->nvls.uc_va[li] + s_max);
  p.fault_word = f.word;
  p.fault_mode = f.mode;
  return launch_ladder(h, L, p, lad, allreduce_nvls_launch, "launch allreduce_nvls_kernel");
}

constexpr ArProtocol kOneShot = {
    "cdprobe_allreduce", kMeasAllReduce, bwcurve_ladder, kHandlePath, nullptr, nullptr, nullptr, true, kArOff,
    oneshot_fault, oneshot_launch};
constexpr ArProtocol kTwoShot = {
    "cdprobe_allreduce_twoshot", kMeasTwoShot, bwcurve_ladder, kHandlePath, &cdprobe::gather,
    [](uint32_t, uint64_t s_max) { return s_max; }, nullptr, false, kAr2Off, twoshot_fault, twoshot_launch};
constexpr ArProtocol kLl = {
    "cdprobe_allreduce_ll", kMeasLl, ll_ladder, CDPROBE_ALLREDUCE_PATH_LL, &cdprobe::ll, ll_area_bytes,
    "cdprobe_allreduce_ll: zero the LL area", true, kLlOff, ll_fault, ll_launch};
constexpr ArProtocol kRing = {
    "cdprobe_allreduce_ring", kMeasRing, bwcurve_ladder, CDPROBE_ALLREDUCE_PATH_RING, &cdprobe::ring, ring_area_bytes,
    "cdprobe_allreduce_ring: zero the ring area", false, kRingOff, ring_fault, ring_launch};
constexpr ArProtocol kPush = {
    "cdprobe_allreduce_push", kMeasPush, bwcurve_ladder, kHandlePath, &cdprobe::push,
    [](uint32_t, uint64_t s_max) { return s_max; }, "cdprobe_allreduce_push: zero the push area", false, kPushOff,
    push_fault, push_launch, true};
constexpr ArProtocol kNvls = {
    "cdprobe_allreduce_nvls", kMeasNvls, bwcurve_ladder, CDPROBE_ALLREDUCE_PATH_NVLS, nullptr, nullptr, nullptr, false,
    kNvlsOff, nvls_fault, nvls_launch, false, true};

// The all-reduces (DESIGN §5g, §5i, §5j, §5k, §5l, §5m): one call of protocol P.
static int allreduce_call(cdprobe* h, uint32_t reps, cdprobe_allreduce_t* out, const ArProtocol& P) {
  Ladder lad;
  if (const int rc = open_ladder(h, out, reps, kArDefaultReps, &lad, P.path, P.rule); rc != CDPROBE_OK) return rc;
  const uint32_t n = h->n_total;
  MeasRecord& rec = h->meas[P.meas];
  // 1. the arguments, the armed fault, the probe mapping rows and whether any area must be zeroed; in a multi-process
  //    domain all are shared, so every process refuses, skips, zeroes or runs together.  An area that must start zeroed
  //    and is yet to be created is stale until it is zeroed
  ArFault f;
  if (rec.fault != 0 && lad.bad.empty())
    if (const char* why = P.decode(h, rec.fault, fault_spot(rec.fault, lad), lad, &f)) lad.bad = why;
  SharedAlloc* m = P.area != nullptr ? &(h->*P.area) : nullptr;
  if (P.zeroing != nullptr) m->stale |= m->bytes == 0;
  bool zero = P.zeroing != nullptr && m->stale;
  uint32_t grid;
  int32_t st[kMaxRanks][kMaxRanks];
  bool nvls = true;
  if (const int rc = agree(h, P.fn, lad.bad, rec.calls + 1, {lad.reps, 0u, 0u}, st, &grid, &zero, P.native,
                           P.nvls ? &nvls : nullptr);
      rc != CDPROBE_OK)
    return rc;
  // a domain that cannot form a multicast object runs nothing, whatever its mappings
  const auto unsupported = [&] {
    for (uint32_t s = 0; s < n; ++s)
      for (uint32_t d = 0; d < n; ++d) st[s][d] = CDPROBE_ERR_UNSUPPORTED;
  };
  if (!nvls) unsupported();
  // 2. the area, built once, by every process in the same call; the NVLS area only for a call that will run.  A
  //    driver that refuses a multicast object of one device leaves a one-rank domain unsupported, with the CUresult in
  //    cdprobe_last_error
  const uint64_t s_max = lad.size[lad.n_sizes - 1];
  if (m != nullptr)
    if (const int rc = ensure_area(h, *m, P.area_bytes(n, s_max)); rc != CDPROBE_OK) return rc;
  if (P.nvls && first_down(st) == nullptr) {
    bool refused = false;
    const int rc = ensure_nvls(h, 2 * s_max, &refused);
    if (refused) unsupported();
    else if (rc != CDPROBE_OK) return rc;
  }
  out->call_seq = ++rec.calls;
  put_ladder(h, lad, out);
  // 3. every rank reads every input and writes every area: when some probe mapping or area mapping of the domain is
  //    down, nothing runs, in any process
  if (m != nullptr) fold_area_status(h, *m, st);
  if (skip_rows(h, st, out)) {
    out->ms = now_ms() - lad.t_begin;
    return CDPROBE_OK;
  }
  // 4. every process zeroes its local ranks' areas before any kernel of this call can push into them
  if (zero && P.zeroing != nullptr) {
    for (uint32_t li = 0; li < h->n_local; ++li) {
      LocalRank& L = h->lr[li];
      CDP_RT(cudaSetDevice(L.ordinal));
      cudaError_t e = cudaMemsetAsync(reinterpret_cast<void*>(m->va[li][L.grank]), 0, m->bytes, L.stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(L.stream);
      if (e != cudaSuccess) return fail_sticky(h, P.zeroing, e);
    }
    m->stale = false;
  }
  // the NVLS input is the first s_max bytes of each rank's source buffer, and its output starts zeroed, on every call
  if (P.nvls) {
    for (uint32_t li = 0; li < h->n_local; ++li) {
      LocalRank& L = h->lr[li];
      CDP_RT(cudaSetDevice(L.ordinal));
      void* const in = reinterpret_cast<void*>(h->nvls.uc_va[li]);
      const void* const src = reinterpret_cast<const void*>(h->mem.va[li][L.grank] + h->plan.src_off);
      cudaError_t e = cudaMemcpyAsync(in, src, s_max, cudaMemcpyDeviceToDevice, L.stream);
      if (e == cudaSuccess) e = cudaMemsetAsync(static_cast<uint8_t*>(in) + s_max, 0, s_max, L.stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(L.stream);
      if (e != cudaSuccess) return fail_sticky(h, "cdprobe_allreduce_nvls: fill the NVLS area", e);
    }
  }

  // 5. scratch for the records, the output (when it is there) and the granule table, grown on every local rank before
  //    any kernel runs; the (S, X) every prefix of the output must have, from the pattern definition: the per-granule
  //    sums of the summed words on the first local rank's GPU, folded into every prefix on the host
  const size_t table_off = kArOutOff + (P.out_in_scratch ? (s_max + 255) / 256 * 256 : 0);
  if (const int rc = ensure_scratch_all(h, table_off + 16 * (h->plan.bpp / kGranuleBytes)); rc != CDPROBE_OK) return rc;
  // an output in the scratch starts zeroed on every call, so a word this call does not store reads as 0 rather than
  // as what an earlier call, an aborted one or another handle's left there
  if (P.out_in_scratch) {
    for (uint32_t li = 0; li < h->n_local; ++li) {
      LocalRank& L = h->lr[li];
      CDP_RT(cudaSetDevice(L.ordinal));
      const cudaError_t e = cudaMemsetAsync(static_cast<uint8_t*>(L.scratch) + kArOutOff, 0, s_max, L.stream);
      if (e != cudaSuccess) return fail_sticky(h, (std::string(P.fn) + ": zero the output").c_str(), e);
    }
  }
  uint64_t want[kBwMaxSizes][2] = {};
  if (const int rc = expected_sums(h, h->lr[0], table_off, AllReduceWord{h->seed, n}, lad.size, lad.n_sizes, want,
                                   (std::string(P.fn) + ": granule checksums").c_str());
      rc != CDPROBE_OK)
    return rc;

  // 6. no process launches before every process is ready, so that no kernel waits at its first domain barrier for a
  //    process still setting up; then every local kernel is launched before any is waited for
  if (const int rc = domain_barrier(h); rc != CDPROBE_OK) return rc;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    LocalRank& L = h->lr[li];
    if (const int rc = P.launch(h, L, domain_lines(h, L, P.lines, rec.calls), lad, f, grid); rc != CDPROBE_OK)
      return rc;
  }

  // 7. collect: per row, the times and every rep's checksums, then the word checks; a row that timed out leaves an area
  //    that must start zeroed stale, to be zeroed before the next call runs
  if (const int rc = collect_rows(h, want, lad, P.fn, out); rc != CDPROBE_OK) return rc;
  if (P.zeroing != nullptr)
    for (uint32_t li = 0; li < h->n_local; ++li) m->stale |= out->status[h->lr[li].grank] == CDPROBE_ERR_TIMEOUT;
  out->ms = now_ms() - lad.t_begin;
  return CDPROBE_OK;
}

// What the checks of one rep of a block leave for the host (check_block), copied back on the checking rank's stream
// behind them: the head of the diagnosis (bad_words, bad_granules, first_bad_n of its DiagOut) and the (S, X) read of
// bwcurve_kernel (its abort word and the Acc of its one rep).
struct MemcpyRepOut {
  unsigned long long diag[3];
  unsigned int abort_flag;
  Acc acc;
};
static_assert(offsetof(DiagOut, bad_words) == 0 && offsetof(DiagOut, first_bad_n) == 16, "the diagnosis head");
static_assert(offsetof(BwScratch, abort_flag) == 0, "the (S, X) read's abort word");

// The pinned, mapped and portable host block of the copy-engine measurements (cdprobe_memcpy, cdprobe_ce_alltoall),
// made by the first call of either (copy_setup) and kept until close: the ticket every local stream waits on
// (cuStreamWaitValue64, through its UVA address), the second ticket a CE all-to-all mode-2 fault holds a copy stream
// on, the tickets handed out so far, the word an armed mode-0 fault stores per local rank, the awaited values the CE
// all-to-all writes into its own ranks' lines when it gives up on a rep, and what each rep's checks left, per local
// rank, block and rep: memcpy's cell [issuer][target], the CE all-to-all's block [owner][sender].  Both calls take
// their tickets from `issued`; tickets only rise, and a handle runs one call at a time, so a GEQ wait on either ticket
// is met only by the rep it was queued for.
struct CopyHost {
  uint64_t ticket, hold, issued;
  uint64_t flip[kMaxRanks];
  uint64_t release[2];
  MemcpyRepOut rep[kMaxRanks][kMaxRanks][kRepSlots];
};

// Where cdprobe_memcpy keeps its device state in a local rank's scratch: the BwScratch of the (S, X) read at 0, the
// diagnosis of a destination of up to bytes_per_pair at diag_off, the granule table of expected_sums at table_off.
struct MemcpyScratch {
  size_t diag_off, table_off;
  explicit MemcpyScratch(uint64_t bpp) {
    diag_off = (sizeof(BwScratch) + 255) / 256 * 256;
    table_off = diag_off + (diag_scratch_bytes(bpp) + 255) / 256 * 256;
  }
};

// The host block and every local rank's rep events, made on the first call of either copy-engine measurement.
static int copy_setup(cdprobe* h) {
  CDP_RT(cudaSetDevice(h->lr[0].ordinal));
  if (h->copy_host == nullptr) {
    void* p = nullptr;
    CDP_RT(cudaHostAlloc(&p, sizeof(CopyHost), cudaHostAllocPortable | cudaHostAllocMapped));
    memset(p, 0, sizeof(CopyHost));
    h->copy_host = static_cast<CopyHost*>(p);
  }
  for (uint32_t li = 0; li < h->n_local; ++li) {
    LocalRank& L = h->lr[li];
    CDP_RT(cudaSetDevice(L.ordinal));
    for (cudaEvent_t& ev : L.rep_ev)
      if (ev == nullptr) CDP_RT(cudaEventCreate(&ev));
  }
  return CDPROBE_OK;
}

// A copy-engine measurement's armed fault once the call has accepted it: timed rep 1 of size k of cell (issuer,
// target) flips destination word `arg` (mode 0), queues no copy (mode 1), or holds the copy `arg` us (mode 2, the CE
// all-to-all's).  issuer kMaxRanks: none.
struct CopyFault {
  uint32_t issuer = kMaxRanks, target = 0, k = 0, mode = 0;
  uint64_t arg = 0;
};

// One copy-engine measurement, as open_copy opens it.
struct CopyCall {
  const char* fn;                      // the entry point
  uint32_t default_reps;
  Measurement meas;                    // its record on the handle: calls that ran, armed fault
  uint64_t max_mode;                   // the highest fault mode it accepts
  const char* bad_fault;               // its refusal of an armed fault
  std::string (*refusal)(cdprobe* h);  // why this process cannot run it, empty when it can; nullptr: it always can
  const char* refused_elsewhere;       // its refusal when only another process cannot run it
};

// The opening of the copy-engine measurements: open_ladder, with out->op; the verdict on op, then on the armed fault
// (`(mode << 48) | ((issuer + 1) << 40) | ((target + 1) << 32) | fault_spot`: a mode below 2 names a word of its size,
// mode 2 a size and a delay under timeout_ms / 2); then, with valid arguments, C.refusal.  All are agreed over every
// process, so every process refuses or runs together, and a refusal is CDPROBE_ERR_UNSUPPORTED.  Then the exchange area
// (cdprobe_alltoall's, built once, by every process in the same call), the call number and the ladder.  *st gets the
// domain's probe mapping status.
template <typename Out>
static int open_copy(cdprobe* h, const CopyCall& C, uint32_t op, uint32_t reps, Out* out, Ladder* lad, CopyFault* f,
                     int32_t (*st)[kMaxRanks]) {
  const int opened = open_ladder(h, out, reps, C.default_reps, lad);
  if (out != nullptr) out->op = op;
  if (opened != CDPROBE_OK) return opened;
  const uint32_t n = h->n_total;
  if (op != CDPROBE_OP_READ && op != CDPROBE_OP_WRITE && lad->bad.empty())
    lad->bad = "op must be CDPROBE_OP_READ or CDPROBE_OP_WRITE";
  MeasRecord& rec = h->meas[C.meas];
  if (const uint64_t v = rec.fault; v != 0 && lad->bad.empty()) {
    const uint64_t mode = v >> 48, fi = (v >> 40) & 0xffu, ft = (v >> 32) & 0xffu;
    const FaultSpot at = fault_spot(v, *lad);
    if (mode > C.max_mode || fi == 0 || fi > n || ft == 0 || ft > n || (fi == ft && !h->plan.diag) || !at.size_ok ||
        (mode < 2 && !at.word_ok) || (mode == 2 && 2 * at.word >= 1000ull * h->cfg.timeout_ms))
      lad->bad = C.bad_fault;
    else
      *f = {(uint32_t)fi - 1, (uint32_t)ft - 1, at.k, (uint32_t)mode, at.word};
  }
  const std::string refusal = C.refusal != nullptr && lad->bad.empty() ? C.refusal(h) : std::string();
  bool refused = !refusal.empty();
  // agree() ors the refusal flag (its `zero`) over every process
  if (const int rc = agree(h, C.fn, lad->bad, rec.calls + 1, {lad->reps, op, 0u}, st, nullptr, &refused);
      rc != CDPROBE_OK)
    return rc;
  if (refused) {
    set_err(!refusal.empty() ? refusal : std::string(C.refused_elsewhere));
    return CDPROBE_ERR_UNSUPPORTED;
  }
  if (const int rc = ensure_area(h, h->area, (size_t)n * h->plan.bpp); rc != CDPROBE_OK) return rc;
  out->call_seq = ++rec.calls;
  out->area_bytes = h->area.bytes;
  put_ladder(h, *lad, out);
  return CDPROBE_OK;
}

// The armed mode-0 fault's store, queued on stream s of local rank li after cell c's copy: destination word `word`
// overwritten, by an 8-byte copy from the host block, with its pattern value xored with 1.
static cudaError_t store_flip(cdprobe* h, uint32_t li, const MemcpyCell& c, uint64_t word, cudaStream_t s) {
  uint64_t* const w = &h->copy_host->flip[li];
  *w = src_word(h->seed, c.src_rank, c.first_word + word) ^ 1ull;
  return cudaMemcpyAsync(reinterpret_cast<uint8_t*>(h->area.va[li][c.dst_rank] + c.dst_off) + 8 * word, w, 8,
                         cudaMemcpyHostToDevice, s);
}

// Waits, polling, until event B of rep `rep` has completed on every local rank in `ranks` (bit li), from the rep's
// release: a copy cannot be aborted, so never an unbounded synchronise.  A failed query returns its error (`failed`)
// and a B not complete timeout_ms after the release CDPROBE_ERR_TIMEOUT (`late`); either makes the handle sticky.
static int wait_reps(cdprobe* h, uint32_t ranks, uint32_t rep, const char* failed, const char* late) {
  const double deadline = now_ms() + h->cfg.timeout_ms;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    if ((ranks >> li & 1u) == 0) continue;
    LocalRank& L = h->lr[li];
    CDP_RT(cudaSetDevice(L.ordinal));
    cudaError_t e;
    while ((e = cudaEventQuery(L.rep_ev[2 * rep + 1])) != cudaSuccess) {
      if (e != cudaErrorNotReady) return fail_sticky(h, failed, e);
      if (now_ms() > deadline) {
        h->sticky = true;
        set_err(late);
        return CDPROBE_ERR_TIMEOUT;
      }
    }
  }
  return CDPROBE_OK;
}

// Folds what the checks of size k of one block left, got[rep] for the warm-up and every timed rep, into entry idx of a
// cdprobe_memcpy_t (a cell) or a cdprobe_ce_alltoall_t (a block): bad_words over every rep and first_bad, the lowest
// bad offset of any; bit k of bad_sizes for a bad word or an (S, X) other than `want` in any rep; the last rep's
// (S, X).  Returns whether any rep's (S, X) read was aborted at its deadline.
template <typename Out>
static bool fold_checks(const MemcpyRepOut* got, uint32_t reps, uint32_t k, const uint64_t* want, uint32_t idx,
                        Out* out) {
  bool aborted = false;
  uint64_t first = UINT64_MAX;
  for (uint32_t rep = 0; rep <= reps; ++rep) {
    const MemcpyRepOut& g = got[rep];
    aborted |= g.abort_flag != 0;
    out->bad_words[idx][k] += g.diag[0];
    if (g.diag[0] != 0) first = std::min(first, (uint64_t)~g.diag[2]);
    if (g.diag[0] != 0 || g.acc.sum != want[0] || g.acc.xr != want[1]) out->bad_sizes[idx] |= 1u << k;
  }
  out->first_bad[idx][k] = first;
  out->sum[idx][k] = got[reps].acc.sum;
  out->xr[idx][k] = got[reps].acc.xr;
  return aborted;
}

// The status of a block once every size is folded: an (S, X) read aborted at its deadline, else a size that failed
// its checks, else 0.
static int32_t copy_verdict(bool aborted, uint32_t bad_sizes) {
  return aborted ? CDPROBE_ERR_TIMEOUT : bad_sizes != 0 ? CDPROBE_ERR_INTEGRITY : 0;
}

// The timed part of rep `rep` of cdprobe_memcpy's cell (L.grank, j), L = h->lr[li], queued on L's stream: the wait
// for the rep's ticket, event A, the copy (none when `drop`), event B.  A failure of the stream wait itself is
// cudaErrorUnknown with the driver's result in *cu.
static cudaError_t memcpy_timed(cdprobe* h, uint32_t li, uint32_t j, uint32_t op, uint64_t ticket, uint64_t bytes,
                                uint32_t rep, bool drop, CUresult* cu) {
  LocalRank& L = h->lr[li];
  const MemcpyCell c = memcpy_cell(h->plan, op, L.grank, j);
  cudaError_t e = cudaSetDevice(L.ordinal);
  if (e != cudaSuccess) return e;
  *cu = h->drv.StreamWaitValue64(L.stream, reinterpret_cast<CUdeviceptr>(&h->copy_host->ticket), ticket,
                                 CU_STREAM_WAIT_VALUE_GEQ);
  if (*cu != CUDA_SUCCESS) return cudaErrorUnknown;
  e = cudaEventRecord(L.rep_ev[2 * rep], L.stream);
  if (e == cudaSuccess && !drop)
    e = cudaMemcpyAsync(reinterpret_cast<void*>(h->area.va[li][c.dst_rank] + c.dst_off),
                        reinterpret_cast<const void*>(h->mem.va[li][c.src_rank] + c.src_off), bytes,
                        cudaMemcpyDeviceToDevice, L.stream);
  if (e == cudaSuccess) e = cudaEventRecord(L.rep_ev[2 * rep + 1], L.stream);
  return e;
}

// The untimed checks of the block cell `c` landed, queued on stream `s` of local rank L = h->lr[li], the block's
// owner, on its own memory and scratch: the diagnosis of every destination word against the source slice's pattern
// (diag_launch), the (S, X) read of the destination (bwcurve_kernel, one rep of one size), the clearing of the
// destination to 0, and the copies of what the checks left into `got`.  cdprobe_memcpy's issuer and
// cdprobe_ce_alltoall's owners check this way.
static cudaError_t check_block(cdprobe* h, uint32_t li, const MemcpyCell& c, uint64_t bytes, MemcpyRepOut* got) {
  LocalRank& L = h->lr[li];
  const Plan& pl = h->plan;
  const MemcpyScratch ms(pl.bpp);
  uint8_t* const dst = reinterpret_cast<uint8_t*>(h->area.va[li][c.dst_rank] + c.dst_off);
  uint8_t* const scratch = static_cast<uint8_t*>(L.scratch);
  cudaStream_t s = L.stream;
  cudaError_t e = (cudaError_t)diag_launch(
      dst, diag_read_spec(h->seed, h->n_total, c.src_rank, c.first_word, bytes / 8, pl.src_bytes / 8),
      scratch + ms.diag_off, L.sm_count, s);
  if (e == cudaSuccess) e = cudaMemsetAsync(scratch, 0, sizeof(BwScratch), s);
  if (e == cudaSuccess) {
    BwCurveParams p;
    memset(&p, 0, sizeof(p));
    p.region = dst;
    p.scratch = reinterpret_cast<BwScratch*>(scratch);
    p.size[0] = bytes;
    p.timeout_ns = timeout_ns(h);
    p.n_sizes = 1;
    p.path = h->path;
    e = (cudaError_t)bwcurve_launch(p, L.ctas, launch_cooperatively(h, L), s);
  }
  if (e == cudaSuccess) e = cudaMemsetAsync(dst, 0, bytes, s);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(got->diag, scratch + ms.diag_off, sizeof(got->diag), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(&got->abort_flag, scratch, sizeof(got->abort_flag), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(&got->acc, scratch + offsetof(BwScratch, rep), sizeof(got->acc), cudaMemcpyDeviceToHost, s);
  return e;
}

// The untimed checks of rep `rep` of the cell, queued on L's stream behind its event B: the armed mode-0 fault's store
// (`flip`: word flip_word), then check_block into the cell's slot of the host block.
static cudaError_t memcpy_check(cdprobe* h, uint32_t li, uint32_t j, uint32_t op, uint64_t bytes, uint32_t rep,
                                bool flip, uint64_t flip_word) {
  LocalRank& L = h->lr[li];
  const MemcpyCell c = memcpy_cell(h->plan, op, L.grank, j);
  cudaError_t e = cudaSetDevice(L.ordinal);
  if (e == cudaSuccess && flip) e = store_flip(h, li, c, flip_word, L.stream);
  if (e == cudaSuccess) e = check_block(h, li, c, bytes, &h->copy_host->rep[li][j][rep]);
  return e;
}

// Rep `rep` of size k of cdprobe_memcpy on every local rank with a cell in this round (target[li] >= 0).  The timed
// part of every rank's rep is queued (memcpy_timed) before the host releases the rep's ticket, so the events bracket
// the copy alone, without the host's enqueue time; the ticket is released even when queuing fails, so no stream is
// left waiting.  Then the host waits until every copy's event B has completed (wait_reps), and only then queues the
// checks (memcpy_check): launching a kernel may have to load it, which must not wait behind a stream that waits on
// the host, and no host submission overlaps a timed copy.
static int memcpy_rep(cdprobe* h, const int32_t* target, uint32_t op, const Ladder& lad, uint32_t k, uint32_t rep,
                      const CopyFault& f) {
  const uint64_t ticket = ++h->copy_host->issued, bytes = lad.size[k];
  auto armed = [&](uint32_t li) {
    return rep == 1 && k == f.k && h->lr[li].grank == f.issuer && (uint32_t)target[li] == f.target;
  };
  cudaError_t e = cudaSuccess;
  CUresult cu = CUDA_SUCCESS;
  uint32_t ranks = 0;
  for (uint32_t li = 0; li < h->n_local && e == cudaSuccess; ++li) {
    if (target[li] < 0) continue;
    ranks |= 1u << li;
    e = memcpy_timed(h, li, (uint32_t)target[li], op, ticket, bytes, rep, armed(li) && f.mode == 1, &cu);
  }
  __atomic_store_n(&h->copy_host->ticket, ticket, __ATOMIC_RELEASE);
  if (cu != CUDA_SUCCESS) {
    h->sticky = true;
    set_err("cdprobe_memcpy: cuStreamWaitValue64: " + h->drv.error_name(cu));
    return CDPROBE_ERR_CUDA;
  }
  if (e != cudaSuccess) return fail_sticky(h, "cdprobe_memcpy: queue a rep", e);
  if (const int rc = wait_reps(h, ranks, rep, "cdprobe_memcpy: wait for a copy",
                               "cdprobe_memcpy: a copy did not complete within timeout_ms of its release");
      rc != CDPROBE_OK)
    return rc;
  for (uint32_t li = 0; li < h->n_local && e == cudaSuccess; ++li)
    if (target[li] >= 0)
      e = memcpy_check(h, li, (uint32_t)target[li], op, bytes, rep, armed(li) && f.mode == 0, f.arg);
  return e != cudaSuccess ? fail_sticky(h, "cdprobe_memcpy: queue the checks", e) : CDPROBE_OK;
}

constexpr CopyCall kMemcpy = {
    "cdprobe_memcpy", 8, kMeasMemcpy, 1,
    "the armed memcpy fault names no cell, size or word of this call, or has a mode above 1", nullptr, nullptr};

// The cells local rank li issues, one per copy stream: its peers in the order rank + 1, rank + 2, ... (mod n), then
// the diagonal with a loop-back slice.  Returns their count.
static uint32_t ce_a2a_targets(const cdprobe* h, uint32_t li, uint32_t* target) {
  const uint32_t g = h->lr[li].grank, n = h->n_total;
  uint32_t c = 0;
  for (uint32_t d = 1; d <= n; ++d)
    if ((g + d) % n != g || h->plan.diag) target[c++] = (g + d) % n;
  return c;
}

// Why this process cannot run cdprobe_ce_alltoall, empty when it can: the driver lacks a stream memory operation, or
// its local ranks would hold more streams on one device than the hardware queues CUDA_DEVICE_MAX_CONNECTIONS gives.
static std::string ce_a2a_refusal(cdprobe* h) {
  std::string err;
  if (h->drv.load_stream_wait(&err) != cudaSuccess || h->drv.load_stream_write(&err) != cudaSuccess)
    return "cdprobe_ce_alltoall: " + err;
  int ordinal[kMaxRanks], worst = 0;
  for (uint32_t li = 0; li < h->n_local; ++li) ordinal[li] = h->lr[li].ordinal;
  const uint32_t need = ce_a2a_queues(h->n_total, h->plan.diag, h->n_local, ordinal, &worst);
  if (need <= h->max_connections) return "";
  return "cdprobe_ce_alltoall: needs " + std::to_string(need) + " queues on ordinal " + std::to_string(worst) +
         ", CUDA_DEVICE_MAX_CONNECTIONS allows " + std::to_string(h->max_connections);
}

constexpr CopyCall kCeA2a = {
    "cdprobe_ce_alltoall", 8, kMeasCeAllToAll, 2,
    "the armed copy-engine all-to-all fault names no cell, size, word or delay of this call, or has a mode above 2",
    ce_a2a_refusal,
    "cdprobe_ce_alltoall: another process cannot run it (no stream memory operations, or more streams than "
    "CUDA_DEVICE_MAX_CONNECTIONS)"};

// The host block and the rep events (copy_setup), and every local rank's copy streams and their events, made on the
// first call and kept until close.
static int ce_a2a_setup(cdprobe* h) {
  if (const int rc = copy_setup(h); rc != CDPROBE_OK) return rc;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    LocalRank& L = h->lr[li];
    uint32_t target[kMaxRanks];
    const uint32_t cells = ce_a2a_targets(h, li, target);
    CDP_RT(cudaSetDevice(L.ordinal));
    for (uint32_t i = 0; i < cells; ++i) {
      if (L.cea_stream[i] == nullptr) CDP_RT(cudaStreamCreateWithFlags(&L.cea_stream[i], cudaStreamNonBlocking));
      for (uint32_t x = 0; x < 3; ++x)
        if (L.cea_copy_ev[i][x] == nullptr)
          CDP_RT(cudaEventCreateWithFlags(&L.cea_copy_ev[i][x], x < 2 ? cudaEventDefault : cudaEventDisableTiming));
    }
  }
  return CDPROBE_OK;
}

// Word `word` (0: opening, 1: landed) of `sender`'s line in `owner`'s flag lines, as local rank li maps them.
static CUdeviceptr ce_a2a_line(const cdprobe* h, uint32_t li, uint32_t owner, uint32_t sender, uint32_t word) {
  return h->mem.va[li][owner] + kCeA2aOff + (uint64_t)sender * sizeof(FlagLine) + 8ull * word;
}

// When the host gives up on a rep whose values are v: writes v into both words of every line of its own ranks, on a
// stream of its own, so that no stream of theirs is left waiting at close.  Best effort: it waits at most timeout_ms.
static void ce_a2a_unblock(cdprobe* h, uint64_t v) {
  CopyHost* const host = h->copy_host;
  host->release[0] = host->release[1] = v;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    LocalRank& L = h->lr[li];
    cudaStream_t s = nullptr;
    if (cudaSetDevice(L.ordinal) != cudaSuccess || cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess)
      continue;
    for (uint32_t j = 0; j < h->n_total; ++j)
      cudaMemcpyAsync(reinterpret_cast<void*>(ce_a2a_line(h, li, L.grank, j, 0)), host->release, 16,
                      cudaMemcpyHostToDevice, s);
    const double deadline = now_ms() + h->cfg.timeout_ms;
    while (cudaStreamQuery(s) == cudaErrorNotReady && now_ms() < deadline) {
    }
    cudaStreamDestroy(s);
  }
}

// Rep `rep` of size k of cdprobe_ce_alltoall on every local rank, all queued before the host releases the rep's
// ticket (DESIGN §5p): on each rank's stream the ticket wait, the opening barrier, event A, the joins of its copy
// streams (and on a push the landed values of every sender), event B; on each copy stream the wait for A, the copy
// between its two events, and on a push the landed value.  The ticket is released even when queuing fails.  Then the
// host waits until every B has completed (wait_reps), reads the times of a timed rep into rank_ns[li][k] and
// copy_ns[li][i][k], and only then queues the checks of every block each local rank owns, on its stream, so no kernel
// launch waits behind a stream that waits on the host.
static int ce_a2a_rep(cdprobe* h, uint32_t op, const Ladder& lad, uint32_t k, uint32_t rep, const CopyFault& f,
                      float (*rank_ns)[kBwMaxSizes][kMaxTimedReps],
                      float (*copy_ns)[kMaxRanks][kBwMaxSizes][kMaxTimedReps]) {
  CopyHost* const host = h->copy_host;
  const Plan& pl = h->plan;
  const uint32_t n = h->n_total;
  const bool push = op == CDPROBE_OP_WRITE;
  const uint64_t ticket = ++host->issued, bytes = lad.size[k];
  const uint64_t v = ce_a2a_value(h->meas[kMeasCeAllToAll].calls, k, rep, lad.reps);
  const auto wait_value = [&](cudaStream_t s, CUdeviceptr a, uint64_t want) {
    return h->drv.StreamWaitValue64(s, a, want, CU_STREAM_WAIT_VALUE_GEQ);
  };
  cudaError_t e = cudaSuccess;
  CUresult cu = CUDA_SUCCESS;
  const char* what = "";
  bool held = false;
  const auto ok = [&] { return e == cudaSuccess && cu == CUDA_SUCCESS; };
  for (uint32_t li = 0; li < h->n_local && ok(); ++li) {
    LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    const cudaStream_t s = L.stream;
    e = cudaSetDevice(L.ordinal);
    what = "cuStreamWaitValue64";
    if (ok()) cu = wait_value(s, reinterpret_cast<CUdeviceptr>(&host->ticket), ticket);
    what = "cuStreamWriteValue64";
    for (uint32_t p = 0; p < n && ok(); ++p)
      if (p != g) cu = h->drv.StreamWriteValue64(s, ce_a2a_line(h, li, p, g, 0), v, CU_STREAM_WRITE_VALUE_DEFAULT);
    what = "cuStreamWaitValue64";
    for (uint32_t p = 0; p < n && ok(); ++p)
      if (p != g) cu = wait_value(s, ce_a2a_line(h, li, g, p, 0), v);
    if (ok()) e = cudaEventRecord(L.rep_ev[2 * rep], s);
    uint32_t target[kMaxRanks];
    const uint32_t cells = ce_a2a_targets(h, li, target);
    for (uint32_t i = 0; i < cells && ok(); ++i) {
      const uint32_t j = target[i];
      const MemcpyCell c = memcpy_cell(pl, op, g, j);
      const bool armed = rep == 1 && k == f.k && g == f.issuer && j == f.target;
      const cudaStream_t cs = L.cea_stream[i];
      cudaEvent_t* const ev = L.cea_copy_ev[i];
      uint8_t* const dst = reinterpret_cast<uint8_t*>(h->area.va[li][c.dst_rank] + c.dst_off);
      e = cudaStreamWaitEvent(cs, L.rep_ev[2 * rep], 0);
      what = "cuStreamWaitValue64";
      if (ok() && armed && f.mode == 2) {
        cu = wait_value(cs, reinterpret_cast<CUdeviceptr>(&host->hold), ticket);
        held = true;
      }
      if (ok()) e = cudaEventRecord(ev[0], cs);
      if (ok() && !(armed && f.mode == 1))
        e = cudaMemcpyAsync(dst, reinterpret_cast<const void*>(h->mem.va[li][c.src_rank] + c.src_off), bytes,
                            cudaMemcpyDeviceToDevice, cs);
      if (ok()) e = cudaEventRecord(ev[1], cs);
      if (ok() && armed && f.mode == 0) e = store_flip(h, li, c, f.arg, cs);
      what = "cuStreamWriteValue64";
      if (ok() && push) cu = h->drv.StreamWriteValue64(cs, ce_a2a_line(h, li, j, g, 1), v, CU_STREAM_WRITE_VALUE_DEFAULT);
      if (ok()) e = cudaEventRecord(ev[2], cs);
      if (ok()) e = cudaStreamWaitEvent(s, ev[2], 0);
    }
    what = "cuStreamWaitValue64";
    for (uint32_t p = 0; p < n && push && ok(); ++p)
      if (p != g || pl.diag) cu = wait_value(s, ce_a2a_line(h, li, g, p, 1), v);
    if (ok()) e = cudaEventRecord(L.rep_ev[2 * rep + 1], s);
  }
  __atomic_store_n(&host->ticket, ticket, __ATOMIC_RELEASE);
  if (held) usleep((useconds_t)f.arg);
  __atomic_store_n(&host->hold, ticket, __ATOMIC_RELEASE);
  if (!ok()) {
    ce_a2a_unblock(h, v);
    if (e != cudaSuccess) return fail_sticky(h, "cdprobe_ce_alltoall: queue a rep", e);
    h->sticky = true;
    set_err(std::string("cdprobe_ce_alltoall: ") + what + ": " + h->drv.error_name(cu));
    return CDPROBE_ERR_CUDA;
  }
  if (const int rc = wait_reps(h, (1u << h->n_local) - 1u, rep, "cdprobe_ce_alltoall: wait for a rep",
                               "cdprobe_ce_alltoall: a rep did not complete within timeout_ms of its release");
      rc != CDPROBE_OK) {
    if (rc == CDPROBE_ERR_TIMEOUT) ce_a2a_unblock(h, v);
    return rc;
  }
  for (uint32_t li = 0; li < h->n_local && rep > 0; ++li) {
    LocalRank& L = h->lr[li];
    uint32_t target[kMaxRanks];
    const uint32_t cells = ce_a2a_targets(h, li, target);
    float ms = 0.f;
    CDP_RT(cudaSetDevice(L.ordinal));
    if ((e = cudaEventElapsedTime(&ms, L.rep_ev[2 * rep], L.rep_ev[2 * rep + 1])) != cudaSuccess)
      return fail_sticky(h, "cdprobe_ce_alltoall: event times", e);
    rank_ns[li][k][rep - 1] = ms * 1e6f;
    for (uint32_t i = 0; i < cells; ++i) {
      if ((e = cudaEventElapsedTime(&ms, L.cea_copy_ev[i][0], L.cea_copy_ev[i][1])) != cudaSuccess)
        return fail_sticky(h, "cdprobe_ce_alltoall: event times", e);
      copy_ns[li][i][k][rep - 1] = ms * 1e6f;
    }
  }
  // every block in rank g's area holds the slice g reads from its sender j, whichever side copied it
  for (uint32_t li = 0; li < h->n_local && e == cudaSuccess; ++li) {
    const uint32_t g = h->lr[li].grank;
    e = cudaSetDevice(h->lr[li].ordinal);
    for (uint32_t j = 0; j < n && e == cudaSuccess; ++j)
      if (j != g || pl.diag) e = check_block(h, li, memcpy_cell(pl, CDPROBE_OP_READ, g, j), bytes, &host->rep[li][j][rep]);
  }
  return e != cudaSuccess ? fail_sticky(h, "cdprobe_ce_alltoall: queue the checks", e) : CDPROBE_OK;
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
  const uint8_t* region = reinterpret_cast<const uint8_t*>(h->mem.va[reader - h->first][target]) + out->region_offset;
  cdp::DiagOut d;
  float ms = 0.f;
  cudaError_t e = cudaEventRecord(L.ev0, L.stream);
  if (e == cudaSuccess) e = (cudaError_t)cdp::diag_launch(region, s, L.scratch, L.sm_count, L.stream);
  if (e == cudaSuccess) e = cudaEventRecord(L.ev1, L.stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&d, L.scratch, sizeof(d), cudaMemcpyDeviceToHost, L.stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(L.stream);
  if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, L.ev0, L.ev1);
  if (e != cudaSuccess) return cdp::fail_sticky(h, "cdprobe_diagnose", e);
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
  if (!cdp::begin_output(out)) return CDPROBE_ERR_ARG;
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
  if (const int rc = cdp::ensure_scratch_all(h, cdp::kRepTableBytes); rc != CDPROBE_OK) return rc;

  // 1. every local issuer's chases, all launched before any is waited for
  cdp::LatencyParams P[cdp::kMaxRanks];
  cdp::RepCells cells[cdp::kMaxRanks];
  for (uint32_t li = 0; li < h->n_local; ++li) {
    cdp::LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    out->row_mask |= 1u << g;
    cdp::LatencyParams& p = P[li];
    memset(&p, 0, sizeof(p));
    p.seed = h->seed;
    p.timeout_ns = cdp::timeout_ns(h);
    p.hops = hops;
    p.reps = reps;
    for (uint32_t j = 0; j < h->n_total; ++j) {
      if (!cdp::live_cell(h, li, j, out->status)) continue;
      cells[li].add(p.n_cells, g * CDPROBE_MAX_GPUS + j);
      cdp::LatencyCell& c = p.cell[p.n_cells++];
      c.region = reinterpret_cast<const uint8_t*>(h->mem.va[li][j]) + cdp::cell_offset(pl, CDPROBE_OP_READ, g, j);
      c.lines = lines;
      c.issuer = g;
      c.target = j;
    }
    if (p.n_cells == 0) continue;
    CDP_RT(cudaSetDevice(L.ordinal));
    const cudaError_t e = (cudaError_t)cdp::latency_launch(p, static_cast<cdp::TimedRep*>(L.scratch), L.stream);
    if (e != cudaSuccess) return cdp::fail_sticky(h, "launch latency_kernel", e);
  }

  // 2. while they run: the digest each chase gives over an intact region
  for (uint32_t li = 0; li < h->n_local; ++li) {
    for (uint32_t k = 0; k < P[li].n_cells; ++k) {
      const cdp::LatencyCell& c = P[li].cell[k];
      const uint64_t first = (uint64_t)cdp::cell_slice(pl, c.issuer, c.target) * (pl.bpp / 8);
      for (uint32_t r = 0; r <= reps; ++r)
        cells[li].want[k] ^= cdp::latency_rep_digest(h->seed, c.issuer, c.target, first, lines, r, hops);
    }
  }

  // 3. collect: ns per hop of the timed reps, the digest of all of them
  if (const int rc = cdp::collect_reps(h, cells, reps, hops, "cdprobe_latency", out); rc != CDPROBE_OK) return rc;
  out->ms = cdp::now_ms() - t_begin;
  return CDPROBE_OK;
}

int cdprobe_pingpong(cdprobe_t* h, uint32_t trips, uint32_t reps, uint32_t fenced, cdprobe_pingpong_t* out) {
  if (!cdp::begin_output(out)) return CDPROBE_ERR_ARG;
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
  cdp::MeasRecord& rec = h->meas[cdp::kMeasPingPong];
  uint32_t f_init = cdp::kPingPongNoFault, f_target = cdp::kPingPongNoFault, f_trip = cdp::kPingPongNoFault;
  if (rec.fault != 0) {
    const uint64_t fi = rec.fault >> 32, ft = (rec.fault >> 16) & 0xffffu, trip = rec.fault & 0xffffu;
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
  // every process runs over the same pair set: the domain's mapping status, from every process's rows
  int32_t st[cdp::kMaxRanks][cdp::kMaxRanks];
  if (const int rc = cdp::agree(h, "cdprobe_pingpong", bad, rec.calls + 1, {trips, reps, fenced}, st); rc != CDPROBE_OK)
    return rc;
  out->call_seq = ++rec.calls;
  for (uint32_t li = 0; li < h->n_local; ++li) out->row_mask |= 1u << h->lr[li].grank;
  if (n == 1) {
    out->ms = cdp::now_ms() - t_begin;
    return CDPROBE_OK;
  }
  // every process has agreed before any kernel polls a peer
  if (const int rc = cdp::domain_barrier(h); rc != CDPROBE_OK) return rc;
  if (const int rc = cdp::ensure_scratch_all(h, cdp::kRepTableBytes); rc != CDPROBE_OK) return rc;
  // a pair is exchanged only when both directions are mapped; the status of its cells is the pair's mapping status
  auto pair_status = [&](uint32_t i, uint32_t j) { return st[i][j] != 0 ? st[i][j] : st[j][i]; };

  // 2. one block per local rank, every one launched before any is waited for
  cdp::PingPongParams P[cdp::kMaxRanks];
  cdp::RepCells cells[cdp::kMaxRanks];
  for (uint32_t li = 0; li < h->n_local; ++li) {
    cdp::LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    cdp::PingPongParams& p = P[li];
    memset(&p, 0, sizeof(p));
    p.call_seq = rec.calls;
    p.timeout_ns = cdp::timeout_ns(h);
    p.n_rounds = pl.rounds;
    p.trips = trips;
    p.reps = reps;
    p.fault_round = cdp::kPingPongNoFault;
    p.fault_trip = f_trip;
    for (uint32_t j = 0; j < n; ++j)
      if (j != g) out->status[g * CDPROBE_MAX_GPUS + j] = pair_status(g, j);
    for (uint32_t r = 0; r < pl.rounds; ++r) {
      const int q = pl.partner[r][g];
      if (q < 0 || pair_status(g, (uint32_t)q) != 0) continue;
      cdp::PingPongRound& R = p.round[r];
      R.remote = reinterpret_cast<uint64_t*>(h->mem.va[li][q] + cdp::kPingOff + (uint64_t)g * sizeof(cdp::FlagLine));
      R.local =
          reinterpret_cast<const uint64_t*>(h->mem.va[li][g] + cdp::kPingOff + (uint64_t)q * sizeof(cdp::FlagLine));
      R.partner = (uint32_t)q;
      R.first = g < (uint32_t)q ? 1u : 0u;
      if (g == f_target && (uint32_t)q == f_init) p.fault_round = r;
      cells[li].add(r, g * CDPROBE_MAX_GPUS + (uint32_t)q);
    }
    if (cells[li].n == 0) continue;
    CDP_RT(cudaSetDevice(L.ordinal));
    const cudaError_t e =
        (cudaError_t)cdp::pingpong_launch(p, fenced != 0, static_cast<cdp::TimedRep*>(L.scratch), L.stream);
    if (e != cudaSuccess) return cdp::fail_sticky(h, "launch pingpong_kernel", e);
  }

  // 3. while they run: the digest of a clean leg for every cell a local rank initiates
  for (uint32_t li = 0; li < h->n_local; ++li) {
    cdp::RepCells& c = cells[li];
    for (uint32_t k = 0; k < c.n; ++k) {
      const uint32_t leg = P[li].round[c.slot[k]].first ? 0u : 1u;
      for (uint32_t rep = 0; rep <= reps; ++rep)
        c.want[k] ^= cdp::pingpong_rep_digest(rec.calls, c.slot[k], leg, rep, trips);
    }
  }

  // 4. collect: ns per round trip of the timed reps, the digest of all of them
  if (const int rc = cdp::collect_reps(h, cells, reps, trips, "cdprobe_pingpong", out); rc != CDPROBE_OK) return rc;
  out->ms = cdp::now_ms() - t_begin;
  return CDPROBE_OK;
}

int cdprobe_atomics(cdprobe_t* h, uint32_t kind, uint32_t ops, uint32_t reps, cdprobe_atomics_t* out) {
  if (!cdp::begin_output(out)) return CDPROBE_ERR_ARG;
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
  cdp::MeasRecord& rec = h->meas[cdp::kMeasAtomics];
  uint32_t f_issuer = cdp::kMaxRanks, f_target = cdp::kMaxRanks;
  if (rec.fault != 0) {
    const uint64_t fi = rec.fault >> 16, ft = rec.fault & 0xffffu;
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
  if (const int rc = cdp::ensure_scratch_all(h, cdp::kRepTableBytes); rc != CDPROBE_OK) return rc;
  out->call_seq = ++rec.calls;

  // 1. every local issuer's cells, all launched before any is waited for; no kernel waits on another rank
  cdp::AtomicsParams P[cdp::kMaxRanks];
  cdp::RepCells cells[cdp::kMaxRanks];
  for (uint32_t li = 0; li < h->n_local; ++li) {
    cdp::LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    out->row_mask |= 1u << g;
    cdp::AtomicsParams& p = P[li];
    memset(&p, 0, sizeof(p));
    p.call_seq = rec.calls;
    p.timeout_ns = cdp::timeout_ns(h);
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
      if (!cdp::live_cell(h, li, j, out->status)) continue;
      if (native == 0) {
        out->status[idx] = CDPROBE_ERR_UNSUPPORTED;
        continue;
      }
      if (g == f_issuer && j == f_target) p.fault_cell = p.n_cells;
      cells[li].add(p.n_cells, idx);
      cdp::AtomicsCell& c = p.cell[p.n_cells++];
      c.word =
          reinterpret_cast<unsigned long long*>(h->mem.va[li][j] + cdp::kAtomOff + (uint64_t)g * sizeof(cdp::AtomLine));
      c.issuer = g;
      c.target = j;
    }
    if (p.n_cells == 0) continue;
    CDP_RT(cudaSetDevice(L.ordinal));
    const cudaError_t e = (cudaError_t)cdp::atomics_launch(p, kind, static_cast<cdp::TimedRep*>(L.scratch), L.stream);
    if (e != cudaSuccess) return cdp::fail_sticky(h, "launch atomics kernel", e);
  }

  // 2. while they run: the digest of clean reps, the same for every cell
  uint64_t want = 0;
  for (uint32_t r = 0; r <= reps; ++r) want ^= cdp::atomics_rep_digest(cdp::atomics_start(rec.calls, kind, r), total);
  for (cdp::RepCells& c : cells) std::fill(c.want, c.want + c.n, want);

  // 3. collect: ns per atomic of the timed reps, the digest of all of them
  if (const int rc = cdp::collect_reps(h, cells, reps, (uint32_t)total, "cdprobe_atomics", out); rc != CDPROBE_OK)
    return rc;
  out->ms = cdp::now_ms() - t_begin;
  return CDPROBE_OK;
}

int cdprobe_bwcurve(cdprobe_t* h, uint32_t reps, cdprobe_bwcurve_t* out) {
  cdp::Ladder lad;
  if (const int rc = cdp::open_ladder(h, out, reps, cdp::kBwDefaultReps, &lad); rc != CDPROBE_OK) return rc;
  const cdp::Plan& pl = h->plan;
  const uint32_t n = h->n_total;
  // 1. the arguments; in a multi-process domain the verdict is shared below, so every process refuses together.  Every
  //    cell is one-sided and the rounds come from the plan, which all processes share, so nothing else must agree
  cdp::MeasRecord& rec = h->meas[cdp::kMeasBwCurve];
  if (const int rc = cdp::agree(h, "cdprobe_bwcurve", lad.bad, rec.calls + 1, {lad.reps, 0u, 0u}, nullptr);
      rc != CDPROBE_OK)
    return rc;
  out->call_seq = ++rec.calls;
  cdp::put_ladder(h, lad, out);

  // 2. which cells run; scratch for the rep records and one cell's granule table, grown on every local rank before any
  //    kernel runs, and the (S, X) each size of each cell that runs must read, from the pattern definition
  bool runs[cdp::kMaxRanks][cdp::kMaxRanks] = {};
  for (uint32_t li = 0; li < h->n_local; ++li)
    for (uint32_t j = 0; j < n; ++j) runs[li][j] = cdp::live_cell(h, li, j, out->status);
  const size_t table_off = (sizeof(cdp::BwScratch) + 255) / 256 * 256;
  std::unique_ptr<cdp::CellSums[]> want;
  if (const int rc = cdp::cell_sums(h, runs, CDPROBE_OP_READ, table_off, lad, "cdprobe_bwcurve: granule checksums",
                                    &want);
      rc != CDPROBE_OK)
    return rc;

  // 3. the rounds: every local kernel of a round is launched before any is waited for
  auto got = std::make_unique<cdp::BwScratch>();
  const auto round = [&](const int32_t* target) -> int {
    for (uint32_t li = 0; li < h->n_local; ++li) {
      if (target[li] < 0) continue;
      cdp::LocalRank& L = h->lr[li];
      const uint32_t q = (uint32_t)target[li];
      cdp::BwCurveParams p;
      memset(&p, 0, sizeof(p));
      p.region = reinterpret_cast<const uint8_t*>(h->mem.va[li][q]) + cdp::cell_offset(pl, CDPROBE_OP_READ, L.grank, q);
      if (const int rc = cdp::launch_ladder(h, L, p, lad, cdp::bwcurve_launch, "launch bwcurve_kernel");
          rc != CDPROBE_OK)
        return rc;
    }
    for (uint32_t li = 0; li < h->n_local; ++li) {
      if (target[li] < 0) continue;
      cdp::LocalRank& L = h->lr[li];
      if (const int rc = cdp::fetch_reps(h, L, got.get(), 1, "cdprobe_bwcurve"); rc != CDPROBE_OK) return rc;
      cdp::bw_summarize(*got, want[li][target[li]], lad.size, lad.n_sizes, lad.reps,
                        L.grank * CDPROBE_MAX_GPUS + (uint32_t)target[li], out);
    }
    return CDPROBE_OK;
  };
  if (const int rc = cdp::walk_rounds(h, runs, round); rc != CDPROBE_OK) return rc;
  out->ms = cdp::now_ms() - lad.t_begin;
  return CDPROBE_OK;
}

int cdprobe_allreduce(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out) {
  return cdp::allreduce_call(h, reps, out, cdp::kOneShot);
}

int cdprobe_allreduce_twoshot(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out) {
  return cdp::allreduce_call(h, reps, out, cdp::kTwoShot);
}

int cdprobe_allreduce_ll(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out) {
  return cdp::allreduce_call(h, reps, out, cdp::kLl);
}

int cdprobe_allreduce_ring(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out) {
  return cdp::allreduce_call(h, reps, out, cdp::kRing);
}

int cdprobe_allreduce_push(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out) {
  return cdp::allreduce_call(h, reps, out, cdp::kPush);
}

int cdprobe_allreduce_nvls(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out) {
  return cdp::allreduce_call(h, reps, out, cdp::kNvls);
}

int cdprobe_alltoall(cdprobe_t* h, uint32_t reps, cdprobe_alltoall_t* out) {
  cdp::Ladder lad;
  if (const int rc = cdp::open_ladder(h, out, reps, cdp::kA2aDefaultReps, &lad); rc != CDPROBE_OK) return rc;
  const cdp::Plan& pl = h->plan;
  const uint32_t n = h->n_total;
  // 1. the arguments, the armed fault and the probe mapping rows; in a multi-process domain all three are shared, so
  //    every process refuses or runs together over the same cells
  uint32_t f_send = cdp::kA2aNoFault, f_recv = cdp::kA2aNoFault, f_k = cdp::kA2aNoFault;
  uint64_t f_word = 0;
  cdp::MeasRecord& rec = h->meas[cdp::kMeasAllToAll];
  if (rec.fault != 0 && lad.bad.empty()) {
    const uint64_t fs = rec.fault >> 40, fr = (rec.fault >> 32) & 0xffu;
    const cdp::FaultSpot at = cdp::fault_spot(rec.fault, lad);
    f_word = at.word;
    if (fs == 0 || fs > n || fr == 0 || fr > n || (fs == fr && !pl.diag) || !at.word_ok) {
      lad.bad = "the armed all-to-all fault names no cell, size or word of this call";
    } else {
      f_send = (uint32_t)fs - 1;
      f_recv = (uint32_t)fr - 1;
      f_k = at.k;
    }
  }
  int32_t st[cdp::kMaxRanks][cdp::kMaxRanks];
  if (const int rc = cdp::agree(h, "cdprobe_alltoall", lad.bad, rec.calls + 1, {lad.reps, 0u, 0u}, st);
      rc != CDPROBE_OK)
    return rc;
  // 2. the exchange area, built once, by every process in the same call
  if (const int rc = cdp::ensure_area(h, h->area, (size_t)n * pl.bpp); rc != CDPROBE_OK) return rc;
  out->call_seq = ++rec.calls;
  out->area_bytes = h->area.bytes;
  cdp::put_ladder(h, lad, out);

  // 3. which cells run: st[s][d], the probe mapping status of sender s's cell to receiver d, or else its exchange-area
  //    mapping status; 0 runs.  Every process derives the same matrix.
  cdp::fold_area_status(h, h->area, st);
  bool any = false;
  for (uint32_t s = 0; s < n; ++s) {
    for (uint32_t d = 0; d < n; ++d) {
      if (s == d && !pl.diag) st[s][d] = CDPROBE_ERR_ARG;  // no such cell
      any |= st[s][d] == 0;
    }
  }
  auto runs = [&](uint32_t s, uint32_t d) { return st[s][d] == 0; };
  const bool local_fault = f_send >= h->first && f_send < h->first + h->n_local;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    const uint32_t g = h->lr[li].grank;
    for (uint32_t j = 0; j < n; ++j) {
      if (j == g && !pl.diag) continue;
      if (!runs(g, j)) out->cell_status[g * CDPROBE_MAX_GPUS + j] = st[g][j];
      if (!runs(j, g)) out->cell_status[j * CDPROBE_MAX_GPUS + g] = st[j][g];
    }
  }
  if (!any) {  // e.g. MIG instances: nothing to exchange anywhere, so no kernel is launched in any process
    out->ms = cdp::now_ms() - lad.t_begin;
    return CDPROBE_OK;
  }

  // 4. the records, grown on every local rank; then no process launches before every process is ready, and every local
  //    kernel is launched before any is waited for
  if (const int rc = cdp::ensure_scratch_all(h, sizeof(cdp::A2aScratch)); rc != CDPROBE_OK) return rc;
  if (const int rc = cdp::domain_barrier(h); rc != CDPROBE_OK) return rc;
  bool launched[cdp::kMaxRanks] = {};
  for (uint32_t li = 0; li < h->n_local; ++li) {
    cdp::LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    const CUdeviceptr* va = h->mem.va[li];
    cdp::AllToAllParams p;
    memset(&p, 0, sizeof(p));
    // the barrier: with every rank a cell joins to this one; rank j pushes to this rank when it maps it, else this
    // rank polls line j of j's own memory through its own mapping
    bool joined = runs(g, g);
    for (uint32_t j = 0; j < n; ++j) {
      if (j == g || !(runs(g, j) || runs(j, g))) continue;
      joined = true;
      if (runs(g, j))
        p.dom.sig_out[j] = reinterpret_cast<uint64_t*>(va[j] + cdp::kA2aOff + (uint64_t)g * sizeof(cdp::FlagLine));
      p.dom.sig_in[j] = reinterpret_cast<const uint64_t*>(
          runs(j, g) ? va[g] + cdp::kA2aOff + (uint64_t)j * sizeof(cdp::FlagLine)
                     : va[j] + cdp::kA2aOff + (uint64_t)j * sizeof(cdp::FlagLine));
    }
    if (!joined) continue;
    p.dom.self = reinterpret_cast<uint64_t*>(va[g] + cdp::kA2aOff + (uint64_t)g * sizeof(cdp::FlagLine));
    p.dom.call_seq = rec.calls;
    // the blocks, in the order rank + 1, rank + 2, ... (mod n), then the diagonal
    p.fault_k = cdp::kA2aNoFault;
    for (uint32_t d = 1; d <= n; ++d) {
      const uint32_t j = (g + d) % n;
      if (!runs(g, j)) continue;
      if (local_fault && g == f_send && j == f_recv) {
        p.fault_k = f_k;
        p.fault_block = p.blocks;
        p.fault_word = f_word;
      }
      p.to[p.blocks] = j;
      p.dst[p.blocks++] = reinterpret_cast<uint8_t*>(h->area.va[li][j]) + (uint64_t)g * pl.bpp;
    }
    for (uint32_t s = 0; s < n; ++s) {
      if (!runs(s, g)) continue;
      p.from[p.n_in] = s;
      p.in[p.n_in++] = reinterpret_cast<const uint8_t*>(h->area.va[li][g]) + (uint64_t)s * pl.bpp;
    }
    p.seed = h->seed;
    p.rank = g;
    out->blocks[g] = p.blocks;
    if (const int rc = cdp::launch_ladder(h, L, p, lad, cdp::alltoall_launch, "launch alltoall_kernel");
        rc != CDPROBE_OK)
      return rc;
    launched[li] = true;
  }

  // 5. collect: per rank, the egress times; per cell it receives, the word checks and the last rep's (S, X)
  auto got = std::make_unique<cdp::A2aScratch>();
  for (uint32_t li = 0; li < h->n_local; ++li) {
    if (!launched[li]) continue;
    cdp::LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    if (const int rc = cdp::fetch_reps(h, L, got.get(), 1, "cdprobe_alltoall"); rc != CDPROBE_OK) return rc;
    const cdp::A2aScratch& s = *got;
    const bool timed = cdp::bw_times(s.rep, lad.size, lad.n_sizes, lad.reps, (double)out->blocks[g], g, out);
    for (uint32_t i = 0; i < n; ++i) {
      if (!runs(i, g)) continue;
      const uint32_t cell = i * CDPROBE_MAX_GPUS + g;
      out->cell_measured[cell] = 1;
      if (!timed) {
        out->cell_status[cell] = CDPROBE_ERR_TIMEOUT;
        continue;
      }
      for (uint32_t k = 0; k < lad.n_sizes; ++k) {
        out->sum[cell][k] = s.sum[i][k];
        out->xr[cell][k] = s.xr[i][k];
      }
      cdp::word_checks(s.bad_words[i], s.first_bad_n[i], lad.n_sizes, cell, &out->cell_status[cell], out);
    }
  }
  out->ms = cdp::now_ms() - lad.t_begin;
  return CDPROBE_OK;
}

int cdprobe_memcpy(cdprobe_t* h, uint32_t op, uint32_t reps, cdprobe_memcpy_t* out) {
  // 1-2. the arguments, the armed fault and the probe mapping rows, shared in a multi-process domain so that every
  //      process refuses or runs together over the same rounds; then the exchange area
  cdp::Ladder lad;
  cdp::CopyFault f;
  int32_t st[cdp::kMaxRanks][cdp::kMaxRanks];
  if (const int rc = cdp::open_copy(h, cdp::kMemcpy, op, reps, out, &lad, &f, st); rc != CDPROBE_OK) return rc;
  const cdp::Plan& pl = h->plan;
  const uint32_t n = h->n_total;

  // 3. which cells run: the issuer maps the target's probe allocation and exchange area (cdprobe_alltoall's rule);
  //    whether any cell of the domain runs, from the status every process shares
  cdp::fold_area_status(h, h->area, st);
  bool any = false;
  for (uint32_t s = 0; s < n; ++s)
    for (uint32_t d = 0; d < n; ++d) any |= (s != d || pl.diag) && st[s][d] == 0;
  bool runs[cdp::kMaxRanks][cdp::kMaxRanks] = {};
  for (uint32_t li = 0; li < h->n_local; ++li) {
    const cdp::LocalRank& L = h->lr[li];
    const uint32_t g = L.grank;
    for (uint32_t j = 0; j < n; ++j) {
      if (!cdp::live_cell(h, li, j, out->status)) continue;
      const int32_t s = h->area.status[g][j], a = s == 0 && !h->area.mapped[li][j] ? cdp::kStatusUnmapped : s;
      if (a != 0) out->status[g * CDPROBE_MAX_GPUS + j] = a;
      runs[li][j] = a == 0;
    }
  }
  if (!any) {  // e.g. MIG instances: nothing to copy anywhere, so nothing is queued in any process
    out->ms = cdp::now_ms() - lad.t_begin;
    return CDPROBE_OK;
  }

  // 4. the driver's stream wait, the host block and the events; scratch for the checks and one cell's granule table,
  //    grown on every local rank before anything is queued; the (S, X) each size of each cell must land, from the
  //    pattern definition: the per-granule sums of the source slice on the issuer's GPU, folded into every prefix on
  //    the host.  A driver without the stream wait is refused here, by this process alone (DESIGN §5n)
  if (std::string err; h->drv.load_stream_wait(&err) != cudaSuccess) {
    cdp::set_err("cdprobe_memcpy: " + err);
    return CDPROBE_ERR_UNSUPPORTED;
  }
  if (const int rc = cdp::copy_setup(h); rc != CDPROBE_OK) return rc;
  std::unique_ptr<cdp::CellSums[]> want;
  if (const int rc = cdp::cell_sums(h, runs, op, cdp::MemcpyScratch(pl.bpp).table_off, lad,
                                    "cdprobe_memcpy: granule checksums", &want);
      rc != CDPROBE_OK)
    return rc;

  // 5. the rounds.  No process starts a size before every process has finished the one before; within a size, one rep
  //    at a time on every local rank at once.  After a size, every local stream is drained, and the checks' records
  //    and the events are read: per rep, the diagnosis's bad words and the (S, X) read against the pattern's
  auto ns = std::make_unique<float[][cdp::kBwMaxSizes][cdp::kMaxTimedReps]>(cdp::kMaxRanks);
  const auto round = [&](const int32_t* target) -> int {
    bool local = false, aborted[cdp::kMaxRanks] = {};
    for (uint32_t li = 0; li < h->n_local; ++li) local |= target[li] >= 0;
    for (uint32_t k = 0; k < lad.n_sizes; ++k) {
      if (const int rc = cdp::domain_barrier(h); rc != CDPROBE_OK) return rc;
      if (!local) continue;
      for (uint32_t rep = 0; rep <= lad.reps; ++rep)
        if (const int rc = cdp::memcpy_rep(h, target, op, lad, k, rep, f); rc != CDPROBE_OK) return rc;
      for (uint32_t li = 0; li < h->n_local; ++li) {
        if (target[li] < 0) continue;
        const cdp::LocalRank& L = h->lr[li];
        const uint32_t j = (uint32_t)target[li], idx = L.grank * CDPROBE_MAX_GPUS + j;
        CDP_RT(cudaSetDevice(L.ordinal));
        if (const cudaError_t e = cudaStreamSynchronize(L.stream); e != cudaSuccess)
          return cdp::fail_sticky(h, "cdprobe_memcpy: check a size", e);
        for (uint32_t rep = 1; rep <= lad.reps; ++rep) {
          float ms_rep = 0.f;
          const cudaError_t e = cudaEventElapsedTime(&ms_rep, L.rep_ev[2 * rep], L.rep_ev[2 * rep + 1]);
          if (e != cudaSuccess) return cdp::fail_sticky(h, "cdprobe_memcpy: event times", e);
          ns[li][k][rep - 1] = ms_rep * 1e6f;
        }
        aborted[li] |= cdp::fold_checks(h->copy_host->rep[li][j], lad.reps, k, want[li][j][k], idx, out);
      }
    }
    // per cell: the times, unless an (S, X) read passed its deadline, and the verdict of every size's checks
    for (uint32_t li = 0; li < h->n_local; ++li) {
      if (target[li] < 0) continue;
      const uint32_t idx = h->lr[li].grank * CDPROBE_MAX_GPUS + (uint32_t)target[li];
      out->measured[idx] = 1;
      if (!aborted[li]) cdp::ladder_times(ns[li], lad.size, lad.n_sizes, lad.reps, 1.0, idx, out);
      out->status[idx] = cdp::copy_verdict(aborted[li], out->bad_sizes[idx]);
    }
    return CDPROBE_OK;
  };
  if (const int rc = cdp::walk_rounds(h, runs, round); rc != CDPROBE_OK) return rc;
  out->ms = cdp::now_ms() - lad.t_begin;
  return CDPROBE_OK;
}

int cdprobe_ce_alltoall(cdprobe_t* h, uint32_t op, uint32_t reps, cdprobe_ce_alltoall_t* out) {
  // 1-2. the arguments, the armed fault, the probe mapping rows and whether every process can run it, shared in a
  //      multi-process domain so that every process refuses, skips or runs together; then the exchange area
  cdp::Ladder lad;
  cdp::CopyFault f;
  int32_t st[cdp::kMaxRanks][cdp::kMaxRanks];
  if (const int rc = cdp::open_copy(h, cdp::kCeA2a, op, reps, out, &lad, &f, st); rc != CDPROBE_OK) return rc;
  const cdp::Plan& pl = h->plan;
  const uint32_t n = h->n_total;
  const bool push = op == CDPROBE_OP_WRITE;

  // 3. every rank signals every other and every cell copies in every rep: when some probe or exchange-area mapping of
  //    the domain is down, nothing runs, in any process (a stream barrier cannot skip a peer)
  cdp::fold_area_status(h, h->area, st);
  if (const int32_t* down = cdp::first_down(st); down != nullptr) {
    for (uint32_t li = 0; li < h->n_local; ++li) {
      const uint32_t g = h->lr[li].grank;
      out->status[g] = *down;
      for (uint32_t j = 0; j < n; ++j) {
        if (j == g && !pl.diag) continue;
        out->cell_status[g * CDPROBE_MAX_GPUS + j] = *down;
        out->cell_status[j * CDPROBE_MAX_GPUS + g] = *down;
      }
    }
    out->ms = cdp::now_ms() - lad.t_begin;
    return CDPROBE_OK;
  }

  // 4. the host block, the copy streams and the events; scratch for the checks and one block's granule table, grown on
  //    every local rank before anything is queued; the (S, X) each size of each block a local rank owns must have,
  //    from the pattern definition: block j of rank g's area holds the slice g reads from j, on a pull and on a push
  if (const int rc = cdp::ce_a2a_setup(h); rc != CDPROBE_OK) return rc;
  bool owns[cdp::kMaxRanks][cdp::kMaxRanks] = {};
  for (uint32_t li = 0; li < h->n_local; ++li)
    for (uint32_t j = 0; j < n; ++j) owns[li][j] = j != h->lr[li].grank || pl.diag;
  std::unique_ptr<cdp::CellSums[]> want;
  if (const int rc = cdp::cell_sums(h, owns, CDPROBE_OP_READ, cdp::MemcpyScratch(pl.bpp).table_off, lad,
                                    "cdprobe_ce_alltoall: granule checksums", &want);
      rc != CDPROBE_OK)
    return rc;

  // 5. the sizes, each behind a domain barrier; within a size, one rep at a time, every rank and cell at once, each rep
  //    behind the checks of the one before.  After a size, every local stream is drained and the checks' records read:
  //    per rep, the diagnosis's bad words and the (S, X) read against the pattern's
  auto rank_ns = std::make_unique<float[][cdp::kBwMaxSizes][cdp::kMaxTimedReps]>(cdp::kMaxRanks);
  auto copy_ns = std::make_unique<float[][cdp::kMaxRanks][cdp::kBwMaxSizes][cdp::kMaxTimedReps]>(cdp::kMaxRanks);
  bool aborted[cdp::kMaxRanks][cdp::kMaxRanks] = {};
  for (uint32_t k = 0; k < lad.n_sizes; ++k) {
    if (const int rc = cdp::domain_barrier(h); rc != CDPROBE_OK) return rc;
    for (uint32_t rep = 0; rep <= lad.reps; ++rep)
      if (const int rc = cdp::ce_a2a_rep(h, op, lad, k, rep, f, rank_ns.get(), copy_ns.get()); rc != CDPROBE_OK)
        return rc;
    for (uint32_t li = 0; li < h->n_local; ++li) {
      const cdp::LocalRank& L = h->lr[li];
      const uint32_t g = L.grank;
      CDP_RT(cudaSetDevice(L.ordinal));
      if (const cudaError_t e = cudaStreamSynchronize(L.stream); e != cudaSuccess)
        return cdp::fail_sticky(h, "cdprobe_ce_alltoall: check a size", e);
      for (uint32_t j = 0; j < n; ++j) {
        if (!owns[li][j]) continue;
        const uint32_t idx = push ? j * CDPROBE_MAX_GPUS + g : g * CDPROBE_MAX_GPUS + j;
        aborted[li][j] |= cdp::fold_checks(h->copy_host->rep[li][j], lad.reps, k, want[li][j][k], idx, out);
      }
    }
  }

  // 6. per rank, the times of its reps (rate: blocks x size / ns); per cell it issues, the median copy time; per block
  //    it owns, the verdict of every size's checks, unless an (S, X) read passed its deadline
  for (uint32_t li = 0; li < h->n_local; ++li) {
    const uint32_t g = h->lr[li].grank;
    uint32_t target[cdp::kMaxRanks];
    const uint32_t cells = cdp::ce_a2a_targets(h, li, target);
    for (uint32_t i = 0; i < cells; ++i) {
      for (uint32_t k = 0; k < lad.n_sizes; ++k) {
        float* const t = copy_ns[li][i][k];
        std::sort(t, t + lad.reps);
        out->copy_ns_median[g * CDPROBE_MAX_GPUS + target[i]][k] = t[lad.reps / 2];
      }
    }
    out->measured[g] = 1;
    out->blocks[g] = cells;
    cdp::ladder_times(rank_ns[li], lad.size, lad.n_sizes, lad.reps, (double)cells, g, out);
    for (uint32_t j = 0; j < n; ++j) {
      if (!owns[li][j]) continue;
      const uint32_t idx = push ? j * CDPROBE_MAX_GPUS + g : g * CDPROBE_MAX_GPUS + j;
      out->cell_measured[idx] = 1;
      out->cell_status[idx] = cdp::copy_verdict(aborted[li][j], out->bad_sizes[idx]);
    }
  }
  out->ms = cdp::now_ms() - lad.t_begin;
  return CDPROBE_OK;
}

}  // extern "C"
