// rep_times_host.cc — the rep-record fold of measure.cc (summarize, ladder_times, bw_times, bw_summarize), compiled
// for the host from a verbatim copy (tests/rep_times.py writes rep_times_fold.inc) and driven through a C ABI by
// tests/test_rep_times_cpu.py.  The records are built here from what the test passes; each call fills one entry of the
// output struct the library fills with it, starting zeroed, and copies that entry out flat.
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "cdprobe.h"
#include "bwcurve.h"
#include "probe_types.h"
#include "timed_rep.cuh"

namespace cdp {
#include "rep_times_fold.inc"
}  // namespace cdp

using cdp::kBwMaxSizes;
using cdp::kMaxTimedReps;
using cdp::kRepSlots;

// One entry of an output struct; fields the entry's struct lacks stay 0.
struct RtEntry {
  uint32_t measured;
  int32_t status;
  uint32_t bad_sizes;
  float t0_ns, peak_gbps;
  uint64_t half_bytes, digest;
  float ns_min[kBwMaxSizes], ns_median[kBwMaxSizes], ns_max[kBwMaxSizes];
  uint64_t sum[kBwMaxSizes], xr[kBwMaxSizes];
};

template <typename Out>
static void ladder_entry(const Out& o, uint32_t idx, uint32_t n_sizes, RtEntry* e) {
  memset(e, 0, sizeof(*e));
  e->measured = o.measured[idx];
  e->status = o.status[idx];
  e->t0_ns = o.t0_ns[idx];
  e->peak_gbps = o.peak_gbps[idx];
  e->half_bytes = o.half_bytes[idx];
  for (uint32_t k = 0; k < n_sizes; ++k) {
    e->ns_min[k] = o.ns_min[idx][k];
    e->ns_median[k] = o.ns_median[idx][k];
    e->ns_max[k] = o.ns_max[idx][k];
  }
}

extern "C" {

uint32_t rt_dims(uint32_t which) { return which == 0 ? kBwMaxSizes : kRepSlots; }

cdp::BwScratch* rt_scratch_new() { return static_cast<cdp::BwScratch*>(calloc(1, sizeof(cdp::BwScratch))); }
void rt_scratch_free(cdp::BwScratch* s) { free(s); }
void rt_scratch_abort(cdp::BwScratch* s, uint32_t v) { s->abort_flag = v; }
void rt_scratch_set(cdp::BwScratch* s, uint32_t k, uint32_t r, uint64_t t_rel, uint64_t t_end, uint64_t sum,
                    uint64_t xr) {
  s->t_rel[k][r] = t_rel;
  s->rep[k][r].t_end = t_end;
  s->rep[k][r].sum = sum;
  s->rep[k][r].xr = xr;
}

// summarize into entry idx of a cdprobe_latency_t: reps + 1 records (rep 0 the warm-up) of ns, digest and status.
void rt_summarize(const uint64_t* ns, const uint64_t* digest, const int32_t* status, uint32_t reps, uint32_t per_rep,
                  uint64_t want, uint32_t idx, RtEntry* e) {
  cdp::TimedRep rep[kRepSlots] = {};
  for (uint32_t k = 0; k <= reps; ++k) rep[k] = {ns[k], digest[k], status[k], 0};
  auto* out = static_cast<cdprobe_latency_t*>(calloc(1, sizeof(cdprobe_latency_t)));
  cdp::summarize(rep, reps, per_rep, want, idx, out);
  memset(e, 0, sizeof(*e));
  e->measured = out->measured[idx];
  e->status = out->status[idx];
  e->digest = out->digest[idx];
  e->ns_min[0] = out->ns_min[idx];
  e->ns_median[0] = out->ns_median[idx];
  e->ns_max[0] = out->ns_max[idx];
  free(out);
}

// ladder_times into entry idx of a cdprobe_memcpy_t, from ns[k * kMaxTimedReps + r].
void rt_ladder_times(const float* ns, const uint64_t* size, uint32_t n_sizes, uint32_t reps, double scale,
                     uint32_t idx, RtEntry* e) {
  auto* t = new float[kBwMaxSizes][kMaxTimedReps];
  memcpy(t, ns, sizeof(float) * kBwMaxSizes * kMaxTimedReps);
  auto* out = static_cast<cdprobe_memcpy_t*>(calloc(1, sizeof(cdprobe_memcpy_t)));
  cdp::ladder_times(t, size, n_sizes, reps, scale, idx, out);
  ladder_entry(*out, idx, n_sizes, e);
  free(out);
  delete[] t;
}

// bw_times into entry idx of a cdprobe_alltoall_t; returns what bw_times returns.
int rt_bw_times(const cdp::BwScratch* s, const uint64_t* size, uint32_t n_sizes, uint32_t reps, double scale,
                uint32_t idx, RtEntry* e) {
  auto* out = static_cast<cdprobe_alltoall_t*>(calloc(1, sizeof(cdprobe_alltoall_t)));
  const bool timed = cdp::bw_times(*s, size, n_sizes, reps, scale, idx, out);
  ladder_entry(*out, idx, n_sizes, e);
  free(out);
  return timed ? 1 : 0;
}

// bw_summarize into entry idx of a cdprobe_bwcurve_t, against want[k * 2 + {0, 1}].
void rt_bw_summarize(const cdp::BwScratch* s, const uint64_t* want, const uint64_t* size, uint32_t n_sizes,
                     uint32_t reps, uint32_t idx, RtEntry* e) {
  auto* out = static_cast<cdprobe_bwcurve_t*>(calloc(1, sizeof(cdprobe_bwcurve_t)));
  cdp::bw_summarize(*s, reinterpret_cast<const uint64_t(*)[2]>(want), size, n_sizes, reps, idx, out);
  ladder_entry(*out, idx, n_sizes, e);
  e->bad_sizes = out->bad_sizes[idx];
  for (uint32_t k = 0; k < n_sizes; ++k) {
    e->sum[k] = out->sum[idx][k];
    e->xr[k] = out->xr[idx][k];
  }
  free(out);
}

}  // extern "C"
