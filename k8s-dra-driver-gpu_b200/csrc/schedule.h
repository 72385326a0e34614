// schedule.h — see schedule.cc.
#pragma once
#include <stdint.h>

#include "../../include/cdprobe.h"
#include "plan.h"
#include "probe_types.h"

namespace cdp {

struct ScheduleInput {
  const Plan* plan = nullptr;
  uint32_t rank = 0;         // global rank the table is for
  uint32_t ops = 0;          // CDPROBE_OP_*
  uint32_t flags = 0;        // CDPROBE_FLAG_* (OVERLAP_VERIFY, UNIDIRECTIONAL matter)
  uint32_t ctas = 0;         // CTAs of this rank's kernel
  uint32_t verify_ctas = 32; // CTAs of an overlapped verify job
  const int32_t (*status)[kMaxRanks] = nullptr;  // [issuer][owner] mapping status; null = every pair mapped
};

// Fills phases[0..kMaxPhases) / n_phases / peer_mask. CDPROBE_ERR_ARG when the table would overflow.
int make_phases(const ScheduleInput& in, Phase* phases, uint32_t* n_phases, uint32_t* peer_mask);

// The payload one run moves between devices (DESIGN §5o), in bytes per device: every rank r in ran_mask walks the
// phase table make_phases gives `in` with in.rank = r.  A read job of r with peer j (r reads j's slice) adds
// bytes_per_pair to j's tx and r's rx; a write job to r's tx and j's rx; a warm-up job adds its prefix,
// min(warm_bytes, bytes_per_pair), as a read (warm_bytes 0: the run did not warm).  Only jobs whose two ranks are on
// different devices count: dev[r] names rank r's device, tx[d] and rx[d] (n entries each) are device d's.  Verify
// jobs, barrier flags and read requests are not payload.
void link_payload(const ScheduleInput& in, uint32_t ran_mask, const uint32_t* dev, uint64_t warm_bytes, uint64_t* tx,
                  uint64_t* rx);

}  // namespace cdp
