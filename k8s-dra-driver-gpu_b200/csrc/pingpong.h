// pingpong.h — host-callable launcher of the signal round trip in pingpong_kernels.cu (cdprobe_pingpong).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "probe_types.h"
#include "timed_rep.cuh"

namespace cdp {

constexpr uint32_t kPingPongDefaultTrips = 256;
constexpr uint32_t kPingPongDefaultReps = 8;
constexpr uint32_t kPingPongMaxTrips = 1u << 16;
constexpr uint32_t kPingPongNoFault = 0xFFFFFFFFu;

struct PingPongRound {    // what one rank does in one round of the tournament
  uint64_t* remote;       // its own line ping[rank] in the partner's memory, through its mapping; null: idle this round
  const uint64_t* local;  // the partner's line ping[partner] in its own memory, through its local VA
  uint32_t partner;
  uint32_t first;         // 1: this rank initiates leg 0 (it is the lower rank of the pair), 0: leg 1
};

struct PingPongParams {
  PingPongRound round[kMaxRanks];
  uint64_t call_seq;
  uint64_t timeout_ns;      // device deadline from kernel entry, checked every 64 spins of a poll
  uint32_t n_rounds, trips, reps;  // reps: timed reps (rep 0, the warm-up, comes on top)
  uint32_t fault_round;     // test-only skip-ahead echo: the round in which this rank answers the armed initiator
  uint32_t fault_trip;      // ... and the trip of timed rep 1 it answers with the next trip's echo (kPingPongNoFault: none)
};

// Enqueues one 32-thread block for one rank on `stream`; the cell it initiates in round r leaves its reps at
// out[r * kRepSlots + rep], CDPROBE_ERR_INTEGRITY marking a rep with an unexpected echo.  Returns a cudaError_t.
int pingpong_launch(const PingPongParams& p, bool fenced, TimedRep* out, cudaStream_t stream);

}  // namespace cdp
