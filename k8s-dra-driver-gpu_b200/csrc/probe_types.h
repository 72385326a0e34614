// probe_types.h — structures shared by the host runtime and the sm_90a kernels.
//
// HBM layout of one rank's probe allocation (one cuMemCreate handle, mapped
// into every peer's address space with cuMemMap/cuMemSetAccess):
//
//   [0, kCtrlBytes)                  Ctrl: barrier flags, published checksums
//   [src_off,  src_off  + src_bytes) source buffer  (read probe: peers load it)
//   [land_off, land_off + land_bytes) landing slots (write probe: peers store here)
//
// Every offset is 2 MiB granular (VMM granularity); slices/slots are 128 B
// aligned (SURVEY.md §8d).
#pragma once
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define CDP_HD __host__ __device__
#else
#define CDP_HD
#endif

namespace cdp {

constexpr int kMaxRanks = 16;
constexpr int kMaxPhases = 64;
constexpr uint32_t kUnitBytes = 8192;      // work unit of one warp == one TMA stage
constexpr uint32_t kGranuleBytes = 16384;  // checksum rotation granule (spec constant)
constexpr int kWarpsPerCta = 8;
constexpr int kThreads = kWarpsPerCta * 32;
constexpr int kStages = 3;                 // TMA stages per warp (24 KiB in flight per warp)
constexpr uint32_t kSmemBytes = kWarpsPerCta * kStages * kUnitBytes + 1024;
constexpr uint64_t kCtrlBytes = 2ull << 20;
constexpr uint64_t kVmmGranule = 2ull << 20;
constexpr uint32_t kLdstVecs = 16;         // 16-byte vectors in flight per lane on the ld/st path

constexpr uint64_t kDefaultSeed = 0xCD5EED0000000001ull;
constexpr uint64_t kGolden = 0x9E3779B97F4A7C15ull;

enum JobKind : uint8_t { kJobNone = 0, kJobRead = 1, kJobWrite = 2, kJobVerify = 3, kJobWarm = 4 };
enum PhaseCode : int32_t { kCodeOk = 0, kCodeSkipped = 1, kCodeAborted = 2 };
enum VerdictCode : uint64_t { kVerdictNone = 0, kVerdictOk = 1, kVerdictMismatch = 2, kVerdictNotWritten = 3 };

struct alignas(128) FlagLine {
  uint64_t v;
  uint64_t pad[15];
};

struct WrPub {        // written by the remote writer of a landing slot, every run
  uint64_t sum, xr, seq, pad;
};

struct alignas(32) Acc {
  unsigned long long sum, xr, t_end, pad;
};

struct Ctrl {
  // ---- written by peers over NVLink ------------------------------------
  FlagLine flags[kMaxRanks];          // flags[j].v = last barrier target rank j signalled
  WrPub wr[kMaxRanks];                // index = landing slot
  uint64_t verdict[kMaxRanks];        // index = verifier rank; value = run_seq * 4 + VerdictCode
  // ---- published by the owner at open (read by peers) ------------------
  uint64_t src_sum[kMaxRanks];        // per source slice
  uint64_t src_xor[kMaxRanks];
  // ---- local only ------------------------------------------------------
  alignas(128) unsigned int grid_arrive;
  alignas(128) unsigned long long grid_release;
  alignas(128) unsigned int abort_flag;
  alignas(128) uint64_t t_rel[kMaxPhases + 2];   // release time of barrier b
  uint64_t t_arr[kMaxPhases + 2];                // arrive time of barrier b (all local CTAs done)
  Acc acc[kMaxPhases][2];
};
static_assert(sizeof(Ctrl) <= kCtrlBytes, "Ctrl must fit its granule");

struct Job {            // 16 bytes
  uint8_t kind;         // JobKind
  int8_t peer;          // rank whose memory is touched (self for verify/diag)
  uint8_t slot;         // landing slot (write/verify) or source slice (read)
  uint8_t writer;       // verify: rank that wrote the slot
  uint16_t cta0;        // first CTA of the job
  uint16_t nctas;       // CTAs of the job
  uint64_t salt;        // write: pattern salt; warm: bytes to stream (0 = skip); verify: index b >= 1 of the barrier
                        // whose signal from `writer` the job waits for before it reads the slot (0 = none)
};

struct Phase {          // 40 bytes
  Job job[2];
  uint32_t sync_mask;   // ranks this GPU exchanges barrier flags with when the phase closes (0: this GPU only)
  uint32_t post_mask;   // ranks it only SIGNALS then (after releasing its own CTAs): a write -> read step inside a round,
                        // where the next phase needs the partner's data (the verify job waits for it) but not its ports
};

struct PhaseOut {
  uint64_t t_start;     // release time of the barrier that opened the phase
  uint64_t t_arrive;    // arrive time of the barrier that closed it
  uint64_t t_end[2];    // per job: max over CTAs of completion time
  uint64_t sum[2], xr[2];
  uint64_t exp_sum[2], exp_xr[2];
  int32_t code[2];
  uint64_t verdict[2];  // write jobs: verdict word received from the verifier
};

struct ResultRow {      // pinned host memory, written by CTA 0 at the end of a run
  volatile uint64_t done;   // == run_seq when the row is complete
  uint64_t t_first, t_last;
  uint32_t aborted, n_phases;
  PhaseOut ph[kMaxPhases];
  uint64_t t_enter, t_exit;  // %globaltimer when CTA 0 entered the kernel / just before it published the row
};

struct ProbeParams {
  uint8_t* base_peer[kMaxRanks];   // rank j's allocation as mapped for this rank; null = unmapped
  ResultRow* row;
  uint64_t seq_base;               // barrier targets of this run are seq_base + 1 .. + n_phases + 1
  uint64_t run_seq;
  uint64_t timeout_ns;
  uint64_t bpp;                    // bytes per pair
  uint64_t src_off, land_off;
  uint32_t rank, n_ranks, n_phases;
  uint32_t peer_mask;              // ranks taking part in the cross-GPU barrier with this rank
  uint32_t use_ldst;               // 0 TMA bulk, 1 ld/st.global.v4
  uint32_t full_mode;              // source has a single slice
  Phase phase[kMaxPhases];
};
static_assert(sizeof(ProbeParams) == 2768, "kernel parameter bytes (bench.py reports them as h2d bytes per step)");
static_assert(sizeof(PhaseOut) == 120 && offsetof(ResultRow, ph) == 32 && sizeof(ResultRow) == 32 + 120 * kMaxPhases + 16,
              "result row bytes (bench.py: d2h per step = 48 + 120 x phases)");

// ---- integer definitions shared with the oracle (oracle/pattern.c restates them) ----
CDP_HD inline uint64_t splitmix64(uint64_t x) {
  uint64_t z = x + kGolden;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// Source pattern (SURVEY.md §8d): word k of rank r's source buffer.
CDP_HD inline uint64_t src_word(uint64_t seed, uint32_t rank, uint64_t k) {
  return splitmix64(seed ^ ((uint64_t)rank << 56) ^ k);
}
// Write pattern: word k of what `src` stores into `dst`'s landing slot.
CDP_HD inline uint64_t write_salt(uint64_t seed, uint32_t src, uint32_t dst, uint64_t run_seq) {
  return splitmix64(seed ^ 0x5752495445ull ^ ((uint64_t)src << 56) ^ ((uint64_t)dst << 48) ^ run_seq);
}
CDP_HD inline uint64_t write_word(uint64_t salt, uint64_t k) {
  uint64_t z = (salt + k) * kGolden;
  return z ^ (z >> 32);
}
CDP_HD inline uint32_t fold6(uint32_t g) {
  return (g ^ (g >> 6) ^ (g >> 12) ^ (g >> 18) ^ (g >> 24) ^ (g >> 30)) & 63u;
}
CDP_HD inline uint64_t rotl64(uint64_t x, uint32_t r) {
  r &= 63u;
  return r ? ((x << r) | (x >> (64u - r))) : x;
}
// Checksum of a slice of 64-bit words w[0..n):
//   S = sum w[k] mod 2^64
//   X = xor over granules g of rotl64(xor of the words of granule g, fold6(g)),
//       granule = 16 KiB = 2048 words, g counted from the slice start.

}  // namespace cdp
