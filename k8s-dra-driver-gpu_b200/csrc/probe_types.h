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

// Work counters of the single-GPU loop-back pass (probe_kernels.cu, loopback_pass).  Every run starts from
// zero: the CTA that writes the result row clears them again (open and an aborted run zero all of Ctrl from
// grid_arrive on).  Each hot word has its own 128-byte line.
struct LoopBack {
  struct alignas(128) Counter {
    unsigned long long v;
  };
  Counter claim[3];                   // next unclaimed unit of the write, the source read and the verify
  Counter written;                    // units whose stores have completed
  Counter done;                       // CTAs that have finished all their work
  unsigned long long t_first_n[2];    // ~(earliest first issue) of the write and of the source read (0 = none yet)
  unsigned long long t_enter_n;       // ~(earliest CTA entry)
};

// Test-only fault injection (cdprobe_corrupt_landing): after this rank's write into `target`'s landing slot has
// completed and before anyone verifies it, the kernel xors mask[e] into word word[e] of the slot, e < n.  n = 0:
// disarmed.  Written by the host between runs only.
constexpr uint32_t kMaxLandingFaults = 8;
struct LandingFault {
  uint32_t n, target;
  uint64_t word[kMaxLandingFaults];
  uint64_t mask[kMaxLandingFaults];
};

struct Ctrl {
  // ---- written by peers over NVLink ------------------------------------
  FlagLine flags[kMaxRanks];          // flags[j].v = last barrier target rank j signalled
  WrPub wr[kMaxRanks];                // index = landing slot
  uint64_t verdict[kMaxRanks];        // index = verifier rank; value = run_seq * 4 + VerdictCode
  // ---- published by the owner at open (read by peers) ------------------
  uint64_t src_sum[kMaxRanks];        // per source slice
  uint64_t src_xor[kMaxRanks];
  // ---- written by the host; before grid_arrive, so the reset after an aborted run keeps it ----
  LandingFault fault;
  // ---- local only ------------------------------------------------------
  alignas(128) unsigned int grid_arrive;
  alignas(128) unsigned long long grid_release;
  alignas(128) unsigned int abort_flag;
  alignas(128) uint64_t t_rel[kMaxPhases + 2];   // release time of barrier b
  uint64_t t_arr[kMaxPhases + 2];                // arrive time of barrier b (all local CTAs done)
  Acc acc[kMaxPhases][2];
  LoopBack lb;
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
  uint32_t path;                   // data path: 0 TMA bulk copies, 1 ld/st.global.v4 with 16 bytes per lane,
                                   // 2 ld/st.global.v4 with 32 contiguous bytes per lane (two accesses)
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

// ---- inverses of the pattern functions (cdprobe_diagnose) -------------------------------------------------
// Both patterns are bijections of a 64-bit word, so an observed word names the (rank, index) or (salt + index)
// that produced it.  The odd multipliers have these inverses mod 2^64.
constexpr uint64_t kInvGolden = 0xF1DE83E19937733Dull;
constexpr uint64_t kInvMix1 = 0x96DE1B173F119089ull;  // of 0xBF58476D1CE4E5B9
constexpr uint64_t kInvMix2 = 0x319642B2D24D8EC3ull;  // of 0x94D049BB133111EB
static_assert(kGolden * kInvGolden == 1ull && 0xBF58476D1CE4E5B9ull * kInvMix1 == 1ull &&
                  0x94D049BB133111EBull * kInvMix2 == 1ull, "modular inverses");
CDP_HD inline uint64_t unsplitmix64(uint64_t z) {
  z = z ^ (z >> 31) ^ (z >> 62);
  z *= kInvMix2;
  z = z ^ (z >> 27) ^ (z >> 54);
  z *= kInvMix1;
  z = z ^ (z >> 30) ^ (z >> 60);
  return z - kGolden;
}
// salt + k of a write-pattern word: y = z ^ (z >> 32) keeps the high half of z, so z = y ^ (y >> 32).
CDP_HD inline uint64_t unwrite_word(uint64_t y) { return (y ^ (y >> 32)) * kInvGolden; }

// Classes of a word that differs from the pattern (include/cdprobe.h CDPROBE_DIAG_*, same values).
enum DiagKind : uint32_t { kDiagFlip = 0, kDiagZero = 1, kDiagDisplaced = 2, kDiagStale = 3, kDiagForeign = 4 };
constexpr int kDiagKinds = 5;
constexpr int kDiagMaxCand = 1 + 8 + kMaxRanks;  // write cells: current salt, 8 earlier runs, every other writer

struct DiagCand {       // a write salt the cell's slot may hold words of
  uint64_t salt;
  uint64_t run_seq;     // the run that writes with it
  uint32_t kind;        // kDiagDisplaced (this writer, this run), kDiagStale or kDiagForeign
  int32_t rank;         // the writer
};

// What one cell's region must hold.  Word k of the region is
//   read cells:  src_word(seed, target, first_word + k)
//   write cells: write_word(cand[0].salt, k)   (cand[0] is the current salt)
struct DiagSpec {
  uint64_t seed;
  uint64_t first_word;  // read: index of the region's word 0 in the target's source pattern
  uint64_t n_words;     // words in the region
  uint64_t src_words;   // read: words in one rank's source buffer
  uint32_t is_write;
  uint32_t target;
  uint32_t n_ranks;
  uint32_t n_cand;      // write: entries of cand
  DiagCand cand[kDiagMaxCand];
};

struct DiagClass {
  uint32_t kind;        // DiagKind
  int32_t rank;         // whose pattern the word is (-1 for FLIP / ZERO)
  uint64_t word;        // DISPLACED / STALE / FOREIGN: the pattern index that produced it
  uint64_t run_seq;     // STALE: the run that wrote it
};

constexpr uint64_t kDiagStaleRuns = 8;  // earlier runs of the same writer a STALE word is traced back to

// Read cell: the region is words [first_word, first_word + n_words) of target's source buffer of src_words words.
inline DiagSpec diag_read_spec(uint64_t seed, uint32_t n_ranks, uint32_t target, uint64_t first_word, uint64_t n_words,
                               uint64_t src_words) {
  DiagSpec s = {};
  s.seed = seed;
  s.n_ranks = n_ranks;
  s.target = target;
  s.first_word = first_word;
  s.n_words = n_words;
  s.src_words = src_words;
  return s;
}
// Write cell: the n_words slot issuer fills in target in run run_seq.  Candidates, in the order they are tried:
// this run's salt (DISPLACED), the issuer's salts of the kDiagStaleRuns runs before (STALE), and every other
// rank's salt into the target in this run (FOREIGN).
inline DiagSpec diag_write_spec(uint64_t seed, uint32_t n_ranks, uint32_t issuer, uint32_t target, uint64_t run_seq,
                                uint64_t n_words) {
  DiagSpec s = {};
  s.seed = seed;
  s.n_ranks = n_ranks;
  s.target = target;
  s.n_words = n_words;
  s.is_write = 1;
  auto cand = [&](uint32_t writer, uint64_t seq, uint32_t kind) {
    DiagCand& c = s.cand[s.n_cand++];
    c.salt = write_salt(seed, writer, target, seq);
    c.run_seq = seq;
    c.kind = kind;
    c.rank = (int32_t)writer;
  };
  cand(issuer, run_seq, kDiagDisplaced);
  for (uint64_t d = 1; d <= kDiagStaleRuns && d < run_seq; ++d) cand(issuer, run_seq - d, kDiagStale);
  for (uint32_t r = 0; r < n_ranks && r < (uint32_t)kMaxRanks; ++r)
    if (r != issuer) cand(r, run_seq, kDiagForeign);
  return s;
}

CDP_HD inline uint64_t diag_expected(const DiagSpec& s, uint64_t k) {
  return s.is_write ? write_word(s.cand[0].salt, k) : src_word(s.seed, s.target, s.first_word + k);
}

// Class of an observed word that differs from the expected one, in this order: ZERO; a word of some rank's
// source pattern (read cells) or of a candidate write salt (write cells) whose index lies inside that buffer;
// anything else is a FLIP of the expected word.
CDP_HD inline DiagClass diag_classify(const DiagSpec& s, uint64_t observed) {
  DiagClass c = {kDiagFlip, -1, 0, 0};
  if (observed == 0) {
    c.kind = kDiagZero;
    return c;
  }
  if (!s.is_write) {
    const uint64_t x = unsplitmix64(observed) ^ s.seed;  // = rank << 56 ^ k
    const uint32_t r = (uint32_t)(x >> 56);
    const uint64_t k = x & ((1ull << 56) - 1);
    if (r < s.n_ranks && k < s.src_words) {
      c.kind = r == s.target ? kDiagDisplaced : kDiagForeign;
      c.rank = (int32_t)r;
      c.word = k;
    }
    return c;
  }
  const uint64_t z = unwrite_word(observed);  // = salt + k
  for (uint32_t i = 0; i < s.n_cand; ++i) {
    const uint64_t k = z - s.cand[i].salt;
    if (k < s.n_words) {
      c.kind = s.cand[i].kind;
      c.rank = s.cand[i].rank;
      c.word = k;
      c.run_seq = c.kind == kDiagStale ? s.cand[i].run_seq : 0;
      return c;
    }
  }
  return c;
}

// ---- the dependent-load chase (cdprobe_latency, DESIGN §5c) ----------------------------------------------------
// A chase ranges over the L = bytes / 128 lines of the source slice issuer i reads from target j.  Hop h loads
// v = word 16 * line of that region (src_word(seed, j, first_word + 16 * line)); the next line is drawn from v, so
// every load waits for the one before.  Mixing in h + 1 keeps a chase that revisits a line from repeating its path.
constexpr uint64_t kLatencyTag = 0x4C4154454E4359ull;  // "LATENCY"
constexpr uint32_t kLineWords = 16;                    // one 128-byte line

// (x * n) >> 64: maps x uniformly into [0, n) without a division, so every line lies inside the region whatever
// word the previous load returned.
CDP_HD inline uint64_t fastrange64(uint64_t x, uint64_t n) {
#if defined(__CUDA_ARCH__)
  return __umul64hi(x, n);
#else
  return (uint64_t)(((unsigned __int128)x * n) >> 64);
#endif
}
// First line of rep r of cell (i, j); r = 0 is the untimed warm-up.
CDP_HD inline uint64_t latency_start(uint64_t seed, uint32_t i, uint32_t j, uint32_t r, uint64_t lines) {
  return fastrange64(splitmix64(seed ^ kLatencyTag ^ ((uint64_t)i << 56) ^ ((uint64_t)j << 48) ^ r), lines);
}
// The line after hop h loaded v.
CDP_HD inline uint64_t latency_next(uint64_t v, uint32_t h, uint64_t lines) {
  return fastrange64(v ^ ((uint64_t)(h + 1) * kGolden), lines);
}
// Xor of every word one rep of the chase loads from an intact region (host side of the digest check).
inline uint64_t latency_rep_digest(uint64_t seed, uint32_t i, uint32_t j, uint64_t first_word, uint64_t lines,
                                   uint32_t rep, uint32_t hops) {
  uint64_t line = latency_start(seed, i, j, rep, lines), digest = 0;
  for (uint32_t h = 0; h < hops; ++h) {
    const uint64_t v = src_word(seed, j, first_word + kLineWords * line);
    digest ^= v;
    line = latency_next(v, h, lines);
  }
  return digest;
}

// ---- the signal round trip (cdprobe_pingpong, DESIGN §5d) -----------------------------------------------------
// One 128-byte line per sender after Ctrl in the Ctrl granule: ping[s] in rank o's memory holds the last word s sent
// to o.  Open zeroes the whole granule; the reset after an aborted run zeroes only [grid_arrive, sizeof(Ctrl)), so
// these lines are never touched by it, and cdprobe_pingpong touches no Ctrl word.
constexpr uint64_t kPingOff = 64ull << 10;
static_assert(sizeof(Ctrl) <= kPingOff && kPingOff % 128 == 0 && kPingOff + kMaxRanks * sizeof(FlagLine) <= kCtrlBytes,
              "the pingpong lines sit after Ctrl inside its granule");

// A pingpong word.  Bits [0, 17): 2 * trip + echo; [17, 24): rep (0 = the warm-up); 24: leg; [25, 29): round;
// [29, 64): call_seq.  Words rise strictly along (call, round, leg, rep, trip, echo), so a word of an earlier call,
// round, leg, rep or trip never satisfies a wait for a later one.
constexpr uint32_t kPingTripBits = 17, kPingRepShift = 17, kPingLegShift = 24, kPingRoundShift = 25, kPingCallShift = 29;
CDP_HD inline uint64_t pingpong_word(uint64_t call_seq, uint32_t round, uint32_t leg, uint32_t rep, uint32_t trip,
                                     uint32_t echo) {
  return (call_seq << kPingCallShift) | ((uint64_t)round << kPingRoundShift) | ((uint64_t)leg << kPingLegShift) |
         ((uint64_t)rep << kPingRepShift) | (uint64_t)(2u * trip + echo);
}
// Xor of the echo words trips 0 .. trips - 1 of one rep return: the initiator's digest of a clean rep.  The trip
// field holds 2t + 1 below the rep's base, so the xor is base (when trips is odd) | the xor of 2t + 1 over t < trips.
CDP_HD inline uint64_t pingpong_rep_digest(uint64_t call_seq, uint32_t round, uint32_t leg, uint32_t rep, uint32_t trips) {
  const uint64_t base = pingpong_word(call_seq, round, leg, rep, 0, 0);
  const uint64_t m = trips - 1u;  // xor of 0 .. m
  const uint64_t x = (m & 3u) == 0 ? m : (m & 3u) == 1 ? 1 : (m & 3u) == 2 ? m + 1 : 0;
  return ((trips & 1u) ? base : 0ull) | (x << 1) | (uint64_t)(trips & 1u);
}

// ---- remote atomics (cdprobe_atomics, DESIGN §5e) ------------------------------------------------------------
// One 128-byte line per issuer after the pingpong lines: word 0 of atom[i] in rank j's Ctrl granule is cell (i, j)'s
// word, and only issuer i ever touches it, so no two cells or processes contend.  Open zeroes the whole granule; the
// reset after an aborted run and every other call leave these lines alone.
struct alignas(128) AtomLine {
  unsigned long long v;
  unsigned long long pad[15];
};
constexpr uint64_t kAtomOff = kPingOff + kMaxRanks * sizeof(FlagLine);  // 66 KiB
static_assert(kAtomOff >= kPingOff + kMaxRanks * sizeof(FlagLine) && kAtomOff % 128 == 0 &&
                  kAtomOff + kMaxRanks * sizeof(AtomLine) <= kCtrlBytes,
              "the atomics lines sit after the pingpong lines inside the Ctrl granule");

// The value a rep's opening exch stores.  Bits [0, 22): zero, room for the 32 x 2^16 increments of the largest rep;
// [22, 29): rep (0 = the warm-up); [29, 31): kind; [31, 63): the low 32 bits of call_seq.  Bit 63 is always 0, so
// `1 + (r >> 63)` is 1 for every value the word holds.
constexpr uint32_t kAtomRepShift = 22, kAtomKindShift = 29, kAtomCallShift = 31;
CDP_HD inline uint64_t atomics_start(uint64_t call_seq, uint32_t kind, uint32_t rep) {
  return ((call_seq & 0xFFFFFFFFull) << kAtomCallShift) | ((uint64_t)(kind & 3u) << kAtomKindShift) |
         ((uint64_t)(rep & 127u) << kAtomRepShift);
}
// Xor of start, start + 1, ..., start + total - 1: the values one clean rep's increments return, over every lane
// (total = lanes x ops < 2^22).  The low bits of start are zero, so start + k = start | k, and the xor is start (when
// total is odd) | the xor of 0 .. total - 1.
CDP_HD inline uint64_t atomics_rep_digest(uint64_t start, uint64_t total) {
  if (total == 0) return 0;
  const uint64_t m = total - 1;  // xor of 0 .. m
  const uint64_t x = (m & 3u) == 0 ? m : (m & 3u) == 1 ? 1 : (m & 3u) == 2 ? m + 1 : 0;
  return ((total & 1u) ? start : 0ull) | x;
}
// Sum of the same values mod 2^64: what the warp's returns add up to in a clean CONTENDED rep.
CDP_HD inline uint64_t atomics_rep_sum(uint64_t start, uint64_t total) {
  return total * start + (total & 1u ? total * ((total - 1) / 2) : (total / 2) * (total - 1));
}

// ---- the bandwidth-versus-size curve (cdprobe_bwcurve, DESIGN §5f) -------------------------------------------------
constexpr uint32_t kBwMaxSizes = 24;     // CDPROBE_BWCURVE_MAX_SIZES
constexpr uint64_t kBwMinSize = 4096;
constexpr uint64_t kGranuleWords = kGranuleBytes / 8;

// The sizes a cell is read at: 4096 << k for every k with 4096 << k < bpp, then bpp itself.  Returns how many, or 0
// when that is more than kBwMaxSizes (bpp > 32 GiB).  size has room for kBwMaxSizes.
CDP_HD inline uint32_t bwcurve_ladder(uint64_t bpp, uint64_t* size) {
  uint32_t n = 0;
  for (uint64_t s = kBwMinSize; s < bpp; s <<= 1) {
    if (n == kBwMaxSizes) return 0;
    size[n++] = s;
  }
  if (n == kBwMaxSizes) return 0;
  size[n++] = bpp;
  return n;
}

// (S, X) of the first n_words words of a region from gsum[g] and gxor[g], the sum and xor of the words of each whole
// granule g of the region.  The words of a last, partial granule (at most kGranuleWords - 1) come from word(k), word k
// of the region.
template <typename Word>
CDP_HD inline void prefix_checksum(const uint64_t* gsum, const uint64_t* gxor, uint64_t n_words, const Word& word,
                                   uint64_t* sum, uint64_t* xr) {
  const uint64_t whole = n_words / kGranuleWords;
  uint64_t s = 0, x = 0, px = 0;
  for (uint64_t g = 0; g < whole; ++g) {
    s += gsum[g];
    x ^= rotl64(gxor[g], fold6((uint32_t)g));
  }
  for (uint64_t k = whole * kGranuleWords; k < n_words; ++k) {
    const uint64_t w = word(k);
    s += w;
    px ^= w;
  }
  *sum = s;
  *xr = x ^ rotl64(px, fold6((uint32_t)whole));
}

struct SrcRegionWord {  // word k of a source region: words first_word... of rank's pattern
  uint64_t seed, first_word;
  uint32_t rank;
  CDP_HD uint64_t operator()(uint64_t k) const { return src_word(seed, rank, first_word + k); }
};

// (S, X) of the first n_words words of a source region, words first_word... of rank's pattern (prefix_checksum).
CDP_HD inline void bwcurve_prefix_checksum(const uint64_t* gsum, const uint64_t* gxor, uint64_t seed, uint32_t rank,
                                           uint64_t first_word, uint64_t n_words, uint64_t* sum, uint64_t* xr) {
  prefix_checksum(gsum, gxor, n_words, SrcRegionWord{seed, first_word, rank}, sum, xr);
}

// ---- the one-shot all-reduce (cdprobe_allreduce, DESIGN §5g) -------------------------------------------------------
// Word w of the output every rank computes: the sum mod 2^64 of word w of every rank's source buffer.  Integer addition
// wraps exactly and commutes, so the order in which a rank adds its inputs does not change the result.
CDP_HD inline uint64_t allreduce_word(uint64_t seed, uint32_t n, uint64_t w) {
  uint64_t s = 0;
  for (uint32_t j = 0; j < n; ++j) s += src_word(seed, j, w);
  return s;
}
struct AllReduceWord {
  uint64_t seed;
  uint32_t n;
  CDP_HD uint64_t operator()(uint64_t k) const { return allreduce_word(seed, n, k); }
};
// (S, X) of the first n_words words of the output, from the per-granule sums of the summed words (prefix_checksum).
// S is the sum of the ranks' prefix sums; X is not made of the ranks' X, since xor does not distribute over the sum.
CDP_HD inline void allreduce_prefix_checksum(const uint64_t* gsum, const uint64_t* gxor, uint64_t seed, uint32_t n,
                                             uint64_t n_words, uint64_t* sum, uint64_t* xr) {
  prefix_checksum(gsum, gxor, n_words, AllReduceWord{seed, n}, sum, xr);
}

// The domain barrier of cdprobe_allreduce: one 128-byte line per sender after the atomics lines, in the Ctrl granule.
// line[s] in rank o's memory holds the last (call_seq << 16) | (b + 1) rank s signalled to o.  The values rise across
// calls and barriers, so no call resets them; open zeroes the granule, and nothing else touches these lines.
constexpr uint64_t kArOff = kAtomOff + kMaxRanks * sizeof(AtomLine);  // 68 KiB
static_assert(kArOff % 128 == 0 && kArOff + kMaxRanks * sizeof(FlagLine) <= kCtrlBytes,
              "the all-reduce lines sit after the atomics lines inside the Ctrl granule");
constexpr uint32_t kArBarrierBits = 16;  // barriers per call: at most kBwMaxSizes x (kMaxTimedReps + 2) < 2^16
constexpr uint32_t kArNoFault = ~0u;

}  // namespace cdp
