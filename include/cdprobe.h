/*
 * cdprobe.h — C ABI of libcdprobe.so: the ComputeDomain fabric-validation probe.
 *
 * This is the drop-in boundary for the compute-domain-daemon's domain-ready
 * gate.  The reference's gate is `check()` in
 *   cmd/compute-domain-daemon/main.go:435-459
 * (exec `nvidia-imex-ctl -q`, compare stdout with "READY\n"; a no-op when
 * CLIQUE_ID is empty, main.go:436-439).  The reference has no NVLink probe
 * (SURVEY.md F1); the functions below are what a Go shim `pkg/fabricprobe`
 * binds over cgo (see INTEGRATION.md) so that `run()` (main.go:212-347) can
 * execute an all-pairs NVLink reachability + bandwidth probe on the GPUs the
 * daemon owns and `check()` can consult its verdict.
 *
 * Rules of the ABI (SURVEY.md §8b):
 *   - plain C, fixed-width integers, caller-allocated outputs, no pointers
 *     cross back except the opaque handle;
 *   - 0 = ok, <0 = cdprobe error enum (below); the CUDA/driver status that
 *     caused a CDPROBE_ERR_CUDA is available from cdprobe_last_error();
 *   - the library never prints and never aborts (klog owns stdout/stderr in
 *     the daemon: cmd/compute-domain-daemon/process.go:92-96);
 *   - a handle is not thread-safe; distinct handles are independent;
 *   - there is NO CPU fallback: without a CUDA driver + sm_90 device
 *     cdprobe_open() fails with CDPROBE_ERR_NO_DEVICE / _UNSUPPORTED.
 *
 * All integer results (reachability bits, checksums, schedule) are exact;
 * GB/s values are measurements (run-to-run tolerance +-2 %, north_star).
 */
#ifndef CDPROBE_H_
#define CDPROBE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define CDPROBE_API __attribute__((visibility("default")))
#else
#define CDPROBE_API
#endif

#define CDPROBE_ABI_VERSION 2u         /* 2: neighbourhood barriers (sync_mask), calibrated gate, ce_copy */
#define CDPROBE_MAX_GPUS 16          /* ranks in one probe domain (8 on HGX H100) */
#define CDPROBE_MAX_PHASES 64
#define CDPROBE_NVLINK_MAX_LINKS 18  /* == NVML_NVLINK_MAX_LINKS (nvml.h:389) */

/* Error enum (return values). */
#define CDPROBE_OK 0
#define CDPROBE_ERR_ABI (-1)         /* abi field mismatch */
#define CDPROBE_ERR_ARG (-2)         /* invalid argument / config */
#define CDPROBE_ERR_NO_DEVICE (-3)   /* no CUDA driver, or no usable GPU */
#define CDPROBE_ERR_CUDA (-4)        /* a CUDA call failed; see cdprobe_last_error */
#define CDPROBE_ERR_TIMEOUT (-5)     /* timeout_ms expired (device or host watchdog) */
#define CDPROBE_ERR_RENDEZVOUS (-6)  /* multi-process handle exchange failed */
#define CDPROBE_ERR_NOMEM (-7)
#define CDPROBE_ERR_UNSUPPORTED (-8) /* device lacks VMM / cooperative launch / sm_90 */
#define CDPROBE_ERR_STATE (-9)       /* handle unusable after a sticky CUDA error */
#define CDPROBE_ERR_INTEGRITY (-10)  /* self-check of published checksums failed */

/* cdprobe_config_t.mode — SURVEY.md §8(d) "Modes & algorithmic bytes". */
#define CDPROBE_MODE_REACH_ONLY 0u   /* 64 KiB per ordered pair: latency floor */
#define CDPROBE_MODE_SLICED 1u       /* bytes_per_pair = floor(B/(N-1)/128)*128 */
#define CDPROBE_MODE_FULL 2u         /* bytes_per_pair = B */

/* cdprobe_config_t.ops */
#define CDPROBE_OP_READ 1u           /* rank i loads peer j's slice, checksums it */
#define CDPROBE_OP_WRITE 2u          /* rank i stores a pattern into peer j; j verifies */

/* cdprobe_config_t.flags */
#define CDPROBE_FLAG_FABRIC_HANDLES 0x01u  /* CU_MEM_HANDLE_TYPE_FABRIC when /dev/nvidia-caps-imex-channels/channel0 opens */
#define CDPROBE_FLAG_MIG_AWARE 0x02u       /* MIG devices: skip peer mapping, identity matrix (SURVEY H8) */
#define CDPROBE_FLAG_LOCAL_DIAG 0x04u      /* also measure the diagonal (loop-back into local HBM; always on when n == 1) */
#define CDPROBE_FLAG_PATH_LDST 0x08u       /* 128-bit ld/st.global instead of TMA bulk copies */
#define CDPROBE_FLAG_NO_COOPERATIVE 0x10u  /* plain launch (tests that put 2 ranks on one device) */
#define CDPROBE_FLAG_OVERLAP_VERIFY 0x20u  /* verify landing slots on spare CTAs while the next round runs (default) */
#define CDPROBE_FLAG_SIMULATE_MIG 0x200u   /* treat every local GPU as a MIG instance (BASELINE config 4 without MIG hardware) */
#define CDPROBE_FLAG_SERIAL_VERIFY 0x100u  /* opt out of the overlapped verify: verify every slot after the rounds */
#define CDPROBE_FLAG_ALLOW_SAME_DEVICE 0x40u /* several ranks may name the same CUDA ordinal (testing).  Each rank
                                              has its own stream; with more than 8 ranks on one device in one
                                              process, set CUDA_DEVICE_MAX_CONNECTIONS >= the rank count before the
                                              process creates its CUDA context, or two ranks' kernels may share a
                                              hardware queue and one wait behind the other at a barrier */
#define CDPROBE_FLAG_ALL_RANK_BARRIERS 0x400u /* every tournament phase closes with an all-rank flag exchange (round-1
                                              behaviour); default: only the ranks whose traffic shares an NVLink
                                              port with this rank's in the two phases either side of the barrier */
#define CDPROBE_FLAG_PAIR_BARRIERS 0x800u  /* keep the pair's flag exchange between the write and the read phase of a round
                                              (default: no wait there — the rank only signals its partner and the
                                              verify job waits for that signal itself) */
#define CDPROBE_FLAG_UNIDIRECTIONAL 0x80u  /* each round in two halves: one rank of a pair issues at a time, so a
                                              port carries payload one way only (per-link figure; 2x the phases) */

typedef struct cdprobe cdprobe_t;

typedef struct {
  uint32_t abi;                         /* CDPROBE_ABI_VERSION */
  uint32_t n_gpus;                      /* GPUs driven by THIS process; 0 = all visible */
  int32_t ordinals[CDPROBE_MAX_GPUS];   /* CUDA ordinals; ignored when n_gpus == 0 */
  uint64_t bytes;                       /* B: per-GPU probe buffer (1 GiB for the headline config) */
  uint32_t mode;                        /* CDPROBE_MODE_* */
  uint32_t ops;                         /* CDPROBE_OP_* bits; 0 = read|write */
  uint32_t timeout_ms;                  /* device + host watchdog; 0 = 5000 */
  uint32_t flags;                       /* CDPROBE_FLAG_* */
  uint64_t seed;                        /* 0 = 0xCD5EED0000000001 */
  float min_fraction;                   /* verdict threshold on pair GB/s, as a fraction of the reference figure below;
                                           0 = default (0.65) */
  float link_peak_gbps;                 /* reference figure of the gate.
                                           0 (default) = nominal H100 SXM NVLink 4 per direction (450 GB/s, data
                                           sheet) for every op and schedule, de-rated for the 6 us a phase spends
                                           ramping and draining (measured on an H100 at N = 1):
                                               expected(bytes_per_pair) = bytes_per_pair / (bytes_per_pair / 450 + 6 us)
                                           What healthy H100 NVLink delivers to SM-issued traffic has not been
                                           measured; the default fraction leaves room below nominal for it.
                                           >0 = absolute: threshold = min_fraction x link_peak_gbps */
  uint32_t ctas;                        /* CTAs of the persistent kernel; 0 = one per SM */
  uint32_t world_size;                  /* processes in the probe domain; 0/1 = single process */
  uint32_t rank;                        /* this process's index in [0, world_size) */
  uint32_t reserved0;
  char session[64];                     /* rendezvous name shared by all processes (world_size > 1) */
} cdprobe_config_t;

/* Matrices are row-major [issuer * CDPROBE_MAX_GPUS + target], issuer = the
 * rank whose SMs issue the loads (read) or stores (write).  A process fills
 * the rows of its local ranks (row_mask); cdprobe_gather() completes them. */
typedef struct {
  uint32_t abi;
  uint32_t n;                           /* total ranks in the domain */
  uint32_t row_mask;                    /* bit r set: row r is filled in */
  uint32_t verdict;                     /* 1: every filled off-diagonal cell reachable and >= min_fraction */
  uint8_t reach_read[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];
  uint8_t reach_write[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];
  float gbps_read[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];
  float gbps_write[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];
  int32_t status[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS]; /* 0 ok; <0 CDPROBE_ERR_*; >0 CUresult of the mapping */
  uint64_t sum_read[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];  /* checksum S the issuer computed (parity tests) */
  uint64_t xor_read[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];  /* checksum X */
  uint64_t sum_write[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS]; /* checksum of the pattern the issuer generated */
  uint64_t xor_write[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];
  uint64_t bytes_per_pair;
  uint64_t run_seq;                     /* sequence number of this run on the handle: the source checksum pass of
                                           cdprobe_open is 1, so the first cdprobe_run is 2, and each run adds 1 */
  uint32_t rounds;                      /* tournament rounds (N-1 for even N) */
  uint32_t phases;                      /* device phases executed */
  uint32_t launches;                    /* kernels launched by this call (one per local rank) */
  uint32_t aborted;                     /* 1: a device watchdog fired */
  uint32_t warmed;                      /* 1: this run streamed the link wake-up prefix (phase 0) */
  uint32_t reserved1;
  double probe_ms;                      /* host wall clock of this cdprobe_run call, up to the moment every local row is
                                           published; the kernels retire after it, so event_ms may exceed it by a few us */
  double device_ms[CDPROBE_MAX_GPUS];   /* per local rank: first barrier release -> last arrive (%globaltimer) */
  double barrier_us[CDPROBE_MAX_GPUS];  /* per local rank: sum of (release - arrive) over all barriers */
  double event_ms[CDPROBE_MAX_GPUS];    /* per local rank: kernel duration by CUDA events on the launch stream
                                           (only with CDPROBE_OPT_EVENT_TIMING; 0 otherwise) */
  float min_gbps_read;                  /* over filled off-diagonal cells (diagonal when n == 1) */
  float min_gbps_write;
  float gate_gbps_read;                 /* the GB/s threshold this run's verdict applied to reads (0: bandwidth not judged) */
  float gate_gbps_write;
  double kernel_ms[CDPROBE_MAX_GPUS];   /* per local rank: CTA 0 entering the kernel -> result row published (%globaltimer);
                                           event_ms - kernel_ms = launch and completion latency outside the kernel,
                                           kernel_ms - device_ms = residency barrier before the first phase + row output */
  uint32_t unreachable_pairs;           /* filled off-diagonal cells with reach_read & reach_write == 0 (MIG-excluded cells not counted) */
  uint32_t slow_pairs;                  /* filled off-diagonal cells that are reachable but under the gate */
} cdprobe_result_t;

typedef struct {
  uint32_t abi;
  uint32_t n;                           /* total ranks */
  uint32_t n_local;
  uint32_t first_local_rank;
  int32_t ordinal[CDPROBE_MAX_GPUS];    /* per local rank */
  uint32_t sm_count[CDPROBE_MAX_GPUS];
  uint32_t ctas[CDPROBE_MAX_GPUS];
  uint32_t mig[CDPROBE_MAX_GPUS];
  char uuid[CDPROBE_MAX_GPUS][48];      /* "GPU-xxxxxxxx-xxxx-xxxx-xxxx-xxxxxxxxxxxx" per local rank */
  uint32_t handle_type;                 /* 0 none (in-process), 1 POSIX fd, 8 fabric */
  uint32_t path;                        /* 0 TMA bulk, 1 ld/st */
  uint64_t bytes_per_pair;
  uint64_t alloc_bytes;                 /* HBM per rank */
  uint64_t src_sum[CDPROBE_MAX_GPUS][CDPROBE_MAX_GPUS]; /* [local rank][slice]: device-computed checksum S of the source slices */
  uint64_t src_xor[CDPROBE_MAX_GPUS][CDPROBE_MAX_GPUS];
  uint32_t n_slices;
  uint32_t smem_bytes;
  double open_ms;                       /* contexts + VMM + mapping */
  double fill_ms;                       /* pattern fill + slice checksums */
} cdprobe_info_t;

/* Plan (host-only arithmetic; usable without a GPU). */
typedef struct {
  uint32_t abi;
  uint32_t n;
  uint32_t rounds;
  uint32_t n_slots;                     /* landing slots per rank */
  uint32_t n_slices;                    /* source slices per rank */
  uint32_t reserved;
  uint64_t bytes_per_pair;
  uint64_t src_bytes;
  uint64_t land_bytes;
  int8_t partner[CDPROBE_MAX_GPUS][CDPROBE_MAX_GPUS]; /* [round][rank], -1 = idle */
} cdprobe_plan_t;

/* Per-phase timeline of the last run of one local rank (ns, relative to the first barrier release). */
typedef struct {
  uint32_t abi;
  uint32_t n_phases;
  uint8_t kind0[CDPROBE_MAX_PHASES], kind1[CDPROBE_MAX_PHASES];  /* 0 none, 1 read, 2 write, 3 verify, 4 warm-up */
  int8_t peer0[CDPROBE_MAX_PHASES], peer1[CDPROBE_MAX_PHASES];
  uint8_t sync_all[CDPROBE_MAX_PHASES];                          /* closing barrier spans all ranks */
  uint16_t sync_mask[CDPROBE_MAX_PHASES];                        /* ranks of the closing barrier's flag exchange */
  uint16_t post_mask[CDPROBE_MAX_PHASES];                        /* ranks only signalled at the closing barrier (no wait) */
  uint64_t t_start[CDPROBE_MAX_PHASES];                          /* opening barrier released */
  uint64_t t_end0[CDPROBE_MAX_PHASES], t_end1[CDPROBE_MAX_PHASES]; /* last CTA of job 0 / job 1 done */
  uint64_t t_arrive[CDPROBE_MAX_PHASES];                         /* every local CTA reached the closing barrier */
} cdprobe_trace_t;

/* The phase table of one rank (host-only; what cdprobe_run hands to that rank's kernel when every pair is mapped). */
typedef struct {
  uint32_t abi;
  uint32_t n_phases;
  uint32_t peer_mask;                              /* ranks in this rank's cross-GPU barrier */
  uint32_t reserved;
  uint8_t kind[2][CDPROBE_MAX_PHASES];             /* [job][phase]: 0 none, 1 read, 2 write, 3 verify, 4 warm-up */
  int8_t peer[2][CDPROBE_MAX_PHASES];              /* rank whose memory the job touches */
  uint8_t slot[2][CDPROBE_MAX_PHASES];             /* landing slot (write/verify) or source slice (read/warm) */
  uint8_t writer[2][CDPROBE_MAX_PHASES];           /* verify: the rank that wrote the slot */
  uint16_t cta0[2][CDPROBE_MAX_PHASES], nctas[2][CDPROBE_MAX_PHASES];
  uint8_t sync_all[CDPROBE_MAX_PHASES];            /* closing barrier spans all ranks */
  uint16_t sync_mask[CDPROBE_MAX_PHASES];          /* ranks this rank exchanges flags with when the phase closes */
  uint16_t post_mask[CDPROBE_MAX_PHASES];          /* ranks it only signals then (no wait) */
  uint8_t wait_barrier[2][CDPROBE_MAX_PHASES];     /* [job][phase] verify jobs: 1-based barrier index whose signal from
                                                      `writer` the job waits for before reading the slot (0 = none) */
} cdprobe_schedule_t;

/* Node topology as NVML reports it (no CUDA; internal/common topology enumeration, SURVEY §8f n2). */
typedef struct {
  uint32_t abi;
  uint32_t n;                                     /* GPUs NVML enumerates, in NVML index order */
  char uuid[CDPROBE_MAX_GPUS][96];                /* nvmlDeviceGetUUID */
  char pci_bus_id[CDPROBE_MAX_GPUS][32];
  uint8_t mig[CDPROBE_MAX_GPUS];                  /* MIG mode currently enabled */
  uint8_t links_active[CDPROBE_MAX_GPUS];         /* NvLinkState == ENABLED over the 18 links */
  uint32_t link_mask[CDPROBE_MAX_GPUS];           /* bit l set: link l is ENABLED (which physical link is down, not only how many) */
  uint8_t fabric_state[CDPROBE_MAX_GPUS];         /* nvmlGpuFabricInfo_t.state */
  char clique_id[96];                             /* "<clusterUUID>.<cliqueId>" or "" (nvlib.go:208-363) */
  char clique_error[160];                         /* non-empty: getCliqueID would return this error */
} cdprobe_topology_t;

/* Diagnosis of one cell (cdprobe_diagnose): its region re-read after a run and compared word for word with the
 * pattern it must hold.  A word that differs is classified, in this order: */
#define CDPROBE_DIAG_SAMPLES 16
#define CDPROBE_DIAG_FLIP 0u       /* none of the below: bits of the expected word flipped */
#define CDPROBE_DIAG_ZERO 1u       /* word is 0 (never written since open) */
#define CDPROBE_DIAG_DISPLACED 2u  /* the expected pattern's word from another index */
#define CDPROBE_DIAG_STALE 3u      /* write cells: this writer's pattern from one of the 8 runs before */
#define CDPROBE_DIAG_FOREIGN 4u    /* another rank's pattern */
typedef struct {
  uint64_t offset;                      /* bytes from the region start */
  uint64_t expected, observed;
  uint64_t word;                        /* DISPLACED/STALE/FOREIGN: the pattern index that produced `observed`
                                           (read cells: index in that rank's source buffer; write cells: in the slot) */
  uint64_t run_seq;                     /* STALE: the run that wrote it (0 otherwise) */
  uint32_t kind;                        /* CDPROBE_DIAG_* */
  int32_t rank;                         /* whose pattern it is (-1 for FLIP/ZERO) */
} cdprobe_diag_sample_t;

typedef struct {
  uint32_t abi;
  uint32_t op;                          /* CDPROBE_OP_READ or CDPROBE_OP_WRITE */
  uint32_t issuer, target, reader;
  uint32_t n_samples;                   /* min(CDPROBE_DIAG_SAMPLES, bad_words) */
  uint64_t run_seq;                     /* the run whose pattern is expected (the last cdprobe_run) */
  uint64_t region_offset;               /* region start in the target's allocation */
  uint64_t bytes;                       /* region size (bytes_per_pair) */
  uint64_t bad_words;                   /* 64-bit words that differ from the pattern */
  uint64_t bad_granules;                /* 16 KiB granules (from the region start) holding a bad word */
  uint64_t zero_words;                  /* bad words that read 0 */
  uint64_t first_bad, last_bad;         /* byte offsets of the first / last bad word; UINT64_MAX / 0 when clean */
  uint64_t kind_count[5];               /* bad words per CDPROBE_DIAG_* class */
  uint64_t bit_flips[64];               /* FLIP words only: how often bit b differed */
  double ms;                            /* CUDA-event time of the diagnosis on the reader's stream */
  cdprobe_diag_sample_t sample[CDPROBE_DIAG_SAMPLES]; /* the lowest-offset bad words, in offset order */
} cdprobe_diag_t;

/* Dependent-load latency per ordered pair (cdprobe_latency): issuer i's GPU chases `hops` 8-byte loads through its
 * own mapping of target j's source slice, each address taken from the word the load before returned (DESIGN §5c).
 * Matrices are row-major [issuer * CDPROBE_MAX_GPUS + target], like cdprobe_result_t. */
typedef struct {
  uint32_t abi;
  uint32_t n;                           /* total ranks in the domain */
  uint32_t row_mask;                    /* bit r set: row r is filled in (the rows of this process's ranks) */
  uint32_t hops, reps;                  /* as applied: 0 -> 1024 and 8; hops in [1, 1 << 20], reps in [1, 64] */
  uint32_t reserved;
  uint64_t region_bytes;                /* bytes one chase ranges over (bytes_per_pair) */
  uint8_t measured[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];  /* 1: the cell was chased */
  int32_t status[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];    /* 0 ok; CDPROBE_ERR_INTEGRITY: the digest differs from the
                                                             pattern's; CDPROBE_ERR_TIMEOUT: the chase passed timeout_ms;
                                                             else the mapping's status as in cdprobe_result_t */
  float ns_min[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];      /* ns per hop over the timed reps (0 when not timed) */
  float ns_median[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];   /* element reps / 2 of the sorted reps */
  float ns_max[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];
  uint64_t digest[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];   /* xor of every loaded word, warm-up rep included */
  double ms;                            /* host wall clock of the call */
} cdprobe_latency_t;

/* Signal round trip per ordered pair (cdprobe_pingpong): initiator i stores a word into its line in target j's
 * memory, j polls its local copy and stores the echo into its line in i's memory, i polls for the echo — the K3
 * barrier's signal, both ways (DESIGN §5d).  Matrices are row-major [initiator * CDPROBE_MAX_GPUS + target]. */
typedef struct {
  uint32_t abi;
  uint32_t n;                           /* total ranks in the domain */
  uint32_t row_mask;                    /* bit r set: row r is filled in (the rows of this process's ranks) */
  uint32_t trips, reps;                 /* as applied: 0 -> 256 and 8; trips in [1, 1 << 16], reps in [1, 64] */
  uint32_t fenced;                      /* 1: fence.sys before every store (the barrier's signal after a publication) */
  uint64_t call_seq;                    /* 1-based count of cdprobe_pingpong calls on this handle, equal in every
                                           process (0 when the call was refused) */
  uint8_t measured[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];  /* 1: the cell's round trips ran */
  int32_t status[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];    /* 0 ok; CDPROBE_ERR_INTEGRITY: an echo or the digest differs
                                                             from the expected words; CDPROBE_ERR_TIMEOUT: a poll passed
                                                             timeout_ms; else the pair's mapping status */
  float ns_min[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];      /* ns per round trip over the timed reps (0 when not timed) */
  float ns_median[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];   /* element reps / 2 of the sorted reps */
  float ns_max[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];
  uint64_t digest[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];   /* xor of every echo word the initiator received, warm-up
                                                             rep included */
  double ms;                            /* host wall clock of the call */
} cdprobe_pingpong_t;

/* Remote atomics per ordered pair (cdprobe_atomics): issuer i's GPU runs system-scope 64-bit atomics on cell (i, j)'s
 * own word in target j's memory, through i's mapping of j; the owner's L2 performs them and returns each result to i
 * (DESIGN §5e).  Matrices are row-major [issuer * CDPROBE_MAX_GPUS + target]. */
#define CDPROBE_ATOMIC_FETCH_ADD 0u   /* one lane: a dependent atom.add chain, op k returns start + k */
#define CDPROBE_ATOMIC_CAS 1u         /* one lane: a dependent atom.cas chain, every CAS must succeed */
#define CDPROBE_ATOMIC_CONTENDED 2u   /* 32 lanes of one warp: fetch-add chains on the same word */
typedef struct {
  uint32_t abi;
  uint32_t n;                           /* total ranks in the domain */
  uint32_t row_mask;                    /* bit r set: row r is filled in (the rows of this process's ranks) */
  uint32_t kind;                        /* CDPROBE_ATOMIC_* */
  uint32_t ops, reps;                   /* as applied: 0 -> 1024 and 8; ops in [1, 1 << 16] per lane, reps in [1, 64] */
  uint32_t lanes;                       /* lanes issuing atomics: 1, or 32 for CDPROBE_ATOMIC_CONTENDED */
  uint32_t reserved;
  uint64_t call_seq;                    /* 1-based count of cdprobe_atomics calls on this handle (0: refused) */
  uint8_t measured[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];  /* 1: the cell's atomics ran */
  uint8_t native[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];    /* 1: same device, or CUDA reports native atomics for the pair;
                                                             0: CUDA reports none (the cell is not run); 2: the target's
                                                             device is not visible in this process (the cell runs) */
  int32_t status[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];    /* 0 ok; CDPROBE_ERR_INTEGRITY: a return, the read-back or the
                                                             digest differs from the expected values; CDPROBE_ERR_TIMEOUT:
                                                             the cell passed timeout_ms; CDPROBE_ERR_UNSUPPORTED: no
                                                             native atomics; else the mapping's status */
  float ns_min[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];      /* ns per atomic over the timed reps (0 when not timed);
                                                             CONTENDED: per atomic on one word under 32-way contention */
  float ns_median[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];   /* element reps / 2 of the sorted reps */
  float ns_max[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];
  uint64_t digest[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];   /* xor of every value the atomics returned, warm-up rep
                                                             included */
  double ms;                            /* host wall clock of the call */
} cdprobe_atomics_t;

/* Bandwidth versus transfer size per ordered pair (cdprobe_bwcurve): issuer i's GPU reads growing prefixes of the
 * source slice it reads from target j, through i's mapping of j, on the probe's read data path and grid (DESIGN §5f).
 * Cells are row-major [issuer * CDPROBE_MAX_GPUS + target]; size k of a cell is [cell][k]. */
#define CDPROBE_BWCURVE_MAX_SIZES 24  /* bytes_per_pair up to 32 GiB */
typedef struct {
  uint32_t abi;
  uint32_t n;                           /* total ranks in the domain */
  uint32_t row_mask;                    /* bit r set: row r is filled in (the rows of this process's ranks) */
  uint32_t reps;                        /* as applied: 0 -> 8; in [1, 64] */
  uint32_t n_sizes;                     /* entries of size[] */
  uint32_t path;                        /* the read data path used (CDPROBE_OPT_PATH) */
  uint64_t call_seq;                    /* 1-based count of cdprobe_bwcurve calls on this handle, equal in every
                                           process (0 when the call was refused) */
  uint64_t size[CDPROBE_BWCURVE_MAX_SIZES]; /* bytes read per rep: 4096 << k for every 4096 << k < bytes_per_pair,
                                               then bytes_per_pair */
  uint8_t measured[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];  /* 1: the cell ran */
  int32_t status[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];    /* 0 ok; CDPROBE_ERR_INTEGRITY: some rep's (S, X) differs from
                                                             the pattern's; CDPROBE_ERR_TIMEOUT: the cell's kernel passed
                                                             timeout_ms (no times); else the mapping's status */
  uint32_t bad_sizes[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS]; /* bit k set: a rep of size[k], warm-up included, read a
                                                              checksum other than the pattern's */
  float t0_ns[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];       /* ns_median of size[0] */
  float peak_gbps[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];   /* max over k of size[k] / ns_median[k] (bytes per ns) */
  uint64_t half_bytes[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS]; /* the smallest size[k] whose size[k] / ns_median[k]
                                                               reaches peak / 2 (computed before peak is rounded) */
  float ns_min[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];    /* ns per rep over the timed reps
                                                                                      (0 when not timed) */
  float ns_median[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* element reps / 2 of the sorted
                                                                                      reps */
  float ns_max[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];
  uint64_t sum[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];    /* checksum S the last timed rep
                                                                                      read */
  uint64_t xr[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];     /* checksum X */
  double ms;                            /* host wall clock of the call */
} cdprobe_bwcurve_t;

/* One-shot all-reduce across the domain (cdprobe_allreduce): every rank r reads the first size bytes of every rank's
 * source buffer, its own and the peers' through its mappings, and sums them word by word mod 2^64 into its own memory
 * (DESIGN §5g).  Rows are ranks: entry [r] is rank r, and size k of rank r is [r][k].  The times are per rank; the
 * algorithm bandwidth is size / ns, and each rank's NVLink ingress is (n - 1) x that. */
typedef struct {
  uint32_t abi;
  uint32_t n;                           /* total ranks in the domain */
  uint32_t row_mask;                    /* bit r set: row r is filled in (the rows of this process's ranks) */
  uint32_t reps;                        /* as applied: 0 -> 8; in [1, 64] */
  uint32_t n_sizes;                     /* entries of size[] */
  uint32_t path;                        /* the read data path used (CDPROBE_OPT_PATH); cdprobe_allreduce_ll,
                                           cdprobe_allreduce_ring and cdprobe_allreduce_nvls have one data path each,
                                           ignore CDPROBE_OPT_PATH and report CDPROBE_ALLREDUCE_PATH_LL,
                                           CDPROBE_ALLREDUCE_PATH_RING and CDPROBE_ALLREDUCE_PATH_NVLS */
  uint64_t call_seq;                    /* 1-based count of cdprobe_allreduce calls on this handle, equal in every
                                           process (0 when the call was refused); of cdprobe_allreduce_twoshot,
                                           cdprobe_allreduce_ll, cdprobe_allreduce_ring, cdprobe_allreduce_push or
                                           cdprobe_allreduce_nvls calls for those */
  uint64_t size[CDPROBE_BWCURVE_MAX_SIZES]; /* bytes per input and of the output per rep: the cdprobe_bwcurve ladder */
  uint8_t measured[CDPROBE_MAX_GPUS];   /* 1: the rank ran */
  int32_t status[CDPROBE_MAX_GPUS];     /* 0 ok; CDPROBE_ERR_INTEGRITY: some rep's (S, X) or the word check differs from
                                           the pattern's sum; CDPROBE_ERR_TIMEOUT: the rank's kernel passed timeout_ms
                                           (no times); else the mapping status of the domain's first cell that is down,
                                           row-major, which stops every rank */
  uint32_t bad_sizes[CDPROBE_MAX_GPUS]; /* bit k set: a rep of size[k], warm-up included, stored an output whose (S, X)
                                           differs, or the word check of size[k] found a bad word */
  float t0_ns[CDPROBE_MAX_GPUS];        /* ns_median of size[0] */
  float peak_gbps[CDPROBE_MAX_GPUS];    /* max over k of size[k] / ns_median[k] (bytes per ns): algorithm bandwidth */
  uint64_t half_bytes[CDPROBE_MAX_GPUS]; /* the smallest size[k] whose size[k] / ns_median[k] reaches peak / 2
                                            (computed before peak is rounded) */
  float ns_min[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];    /* ns per rep over the timed reps (0 when not timed) */
  float ns_median[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* element reps / 2 of the sorted reps */
  float ns_max[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];
  uint64_t sum[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];    /* checksum S of the output the last timed rep stored */
  uint64_t xr[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];     /* checksum X */
  uint64_t bad_words[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* words of that output that differ from the sum of
                                                                      the pattern words (the word check) */
  uint64_t first_bad[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* byte offset of the first of them; UINT64_MAX when
                                                                      clean */
  double ms;                            /* host wall clock of the call */
} cdprobe_allreduce_t;
/* cdprobe_allreduce_t.path of cdprobe_allreduce_ll: flag-carrying 16-byte packets (DESIGN §5j) */
#define CDPROBE_ALLREDUCE_PATH_LL 3u
/* cdprobe_allreduce_t.path of cdprobe_allreduce_ring: 16-byte ld/st, one flag per 8 KiB unit (DESIGN §5k) */
#define CDPROBE_ALLREDUCE_PATH_RING 4u
/* cdprobe_allreduce_t.path of cdprobe_allreduce_nvls: multimem.ld_reduce and multimem.st through a multicast object
 * (DESIGN §5m) */
#define CDPROBE_ALLREDUCE_PATH_NVLS 5u

/* One-shot all-to-all across the domain (cdprobe_alltoall): every rank pushes one block to every peer at once, into the
 * peer's exchange area, and every rank checks every word it receives (DESIGN §5h).  Per-rank entries [r] describe rank
 * r as a sender and are filled by the process that hosts r; per-cell entries [s * CDPROBE_MAX_GPUS + d] describe the
 * block from sender s to receiver d and are filled by the process that hosts the receiver d, which checks them (a cell
 * that does not run also has its cell_status filled by the sender's process).  Size k of an entry is [..][k]. */
typedef struct {
  uint32_t abi;
  uint32_t n;                           /* total ranks in the domain */
  uint32_t row_mask;                    /* bit r set: rank r's entries, and the cells it receives, are filled in */
  uint32_t reps;                        /* as applied: 0 -> 8; in [1, 64] */
  uint32_t n_sizes;                     /* entries of size[] */
  uint32_t path;                        /* the write data path used (CDPROBE_OPT_PATH) */
  uint64_t call_seq;                    /* 1-based count of cdprobe_alltoall calls on this handle, equal in every
                                           process (0 when the call was refused) */
  uint64_t area_bytes;                  /* this rank's exchange area: n x bytes_per_pair rounded up to 2 MiB */
  uint64_t size[CDPROBE_BWCURVE_MAX_SIZES]; /* bytes per block per rep: the cdprobe_bwcurve ladder */
  /* per rank, as the sender */
  uint8_t measured[CDPROBE_MAX_GPUS];   /* 1: the rank's kernel ran */
  int32_t status[CDPROBE_MAX_GPUS];     /* 0 ok; CDPROBE_ERR_TIMEOUT: the rank's kernel passed timeout_ms (no times) */
  uint32_t blocks[CDPROBE_MAX_GPUS];    /* blocks the rank pushes per rep: its cells that run */
  float t0_ns[CDPROBE_MAX_GPUS];        /* ns_median of size[0] */
  float peak_gbps[CDPROBE_MAX_GPUS];    /* max over k of blocks x size[k] / ns_median[k] (bytes per ns): egress */
  uint64_t half_bytes[CDPROBE_MAX_GPUS]; /* the smallest size[k] whose egress rate reaches peak / 2 (computed before
                                            peak is rounded) */
  float ns_min[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];    /* ns per rep over the timed reps (0 when not timed) */
  float ns_median[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* element reps / 2 of the sorted reps */
  float ns_max[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];
  /* per cell [sender * CDPROBE_MAX_GPUS + receiver] */
  uint8_t cell_measured[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS]; /* 1: the block was pushed and checked */
  int32_t cell_status[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];   /* 0 ok; CDPROBE_ERR_INTEGRITY: a word check found a bad
                                                                 word; CDPROBE_ERR_TIMEOUT: the receiver's kernel passed
                                                                 timeout_ms; else (cell_measured 0) the sender's mapping
                                                                 status of the receiver, probe allocation or exchange
                                                                 area */
  uint32_t bad_sizes[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];    /* bit k set: some rep of size[k], warm-up included,
                                                                 delivered a bad word */
  uint64_t bad_words[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* words of the block that differ
                                                                 from the pattern, summed over every rep of size[k] */
  uint64_t first_bad[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* byte offset of the lowest of
                                                                 them; UINT64_MAX when clean */
  uint64_t sum[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* checksum S of the block as the
                                                                 receiver read it in the last timed rep */
  uint64_t xr[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];  /* checksum X */
  double ms;                            /* host wall clock of the call */
} cdprobe_alltoall_t;

/* Copy-engine bandwidth versus transfer size per ordered pair (cdprobe_memcpy): issuer i's stream copies growing
 * prefixes of a source slice with cudaMemcpyAsync, from target j into i's exchange area (a pull, CDPROBE_OP_READ) or
 * from i into j's (a push, CDPROBE_OP_WRITE), and i's GPU checks every word that landed (DESIGN §5n).  Cells are
 * row-major [issuer * CDPROBE_MAX_GPUS + target]; size k of a cell is [cell][k]. */
typedef struct {
  uint32_t abi;
  uint32_t n;                           /* total ranks in the domain */
  uint32_t row_mask;                    /* bit r set: row r is filled in (the rows of this process's ranks) */
  uint32_t reps;                        /* as applied: 0 -> 8; in [1, 64] */
  uint32_t n_sizes;                     /* entries of size[] */
  uint32_t op;                          /* as passed: CDPROBE_OP_READ (pull) or CDPROBE_OP_WRITE (push) */
  uint64_t call_seq;                    /* 1-based count of cdprobe_memcpy calls on this handle, equal in every
                                           process (0 when the call was refused) */
  uint64_t area_bytes;                  /* this rank's exchange area (cdprobe_alltoall's): n x bytes_per_pair rounded
                                           up to 2 MiB */
  uint64_t size[CDPROBE_BWCURVE_MAX_SIZES]; /* bytes copied per rep: the cdprobe_bwcurve ladder */
  uint8_t measured[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];  /* 1: the cell ran */
  int32_t status[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];    /* 0 ok; CDPROBE_ERR_INTEGRITY: some rep of some size landed a
                                                             word other than the pattern's; CDPROBE_ERR_TIMEOUT: an
                                                             (S, X) read of the cell passed timeout_ms (no times); else
                                                             the status of the issuer's probe or exchange-area mapping */
  uint32_t bad_sizes[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS]; /* bit k set: a rep of size[k], warm-up included, landed a
                                                              bad word or an (S, X) other than the pattern's */
  float t0_ns[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];       /* ns_median of size[0] */
  float peak_gbps[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];   /* max over k of size[k] / ns_median[k] (bytes per ns) */
  uint64_t half_bytes[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS]; /* the smallest size[k] whose size[k] / ns_median[k]
                                                               reaches peak / 2 (computed before peak is rounded) */
  float ns_min[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];    /* ns per copy over the timed reps, by
                                                                                      CUDA events (0 when not timed) */
  float ns_median[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* element reps / 2 of the sorted
                                                                                      reps */
  float ns_max[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];
  uint64_t sum[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];    /* checksum S of the destination as
                                                                                      the check read it, last timed rep */
  uint64_t xr[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];     /* checksum X */
  uint64_t bad_words[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* destination words that differ
                                                                   from the pattern, summed over every rep of size[k],
                                                                   warm-up included */
  uint64_t first_bad[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* byte offset of the lowest of
                                                                   them; UINT64_MAX when clean */
  double ms;                            /* host wall clock of the call */
} cdprobe_memcpy_t;

/* Copy-engine all-to-all across the domain (cdprobe_ce_alltoall): in every rep, every cell of the domain copies its
 * block at once, each on its issuer's copy stream of its own, and the ranks signal each other with stream memory
 * operations, GPU to GPU (DESIGN §5p).  The cells are cdprobe_memcpy's.  Per-rank entries [r] describe rank r's rep,
 * from its release until its own copies are complete and every block addressed to it has landed, and are filled by
 * the process that hosts r.  Per-cell entries [issuer * CDPROBE_MAX_GPUS + target] describe the block of cell (issuer,
 * target): its check fields (cell_measured, cell_status, bad_sizes, bad_words, first_bad, sum, xr) are filled by the
 * process that hosts the rank that owns the block's destination and checks it (the issuer on a pull, the target on a
 * push), its copy times (copy_ns_median) by the process that hosts the issuer.  Size k of an entry is [..][k]. */
typedef struct {
  uint32_t abi;
  uint32_t n;                           /* total ranks in the domain */
  uint32_t row_mask;                    /* bit r set: rank r's entries, the copy times of the cells it issues and the
                                           checks of the blocks it owns are filled in */
  uint32_t reps;                        /* as applied: 0 -> 8; in [1, 64] */
  uint32_t n_sizes;                     /* entries of size[] */
  uint32_t op;                          /* as passed: CDPROBE_OP_READ (pull) or CDPROBE_OP_WRITE (push) */
  uint64_t call_seq;                    /* 1-based count of cdprobe_ce_alltoall calls on this handle, equal in every
                                           process (0 when the call was refused) */
  uint64_t area_bytes;                  /* this rank's exchange area (cdprobe_alltoall's): n x bytes_per_pair rounded
                                           up to 2 MiB */
  uint64_t size[CDPROBE_BWCURVE_MAX_SIZES]; /* bytes per block per rep: the cdprobe_bwcurve ladder */
  /* per rank */
  uint8_t measured[CDPROBE_MAX_GPUS];   /* 1: the rank's reps ran */
  int32_t status[CDPROBE_MAX_GPUS];     /* 0 ok; else (measured 0) the status of the domain's first down probe or
                                           exchange-area mapping, row-major */
  uint32_t blocks[CDPROBE_MAX_GPUS];    /* blocks the rank copies per rep: the cells it issues */
  float t0_ns[CDPROBE_MAX_GPUS];        /* ns_median of size[0] */
  float peak_gbps[CDPROBE_MAX_GPUS];    /* max over k of blocks x size[k] / ns_median[k] (bytes per ns) */
  uint64_t half_bytes[CDPROBE_MAX_GPUS]; /* the smallest size[k] whose rate reaches peak / 2 (computed before peak is
                                            rounded) */
  float ns_min[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];    /* ns per rep over the timed reps, by CUDA events A and
                                                                   B on the rank's stream (0 when not timed) */
  float ns_median[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* element reps / 2 of the sorted reps */
  float ns_max[CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];
  /* per cell [issuer * CDPROBE_MAX_GPUS + target] */
  uint8_t cell_measured[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS]; /* 1: the block was copied and checked */
  int32_t cell_status[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];   /* 0 ok; CDPROBE_ERR_INTEGRITY: some rep of some size
                                                                 landed a bad word or an (S, X) other than the
                                                                 pattern's; CDPROBE_ERR_TIMEOUT: an (S, X) read of the
                                                                 block passed timeout_ms; else (cell_measured 0) the
                                                                 status of the domain's first down mapping */
  uint32_t bad_sizes[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS];    /* bit k set: a rep of size[k], warm-up included, landed
                                                                 a bad word or an (S, X) other than the pattern's */
  float copy_ns_median[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* median ns of the block's
                                                                 copy over the timed reps, by CUDA events on its copy
                                                                 stream */
  uint64_t bad_words[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* words of the block that differ
                                                                 from the pattern, summed over every rep of size[k],
                                                                 warm-up included */
  uint64_t first_bad[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* byte offset of the lowest of
                                                                 them; UINT64_MAX when clean */
  uint64_t sum[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES]; /* checksum S of the block as its owner
                                                                 read it in the last timed rep */
  uint64_t xr[CDPROBE_MAX_GPUS * CDPROBE_MAX_GPUS][CDPROBE_BWCURVE_MAX_SIZES];  /* checksum X */
  double ms;                            /* host wall clock of the call */
} cdprobe_ce_alltoall_t;

/* Per-link NVLink counters of one local device over the last sampled cdprobe_run (cdprobe_links, DESIGN §5o): the
 * difference of two NVML samples, one taken just before the run's clock starts, one just after it stops.  Link l is
 * NVML's scopeId l. */
#define CDPROBE_LINK_REPLAY 0u          /* errors[l][k]: NVML_FI_DEV_NVLINK_ERROR_DL_REPLAY */
#define CDPROBE_LINK_RECOVERY 1u        /*               NVML_FI_DEV_NVLINK_ERROR_DL_RECOVERY */
#define CDPROBE_LINK_CRC 2u             /*               NVML_FI_DEV_NVLINK_ERROR_DL_CRC */
/* failed_fields[l] bits: the field of link l that returned an error in either sample (its delta reads 0) */
#define CDPROBE_LINK_FIELD_TX 0x01u
#define CDPROBE_LINK_FIELD_RX 0x02u
#define CDPROBE_LINK_FIELD_REPLAY 0x04u
#define CDPROBE_LINK_FIELD_RECOVERY 0x08u
#define CDPROBE_LINK_FIELD_CRC 0x10u
typedef struct {
  int32_t status;                       /* 0 ok; CDPROBE_ERR_UNSUPPORTED: NVML is missing, lacks the field entry points,
                                           or has no NVLink field for this GPU (PCIe card, MIG instance); > 0: the
                                           nvmlReturn_t that failed (the handle lookup or the field call) */
  uint32_t rank_mask;                   /* bit r set: rank r runs on this device */
  char uuid[48];                        /* as cdprobe_info reports it */
  uint32_t link_mask;                   /* bit l set: link l was ENABLED at the first sample */
  uint32_t lost_mask;                   /* ENABLED at the first sample, not at the second */
  uint32_t error_mask;                  /* some error counter of link l rose */
  uint32_t reserved;
  uint64_t expected_tx_kib;             /* payload the pass's plan sends from this device to other devices (KiB, rounded
                                           down); barrier flags and read requests are not payload */
  uint64_t expected_rx_kib;             /* payload it receives from other devices */
  uint64_t tx_kib[CDPROBE_NVLINK_MAX_LINKS];  /* NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX delta (KiB) */
  uint64_t rx_kib[CDPROBE_NVLINK_MAX_LINKS];  /* NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_RX delta (KiB) */
  uint64_t errors[CDPROBE_NVLINK_MAX_LINKS][3]; /* [link][CDPROBE_LINK_*] deltas */
  uint32_t failed_fields[CDPROBE_NVLINK_MAX_LINKS]; /* CDPROBE_LINK_FIELD_* bits */
  char remote_bus_id[CDPROBE_NVLINK_MAX_LINKS][32]; /* nvmlDeviceGetNvLinkRemotePciInfo_v2 at the first sample: an
                                                       NVSwitch or a peer GPU; "" when NVML does not say */
} cdprobe_link_device_t;
typedef struct {
  uint32_t abi;
  uint32_t n_devices;                   /* rows of dev[]: the distinct devices of this process's ranks */
  uint64_t run_seq;                     /* the cdprobe_run the deltas cover; 0: no sampled run yet */
  double sample_ms;                     /* host time both samples took */
  cdprobe_link_device_t dev[CDPROBE_MAX_GPUS];
} cdprobe_links_t;

CDPROBE_API uint32_t cdprobe_abi_version(void);
CDPROBE_API const char* cdprobe_strerror(int code);
/* Detail of the last failure on the calling thread ("cuMemMap: CUDA_ERROR_..."), "" if none. */
CDPROBE_API const char* cdprobe_last_error(void);

/* Entry points and the reference interface each one extends or stands in for (paths relative to
 * NVIDIA/k8s-dra-driver-gpu @ 2240711):
 *
 *   cdprobe_open      once per daemon process, from run():          cmd/compute-domain-daemon/main.go:212-347
 *                     (also in the cliqueID == "" branch, main.go:244-250, which today only blocks on ctx)
 *   cdprobe_run       the probe pass; at start and on every daemon-set change delivered by
 *                     GetDaemonInfoUpdateChan():                    cmd/compute-domain-daemon/controller.go:137-139,
 *                     update loops main.go:351-431.  Its verdict is what check() consults next to the IMEX gate:
 *                                                                   cmd/compute-domain-daemon/main.go:435-459
 *   cdprobe_close     on ctx cancel, before the child is stopped:   cmd/compute-domain-daemon/main.go:87-102
 *   cdprobe_topology  NVML device walk + clique id, replaces the ad-hoc walk of getCliqueIDStrict/Legacy:
 *                                                                   cmd/compute-domain-kubelet-plugin/nvlib.go:195-363,
 *                     vendor/github.com/NVIDIA/go-nvlib/pkg/nvlib/device/device.go:268-310,464-495
 *   cdprobe_strerror / cdprobe_last_error   text of the Go error:   fmt.Errorf convention of main.go
 *   cdprobe_remap_peer / cdprobe_unmap_peer  emulate NodeUnprepare/NodePrepare churn around a live domain:
 *                                                                   cmd/compute-domain-kubelet-plugin/driver.go:165-232
 *   cdprobe_gather, cdprobe_info, cdprobe_trace, cdprobe_set_option, cdprobe_corrupt, cdprobe_corrupt_landing,
 *   cdprobe_plan, cdprobe_schedule, cdprobe_gate, cdprobe_ce_copy, cdprobe_rendezvous_selftest, cdprobe_diagnose,
 *   cdprobe_latency, cdprobe_pingpong, cdprobe_atomics, cdprobe_bwcurve, cdprobe_allreduce,
 *   cdprobe_allreduce_twoshot, cdprobe_allreduce_ll, cdprobe_allreduce_ring, cdprobe_allreduce_push,
 *   cdprobe_allreduce_nvls, cdprobe_alltoall, cdprobe_memcpy, cdprobe_ce_alltoall, cdprobe_links: diagnostics, benches,
 *   fault injection;
 *   the reference has no counterpart (it has no probe, SURVEY.md F1).
 *   cdprobe_diagnose, cdprobe_latency, cdprobe_pingpong, cdprobe_atomics, cdprobe_bwcurve, cdprobe_allreduce,
 *   cdprobe_allreduce_twoshot, cdprobe_allreduce_ll, cdprobe_allreduce_ring, cdprobe_allreduce_push,
 *   cdprobe_allreduce_nvls, cdprobe_alltoall, cdprobe_memcpy, cdprobe_ce_alltoall and cdprobe_links are optional for
 *   callers: a daemon binds them with dlsym and works without.
 */
CDPROBE_API int cdprobe_open(const cdprobe_config_t* cfg, cdprobe_t** out);
CDPROBE_API int cdprobe_run(cdprobe_t* h, cdprobe_result_t* out);
/* Collective over all processes of the domain: completes rows of other processes. No-op for world_size <= 1. */
CDPROBE_API int cdprobe_gather(cdprobe_t* h, cdprobe_result_t* inout);
CDPROBE_API int cdprobe_info(cdprobe_t* h, cdprobe_info_t* out);
CDPROBE_API int cdprobe_trace(cdprobe_t* h, uint32_t local, cdprobe_trace_t* out);
/* Runtime options (no reopen needed; the bench sweeps them). */
#define CDPROBE_OPT_EVENT_TIMING 1u  /* value 0/1: bracket each kernel with CUDA events, report event_ms */
#define CDPROBE_OPT_CTAS 2u          /* CTAs of the persistent kernel (0 = one per SM; capped at what fits the device);
                                        CDPROBE_ERR_ARG and the handle unchanged for a value over UINT32_MAX */
#define CDPROBE_OPT_PATH 3u          /* 0 = TMA bulk copies, 1 = ld/st.global.v4 (128-bit), 2 = ld/st.global.v4, 32 contiguous bytes per lane */
#define CDPROBE_OPT_TIMEOUT_MS 4u
#define CDPROBE_OPT_OVERLAP_VERIFY 5u /* value 0/1 */
#define CDPROBE_OPT_VERIFY_CTAS 6u   /* CTAs given to the overlapped verify (default 32) */
#define CDPROBE_OPT_UNIDIRECTIONAL 7u /* value 0/1: see CDPROBE_FLAG_UNIDIRECTIONAL */
#define CDPROBE_OPT_WARMUP 8u        /* link wake-up phase: 0 never, 1 auto = after > 5 ms idle (default), 2 always */
#define CDPROBE_OPT_DEBUG_SKIP_RANK 10u /* fault injection: 1-based local rank whose kernel is not launched (0 = off) */
#define CDPROBE_OPT_WARMUP_BYTES 9u  /* bytes each rank streams from its first partner when warming (default 8 MiB, capped at bytes_per_pair) */
#define CDPROBE_OPT_CTAS_RANK 11u    /* value = ((local rank + 1) << 16) | ctas: CTA count of ONE local rank (tests: a throttled issuer);
                                        CDPROBE_ERR_ARG and the handle unchanged when ctas is 0 or value >> 16 is not a
                                        local rank + 1 (bits above 16 included) */
#define CDPROBE_OPT_MIN_FRACTION_PPM 12u /* min_fraction x 1e6 (0 = default) */
#define CDPROBE_OPT_LINK_PEAK_MBPS 13u   /* link_peak_gbps x 1e3 (0 = default reference) */
#define CDPROBE_OPT_SOLO_RANK 14u    /* profiling: 1-based local rank that runs ALONE — only its own read/write jobs, no
                                        cross-GPU barrier, nobody verifies its writes (reach_write stays 0).  A single
                                        self-contained kernel is what `ncu` can replay: NVLink byte counters per launch. */
#define CDPROBE_OPT_ALL_RANK_BARRIERS 15u /* value 0/1: see CDPROBE_FLAG_ALL_RANK_BARRIERS */
#define CDPROBE_OPT_PAIR_BARRIERS 16u     /* value 0/1: see CDPROBE_FLAG_PAIR_BARRIERS */
#define CDPROBE_OPT_PINGPONG_FAULT 17u    /* tests: value = ((initiator + 1) << 32) | ((target + 1) << 16) | trip arms a
                                             skip-ahead echo in cdprobe_pingpong: the responder `target`, in the
                                             process that hosts it, answers that trip of timed rep 1 of cell
                                             (initiator, target) with the echo of trip + 1; 0 disarms */
#define CDPROBE_OPT_ATOMICS_FAULT 18u     /* tests: value = ((issuer + 1) << 16) | (target + 1) arms a lost-step fault in
                                             cdprobe_atomics: in the process that hosts the issuer, the first op of timed
                                             rep 1 of cell (issuer, target) adds 2 (CAS: swaps in v + 2), so exactly
                                             that cell fails its checks; 0 disarms */
#define CDPROBE_OPT_ALLREDUCE_FAULT 19u   /* tests: value = (drop << 48) | ((rank + 1) << 32) | ((k + 1) << 24) | word
                                             arms a fault in cdprobe_allreduce: in the process that hosts `rank`, timed
                                             rep 1 of size[k] adds 1 to output word `word` (< 2^24) before it is stored
                                             (drop 0), or stores nothing of the word's 8 KiB unit (drop 1), so exactly
                                             that row and size fail the word check and rep 1's checksum; 0 disarms */
#define CDPROBE_OPT_ALLTOALL_FAULT 20u    /* tests: value = ((sender + 1) << 40) | ((receiver + 1) << 32) | ((k + 1) << 24)
                                             | word arms a fault in transit in cdprobe_alltoall: in the process that
                                             hosts `sender`, timed rep 1 of size[k] stores word `word` (< 2^24) of
                                             block (sender -> receiver) xored with 1, so exactly that cell and size
                                             fail the receiver's word check; 0 disarms */
#define CDPROBE_OPT_ALLREDUCE_TWOSHOT_FAULT 21u /* tests: value = (drop << 48) | ((receiver + 1) << 32) | ((k + 1) << 24)
                                             | word arms a fault in cdprobe_allreduce_twoshot: in timed rep 1 of size[k],
                                             in the process that hosts the rank whose chunk holds word `word`
                                             (< 2^24), that rank stores the word into receiver's output xored with 1
                                             (drop 0), or skips every store of the word's 8 KiB unit into receiver
                                             (drop 1), so exactly that row and size fail; 0 disarms */
#define CDPROBE_OPT_ALLREDUCE_LL_FAULT 22u /* tests: value = (mode << 48) | ((sender + 1) << 40) | ((receiver + 1)
                                             << 32) | ((k + 1) << 24) | arg arms a fault in cdprobe_allreduce_ll, in
                                             timed rep 1 of size[k], in the process that hosts `sender`: mode 0, the
                                             packet of word `arg` (< 2^24) from sender to receiver (!= sender) carries
                                             its data xored with 1 and the right flags, so exactly that receiver's row
                                             fails at that size; mode 1, the sender waits `arg` us (< timeout_ms / 2)
                                             before its first push of the rep, and every row stays exact; mode 2, in
                                             every rep of size[k], warm-up included, the receiver (== sender) makes no
                                             store to output word `arg` (< size[k] / 8) but still folds it into (S, X),
                                             so exactly that row and size fail the word check; 0 disarms */
#define CDPROBE_OPT_ALLREDUCE_RING_FAULT 23u /* tests: value = (mode << 48) | (phase << 40) | ((sender + 1) << 32) |
                                             ((k + 1) << 24) | arg arms a fault in cdprobe_allreduce_ring, in timed rep
                                             1 of size[k], in the process that hosts `sender`, in phase 0 (the
                                             reduce-scatter) or 1 (the all-gather): mode 0, the sender's push of word
                                             `arg` (< 2^24) to its successor carries it xored with 1 and the right
                                             flag; mode 1, the push stores nothing of the word's 8 KiB unit but still
                                             publishes its flag; mode 2, the sender waits `arg` us (< timeout_ms / 2)
                                             before its first push of the rep, and every row stays exact.  Modes 0 and
                                             1 fail every row in phase 0, and in phase 1 the rows from sender + 1 up to
                                             the rank before the word's chunk owner; 0 disarms */
#define CDPROBE_OPT_ALLREDUCE_PUSH_FAULT 24u /* tests: value = (mode << 48) | ((rank + 1) << 32) | ((k + 1) << 24) |
                                             word arms a fault in cdprobe_allreduce_push, in timed rep 1 of size[k], on
                                             output word `word` (< 2^24): mode 0, sender `rank` contributes its source
                                             word + 1; mode 1, it skips the reduction of the word's 8 KiB unit; mode 2,
                                             it issues that reduction twice (modes 0-2 fail every row); mode 3, the
                                             owner of the word's chunk pushes the word xored with 1 to receiver `rank`
                                             in the all-gather, so only row `rank` fails; 0 disarms */
#define CDPROBE_OPT_ALLREDUCE_NVLS_FAULT 25u /* tests: value = (mode << 48) | ((k + 1) << 24) | word arms a fault in
                                             cdprobe_allreduce_nvls, in timed rep 1 of size[k], on output word `word`
                                             (< 2^24), in the process hosting the owner of the word's chunk: mode 0,
                                             the owner stores the word xored with 1 through the multicast address, so
                                             every row fails at that word; mode 1, it skips the multicast store of the
                                             word's 8 KiB unit, so every row reads that unit as 0s; 0 disarms */
#define CDPROBE_OPT_MEMCPY_FAULT 26u      /* tests: value = (mode << 48) | ((issuer + 1) << 40) | ((target + 1) << 32) |
                                             ((k + 1) << 24) | word arms a fault in cdprobe_memcpy, in timed rep 1 of
                                             size[k] of cell (issuer, target), in the process that hosts the issuer:
                                             mode 0, between the copy and the checks, destination word `word` (< 2^24)
                                             is overwritten with its pattern value xored with 1 (an 8-byte copy from
                                             host memory); mode 1, no copy is queued, so the destination the previous
                                             rep cleared reads as 0s.  Either fails exactly that cell and size; 0
                                             disarms */
#define CDPROBE_OPT_LINK_COUNTERS 27u     /* value 0/1 (default 0): sample every local device's per-link NVLink counters
                                             through NVML around each cdprobe_run, for cdprobe_links.  Turning it on
                                             loads and initialises NVML once and resolves each local device by UUID;
                                             both stay until close.  An NVML failure never fails the call or a run: it
                                             shows in cdprobe_links_t's status */
#define CDPROBE_OPT_CE_ALLTOALL_FAULT 28u /* tests: value = (mode << 48) | ((issuer + 1) << 40) | ((target + 1) << 32) |
                                             ((k + 1) << 24) | arg arms a fault in cdprobe_ce_alltoall, in timed rep 1
                                             of size[k] of cell (issuer, target), in the process that hosts the issuer,
                                             on the cell's copy stream: mode 0, after the copy and before the landed
                                             flag, destination word `arg` (< 2^24) is overwritten with its pattern value
                                             xored with 1 (an 8-byte copy from host memory); mode 1, no copy is queued
                                             but the landed flag is still published, so the destination its owner
                                             cleared reads as 0s; either fails exactly that cell and size.  Mode 2
                                             holds the copy stream on a second host ticket released `arg` us (below
                                             timeout_ms / 2) after the rep's: every cell stays exact, and the rep of
                                             the rank that waits for the block takes at least that long.  0 disarms */
CDPROBE_API int cdprobe_set_option(cdprobe_t* h, uint32_t option, uint64_t value);
/* Copy-engine reference on the probe's own buffers (the same-box ceiling the roofline is quoted against; not part
 * of a probe): copy k moves `bytes` (capped at the source / landing size) `reps` times back to back between local
 * rank local[k] and rank peer[k] — push != 0: local source -> peer landing area, else peer source -> local landing
 * area — on local[k]'s stream.  All n_copies are enqueued before any is waited for (bidirectional: two copies in
 * one call, or one call per process after a host barrier).  ms_out[k] = CUDA-event time of copy k's `reps` copies. */
CDPROBE_API int cdprobe_ce_copy(cdprobe_t* h, uint32_t n_copies, const uint32_t* local, const uint32_t* peer, uint32_t push,
                                uint64_t bytes, uint32_t reps, double* ms_out);
/* Storm/unprepare emulation (SURVEY H10): unmap + remap rank `peer` in local rank `local`'s address space. */
CDPROBE_API int cdprobe_remap_peer(cdprobe_t* h, uint32_t local, uint32_t peer);
/* Fault injection for parity tests: drop local rank's mapping of `peer` (cell becomes unreachable, run still returns). */
CDPROBE_API int cdprobe_unmap_peer(cdprobe_t* h, uint32_t local, uint32_t peer);
/* Fault injection: XOR one 64-bit word of local rank's source buffer (byte_offset from its start) at rest. */
CDPROBE_API int cdprobe_corrupt(cdprobe_t* h, uint32_t local, uint64_t byte_offset, uint64_t xor_mask);
/* Fault injection for tests: on every cdprobe_run until disarmed, right after local rank `local`'s write into
 * `target`'s landing slot has completed and before any rank verifies it, XOR xor_mask[e] into word word[e] of that
 * slot (e < n <= 8).  The writer's published (S, X) is untouched: to the verifier this is a fault in transit, and the
 * run completes normally with that write cell failing.  One cell is armed per handle; arming replaces the previous
 * arming, n = 0 disarms.  While disarmed the kernel only loads the descriptor's count.  CDPROBE_ERR_ARG: bad local or target, n > 8, a
 * word >= bytes_per_pair / 8, a repeated word, a zero mask, or target == the issuer without a loop-back slot;
 * CDPROBE_ERR_STATE: sticky handle, or the issuer does not map the target. */
CDPROBE_API int cdprobe_corrupt_landing(cdprobe_t* h, uint32_t local, uint32_t target, uint32_t n,
                                        const uint64_t* word, const uint64_t* xor_mask);
/* Where and how cell (op, issuer, target) of the last cdprobe_run went wrong: reader (a global rank, local to this
 * process, that maps the target) re-reads the cell's region — the source slice the issuer reads, or the landing slot
 * it writes — and compares it on its GPU with the pattern of that run.  reader = the issuer: what crossed the
 * fabric; reader = the target: what is at rest.  Touches no result, verdict or pattern.  *out is filled with abi, op
 * and the ranks whatever the return code.  CDPROBE_ERR_ARG: bad op, a rank >= n, a reader that is not local;
 * CDPROBE_ERR_STATE: sticky handle, no run yet, or the reader does not map the target. */
CDPROBE_API int cdprobe_diagnose(cdprobe_t* h, uint32_t op, uint32_t issuer, uint32_t target, uint32_t reader,
                                 cdprobe_diag_t* out);
/* Dependent-load latency of every cell whose issuer is local to this process: one untimed warm-up rep, then `reps`
 * timed reps of `hops` dependent loads over the source slice the issuer reads (written only at open, so no run is
 * needed first).  ns per hop by %globaltimer on the issuer; the digest of the loaded words is checked against the
 * pattern (CDPROBE_ERR_INTEGRITY in the cell's status).  A cell whose mapping is down is not read (measured = 0, the
 * mapping status); the diagonal is chased only with a loop-back slice (n == 1 or CDPROBE_FLAG_LOCAL_DIAG).  One-sided,
 * not collective: fills the local rows (row_mask).  Touches no result, pattern, landing slot or run_seq.  *out
 * carries abi and n whatever the return code.  CDPROBE_ERR_ARG: null argument, hops > 1 << 20 or reps > 64;
 * CDPROBE_ERR_STATE: sticky handle. */
CDPROBE_API int cdprobe_latency(cdprobe_t* h, uint32_t hops, uint32_t reps, cdprobe_latency_t* out);
/* Signal round trip of every off-diagonal cell, over the pairs of the tournament (cdprobe_plan partner table): in
 * each round a rank and its partner run two legs, the lower rank initiating first.  A leg is one untimed warm-up rep,
 * then `reps` timed reps of `trips` round trips; ns per round trip by %globaltimer on the initiator.  fenced = 0:
 * st.relaxed.sys stores and ld.acquire.sys polls (the barrier's signal when nothing was published); fenced = 1: a
 * fence.sys before every store (the signal after a publication).  The digest of the echo words is checked against
 * the expected one (CDPROBE_ERR_INTEGRITY in the cell's status).  A pair is exchanged only when both directions are
 * mapped; otherwise both its cells are skipped on both sides (measured = 0, the mapping status).  n == 1 measures
 * nothing.  Collective when world_size > 1: every process calls it with the same arguments, and fills the rows of
 * its own ranks (row_mask).  Touches no result, pattern, landing slot, Ctrl word or run_seq; needs no run first.
 * *out carries abi, n, trips and reps whatever the return code.  CDPROBE_ERR_ARG: null argument, trips > 1 << 16,
 * reps > 64, fenced > 1, arguments that differ between processes, or an armed CDPROBE_OPT_PINGPONG_FAULT whose cell
 * is out of range or whose trip is >= trips - 1 (or == trips - 2 with reps == 1); CDPROBE_ERR_STATE: sticky handle. */
CDPROBE_API int cdprobe_pingpong(cdprobe_t* h, uint32_t trips, uint32_t reps, uint32_t fenced, cdprobe_pingpong_t* out);
/* Remote atomics of every cell whose issuer is local to this process, on the cell's own 8-byte word in the target's
 * memory (no other cell or process touches it).  Each rep opens with an atom.exch of its start value, then `ops`
 * dependent atomics per lane follow: FETCH_ADD and CAS chains on one lane, 32 fetch-add chains on one word for
 * CONTENDED; one untimed warm-up rep, then `reps` timed reps; ns per atomic by %globaltimer on the issuer.  Every
 * return is checked (FETCH_ADD: op k returns start + k; CAS: every compare succeeds; CONTENDED: the warp's returns sum
 * to the range's sum), the word is read back (start + lanes x ops), and the host checks the digest: any difference is
 * CDPROBE_ERR_INTEGRITY in the cell's status.  A cell whose mapping is down, or whose pair CUDA reports without native
 * atomics, is not run; the diagonal runs only with a loop-back slot (n == 1 or CDPROBE_FLAG_LOCAL_DIAG).  One-sided,
 * not collective: fills the local rows (row_mask) and never waits on another rank.  Touches no result, pattern,
 * landing slot, source buffer, Ctrl word, pingpong line or run_seq; needs no run first.  *out carries abi, n, kind,
 * ops and reps whatever the return code.  CDPROBE_ERR_ARG: null argument, kind > 2, ops > 1 << 16, reps > 64, or an
 * armed CDPROBE_OPT_ATOMICS_FAULT that names no cell of the domain; CDPROBE_ERR_STATE: sticky handle. */
CDPROBE_API int cdprobe_atomics(cdprobe_t* h, uint32_t kind, uint32_t ops, uint32_t reps, cdprobe_atomics_t* out);
/* Bandwidth versus transfer size of every cell whose issuer is local to this process: for each size of the ladder,
 * one untimed warm-up rep, then `reps` timed reps, each reading the first size bytes of the source slice the issuer
 * reads from the target (written only at open, so no run is needed first) with the issuer's whole probe grid on the
 * CDPROBE_OPT_PATH data path.  A rep runs between two grid barriers and is timed as a probe phase is, by %globaltimer
 * from the barrier's release to the last CTA's completion.  Every rep's (S, X) is checked against the pattern
 * (bad_sizes, CDPROBE_ERR_INTEGRITY).  The cells run in the tournament's rounds (cdprobe_plan partner table), both
 * ranks of a pair at once, every round after every kernel of the round before has finished in every process; with a
 * loop-back slice (n == 1 or CDPROBE_FLAG_LOCAL_DIAG) a last round reads the diagonal.  A cell whose mapping is down
 * is not read (measured = 0, the mapping status).  A cell whose kernel passes timeout_ms is CDPROBE_ERR_TIMEOUT and the
 * handle stays usable.  Collective when world_size > 1: every process calls it with the same reps, and fills the rows
 * of its own ranks (row_mask).  Touches no result, pattern, landing slot, Ctrl word, pingpong or atomics line, run_seq
 * or warm-up state.  *out carries abi, n and reps whatever the return code.  CDPROBE_ERR_ARG: null argument,
 * reps > 64, bytes_per_pair > 32 GiB, or arguments that differ between processes; CDPROBE_ERR_STATE: sticky
 * handle. */
CDPROBE_API int cdprobe_bwcurve(cdprobe_t* h, uint32_t reps, cdprobe_bwcurve_t* out);
/* One-shot all-reduce of every rank's source buffer, on every rank at once: for each size of the cdprobe_bwcurve
 * ladder, one untimed warm-up rep, then `reps` timed reps.  In a rep, rank r reads the first size bytes of every rank's
 * source buffer (written only at open, so no run is needed first), adding rank r, r + 1, ... (mod n) in that order, on
 * the CDPROBE_OPT_PATH read path with its whole probe grid, and stores the sums with st.global.v4 into its scratch
 * buffer.  A domain barrier opens every rep (flags in the Ctrl granule; only a grid barrier at n == 1), and a rep is
 * timed per rank by %globaltimer from that rank's release to its last CTA's completion; ranks are released a signal
 * latency apart, so no time is domain-wide.  After every rep, warm-up included and untimed, each rank reads back every
 * word of its output, compares it with the pattern's sum and overwrites it with 0, as cdprobe_allreduce_twoshot does,
 * so a unit that a rep does not store reads as 0s; the output also starts zeroed on every call.  Every rep's (S, X) of
 * that read-back is checked against the pattern's sum (bad_sizes, CDPROBE_ERR_INTEGRITY); sum and xr are the last
 * timed rep's, and bad_words and first_bad are summed over every rep of the size, warm-up included.  If any cell of the domain
 * is down (cdprobe_unmap_peer, a failed mapping, MIG), nothing runs: every filled row has measured = 0 and the status
 * of the first such cell, and the call returns CDPROBE_OK.  A rank whose kernel passes timeout_ms is
 * CDPROBE_ERR_TIMEOUT and the handle stays usable.  Collective when world_size > 1: every process calls it with the
 * same reps and fills the rows of its own ranks (row_mask).  The output is bytes_per_pair per rank, so the scratch
 * buffer grows by that much until close (1 GiB at n == 1 with 1 GiB).  Touches no result, pattern, landing slot, Ctrl
 * word, pingpong or atomics line, run_seq, warm-up or bwcurve state.  *out carries abi, n and reps whatever the return
 * code.  CDPROBE_ERR_ARG: null argument, reps > 64, bytes_per_pair > 32 GiB, arguments that differ between processes,
 * or an armed CDPROBE_OPT_ALLREDUCE_FAULT whose rank is >= n, whose k is >= n_sizes, whose word is
 * >= size[k] / 8 or that has a bit above 48 set; CDPROBE_ERR_STATE: sticky handle. */
CDPROBE_API int cdprobe_allreduce(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out);
/* One-shot all-to-all: every rank pushes a block to every peer at once.  For each size of the cdprobe_bwcurve ladder,
 * one untimed warm-up rep, then `reps` timed reps.  In rep r of size k, sender i writes the first size bytes of block
 * (i -> j) at offset i x bytes_per_pair of receiver j's exchange area: the probe's write pattern with the salt
 * write_salt(seed, i, j, alltoall_seq(call_seq, k, r)), whose sequence value has its top bit set, so no rep repeats
 * another's words or a run's.  The blocks of a rank are interleaved unit by unit (rank + 1, rank + 2, ... mod n, then
 * the diagonal) on the CDPROBE_OPT_PATH write path with the rank's whole probe grid.  A rep runs between two domain
 * barriers (flags in the Ctrl granule) and is timed per rank as a probe write phase: from the rank's release to its last
 * CTA's completion stamp, which follows its stores and a fence.sys.  After every rep, warm-up included, every receiver
 * compares every word it received with the pattern.  There is one cell per off-diagonal pair, plus (i, i) with a
 * loop-back slice (n == 1 or CDPROBE_FLAG_LOCAL_DIAG); a cell runs when the sender maps the receiver's probe allocation
 * and exchange area, and otherwise nobody writes or checks it.  If no cell of the domain runs (MIG), no kernel is
 * launched and the call returns CDPROBE_OK.  The exchange area (n x bytes_per_pair per rank, rounded up to 2 MiB) is
 * created on the first call with the probe allocation's handle type, mapped wherever the probe mapping is then up, and
 * kept until close; if creating it fails in any process, every process returns that error, nothing runs, and the next
 * call tries again.  A rank whose kernel passes timeout_ms is CDPROBE_ERR_TIMEOUT and the handle stays usable.
 * Collective when world_size > 1: every process calls it with the same reps.  Needs no run first and touches no
 * result, pattern, source buffer, landing slot, run_seq, warm-up state or other measurement's state.  *out carries abi,
 * n and reps whatever the return code.  CDPROBE_ERR_ARG: null argument, reps > 64, bytes_per_pair > 32 GiB, arguments
 * that differ between processes, or an armed CDPROBE_OPT_ALLTOALL_FAULT that names no cell of the domain, a k >=
 * n_sizes or a word >= size[k] / 8; CDPROBE_ERR_STATE: sticky handle. */
CDPROBE_API int cdprobe_alltoall(cdprobe_t* h, uint32_t reps, cdprobe_alltoall_t* out);
/* Two-shot all-reduce of every rank's source buffer, on every rank at once: a reduce-scatter, then a pushed
 * all-gather.  For each size of the cdprobe_bwcurve ladder, one untimed warm-up rep, then `reps` timed reps.  A size
 * of U = ceil(size / 8 KiB) units is split into chunks: rank r owns units [floor(r U / n), floor((r + 1) U / n)),
 * possibly none.  In a rep, rank r reads its units of every rank's source buffer, adding rank r, r + 1, ... (mod n) as
 * cdprobe_allreduce does on the CDPROBE_OPT_PATH read path with its whole probe grid, and stores each summed unit with
 * st.global.v4 into every rank's gather area, its own first, then r + 1, r + 2, ... (mod n).  Each rank's link
 * traffic per rep is 2 (n - 1) / n x size, the all-reduce's.  Domain barriers open and close every rep (flags in the
 * Ctrl granule; only grid barriers at n == 1), the closing one after a fence.sys in every CTA; a rep is timed per rank
 * by %globaltimer from that rank's opening release to its closing release, when its output is complete.  After every
 * rep, warm-up included and untimed, each rank reads back every word of its output, compares it with the pattern's sum
 * and overwrites it with 0, so a unit that is not delivered in the next rep reads as 0s.  Every rep's (S, X) of that
 * read-back is checked against the pattern's sum (bad_sizes, CDPROBE_ERR_INTEGRITY).  Row r of *out describes what
 * rank r holds at the end of a rep:
 *   sum, xr:              the (S, X) of rank r's whole output as rank r read it back after the last timed rep;
 *   bad_words, first_bad: summed over every rep of the size, warm-up included, as cdprobe_allreduce's;
 *   peak_gbps:            the algorithm bandwidth, size / ns; the nccl-tests bus bandwidth is peak_gbps x 2 (n - 1) / n.
 * The gather area (bytes_per_pair per rank, rounded up to 2 MiB) is created on the first call with the probe
 * allocation's handle type, mapped wherever the probe mapping is then up, and kept until close; if creating it fails
 * in any process, every process returns that error, nothing runs, and the next call tries again.  If any probe or
 * gather-area mapping of the domain is down (cdprobe_unmap_peer, a failed mapping, MIG), nothing runs: every filled
 * row has measured = 0 and the status of the first such cell, and the call returns CDPROBE_OK.  A rank whose kernel
 * passes timeout_ms is CDPROBE_ERR_TIMEOUT and the handle stays usable.  Collective when world_size > 1: every process
 * calls it with the same reps and fills the rows of its own ranks (row_mask); call_seq counts calls of this function.
 * Needs no run first and touches no result, pattern, source buffer, landing slot, run_seq, warm-up state, exchange
 * area or other measurement's state.  *out carries abi, n and reps whatever the return code.  CDPROBE_ERR_ARG: null
 * argument, reps > 64, bytes_per_pair > 32 GiB, arguments that differ between processes, or an armed
 * CDPROBE_OPT_ALLREDUCE_TWOSHOT_FAULT whose receiver is >= n, whose k is >= n_sizes, whose word is >= size[k] / 8 or
 * that has a bit above 48 set; CDPROBE_ERR_STATE: sticky handle. */
CDPROBE_API int cdprobe_allreduce_twoshot(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out);
/* Low-latency ("LL") all-reduce of every rank's source buffer, on every rank at once: no barrier and no fence per
 * rep.  For each size of the LL ladder (the cdprobe_bwcurve ladder's sizes of at most 1 MiB; it ends at 1 MiB when
 * bytes_per_pair is larger), one domain barrier (flags in the Ctrl granule; a grid barrier only at n == 1), then one
 * untimed warm-up rep and `reps` timed reps back to back.  In a rep every 64-bit input word of rank r travels to every
 * peer, r + 1, r + 2, ... (mod n), as one 16-byte packet (st.relaxed.sys.v2.u64) of two 8-byte elements, each 32 bits
 * of data and the rep's 32-bit flag, into the peer's LL area; each rank polls its own area (ld.relaxed.sys.v2.u64)
 * until both flags of every packet are the rep's, adds the packets to its own input and stores the sum into its
 * output.  Rank j's input in a rep is its source word plus a per-rank, per-rep salt, subtracted again from the sum, so
 * a packet of another rep that were accepted would leave a wrong word.  Every rank splits the words alike, over the
 * warps of the domain's smallest grid.  A rep is timed per rank by %globaltimer from the end of that rank's previous
 * rep (the warm-up: from the barrier release) to the moment its output is complete, the per-iteration figure
 * nccl-tests reports.  Every rep's (S, X) is folded from the sums as they are stored and checked (bad_sizes).  After
 * the last rep of a size, untimed, each rank reads back every word of its output, compares it with the pattern's sum
 * and overwrites it with 0 (bad_words, first_bad: that one check), and the output starts zeroed on every call, so a
 * word the last rep of a size does not store is seen; one that only earlier reps of the size miss is not.  sum and xr
 * are the last timed rep's; peak_gbps is the algorithm bandwidth, size / ns, and each rank's link ingress per rep is
 * 2 (n - 1) x size (every 8 bytes of data travel in a 16-byte packet).  The LL area (2 x n x 2 x the ladder's largest size per rank, rounded up
 * to 2 MiB) is created on the first call with the probe allocation's handle type, zeroed, mapped wherever the probe
 * mapping is then up, and kept until close; if creating it fails in any process, every process returns that error,
 * nothing runs, and the next call tries again.  If any probe or LL-area mapping of the domain is down
 * (cdprobe_unmap_peer, a failed mapping, MIG), nothing runs: every filled row has measured = 0 and the status of the
 * first such cell, and the call returns CDPROBE_OK.  A rank whose kernel passes timeout_ms is CDPROBE_ERR_TIMEOUT
 * with no times, the handle stays usable, and every LL area is zeroed before the next call runs.  Collective when
 * world_size > 1: every process calls it with the same reps and fills the rows of its own ranks (row_mask); call_seq
 * counts calls of this function.  Needs no run first and touches no result, pattern, source buffer, landing slot,
 * run_seq, warm-up state, exchange or gather area or other measurement's state.  *out carries abi, n, reps and path
 * whatever the return code.  CDPROBE_ERR_ARG: null argument, reps > 64, bytes_per_pair > 32 GiB, arguments that
 * differ between processes, or an armed CDPROBE_OPT_ALLREDUCE_LL_FAULT whose sender or receiver is >= n, whose k is
 * >= n_sizes, whose mode is above 2, whose mode-0 receiver is its sender, whose mode-2 receiver is not its sender,
 * whose mode-0 or mode-2 word is >= size[k] / 8, or whose mode-1 delay is >= timeout_ms / 2; CDPROBE_ERR_STATE: sticky
 * handle. */
CDPROBE_API int cdprobe_allreduce_ll(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out);
/* Ring all-reduce of every rank's source buffer, on every rank at once: each rank talks only to its successor
 * r + 1 (mod n), to which it pushes, and its predecessor r - 1, which pushes to it.  For each size of the
 * cdprobe_bwcurve ladder, one untimed warm-up rep and `reps` timed reps.  The size is cut into cdprobe_allreduce_twoshot's
 * n chunks of 8 KiB units, and a rep is 2 (n - 1) steps: in the reduce-scatter, step s pushes the partial sum of chunk
 * (r - 1 - s) mod n (the received partial plus rank r's own input) into the successor's ring area, so that rank r
 * ends it holding the full sum of chunk r; in the all-gather, step s pushes the full chunk (r - s) mod n on.  Every
 * 8 KiB unit goes with st.global.v4 and is published by its own flag (st.release.sys) that the receiver polls
 * (ld.acquire.sys) before it reads the unit: no barrier and no fence across the domain between the steps, so a flag
 * that overtook its data would leave stale or zero words.  A fenced domain barrier opens every rep (flags in the Ctrl
 * granule; only a grid barrier at n == 1, where the rank stores its own input into its output).  A rep is timed per
 * rank by %globaltimer from its opening release to the moment its output is complete and its pushes are issued, so a
 * slow hop stretches every rank's rep.  After every rep, warm-up included and untimed, each rank reads back every word
 * of its output, compares it with the pattern's sum and overwrites it with 0, as cdprobe_allreduce_twoshot does; row
 * r of *out is as cdprobe_allreduce_twoshot's.  peak_gbps is the algorithm bandwidth, size / ns; the bus bandwidth is
 * peak_gbps x 2 (n - 1) / n, and each rank sends and receives 2 (n - 1) / n x size per rep over one link each.  The
 * ring area (bytes_per_pair per rank plus one 32-bit flag per 8 KiB of it, rounded up to 2 MiB) is created on the
 * first call with the probe allocation's handle type, zeroed, mapped wherever the probe mapping is then up, and kept
 * until close; if creating it fails in any process, every process returns that error, nothing runs, and the next call
 * tries again.  If any probe or ring-area mapping of the domain is down (cdprobe_unmap_peer, a failed mapping, MIG),
 * nothing runs: every filled row has measured = 0 and the status of the first such cell, and the call returns
 * CDPROBE_OK.  A rank whose kernel passes timeout_ms is CDPROBE_ERR_TIMEOUT with no times, the handle stays usable,
 * and every ring area is zeroed before the next call runs.  Collective when world_size > 1: every process calls it
 * with the same reps and fills the rows of its own ranks (row_mask); call_seq counts calls of this function.  Needs no
 * run first and touches no result, pattern, source buffer, landing slot, run_seq, warm-up state, exchange, gather or
 * LL area or other measurement's state.  *out carries abi, n, reps and path whatever the return code.
 * CDPROBE_ERR_ARG: null argument, reps > 64, bytes_per_pair > 32 GiB, arguments that differ between processes, or an
 * armed CDPROBE_OPT_ALLREDUCE_RING_FAULT whose mode is above 2, whose phase is above 1, whose sender is >= n, whose k
 * is >= n_sizes, whose mode-0 or mode-1 word is >= size[k] / 8, lies in a chunk the sender does not push in that phase
 * or is armed at n == 1, or whose mode-2 delay is >= timeout_ms / 2; CDPROBE_ERR_STATE: sticky handle. */
CDPROBE_API int cdprobe_allreduce_ring(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out);
/* Push all-reduce of every rank's source buffer, on every rank at once, in which every byte moves as a write: a
 * reduce-scatter by remote reductions into each unit's owner, then a pushed all-gather.  For each size of the
 * cdprobe_bwcurve ladder, one untimed warm-up rep and `reps` timed reps.  The size is cut into
 * cdprobe_allreduce_twoshot's chunks of 8 KiB units.  In a rep, rank r first adds every unit u of its own source
 * buffer into the push area of u's owner, at u's place: on the TMA path (CDPROBE_OPT_PATH 0) each unit is bulk-loaded
 * into shared memory and sent with cp.reduce.async.bulk .add.u64, so the memory system that owns the target adds it
 * in; on the ld/st paths (1, 2) each 8-byte word goes with its own red.relaxed.sys.global.add.u64, the paths differing
 * only in the load layout.  Up to n ranks add into the same unit at once.  Once every reduction is performed and
 * fenced, a fenced domain barrier leaves rank r's own chunk holding the full sum, and rank r pushes that chunk with
 * st.global.v4 to every peer, r + 1, r + 2, ... (mod n).  The sums are 64-bit wrapping adds, so their order does not
 * matter and the output is cdprobe_allreduce's word for word.  Each rank's link traffic per rep is
 * 2 (n - 1) / n x size, the two-shot's, with every transfer a write.  Three domain barriers per rep (flags in the Ctrl
 * granule; only grid barriers at n == 1, where the rank reduces its input into its own zeroed area and pushes
 * nothing): a fenced one opens the rep, one follows the reductions and a fenced one closes the rep after a fence.sys
 * in every CTA; a rep is timed per rank by %globaltimer from its opening release to its closing release.  After every
 * rep, warm-up included and untimed, each rank reads back every word of its output, compares it with the pattern's
 * sum and overwrites it with 0, the start the next rep's reductions need; row r of *out is as
 * cdprobe_allreduce_twoshot's, and peak_gbps is the algorithm bandwidth, size / ns (bus bandwidth peak_gbps x
 * 2 (n - 1) / n).  The push area (bytes_per_pair per rank, rounded up to 2 MiB) is created on the first call with the
 * probe allocation's handle type, zeroed, mapped wherever the probe mapping is then up, and kept until close; if
 * creating it fails in any process, every process returns that error, nothing runs, and the next call tries again.
 * If any probe or push-area mapping of the domain is down (cdprobe_unmap_peer, a failed mapping, MIG), or two ranks
 * on different devices this process sees lack native peer atomics (cudaDevP2PAttrNativeAtomicSupported; a rank in
 * another process counts as native), nothing runs: every filled row has measured = 0 and the status of the first
 * such cell (CDPROBE_ERR_UNSUPPORTED for missing atomics), and the call returns CDPROBE_OK.  A rank whose kernel
 * passes timeout_ms is CDPROBE_ERR_TIMEOUT with no times, the handle stays usable, and every push area is zeroed
 * before the next call runs.  Collective when world_size > 1: every process calls it with the same reps and fills the
 * rows of its own ranks (row_mask); call_seq counts calls of this function.  Needs no run first and touches no
 * result, pattern, source buffer, landing slot, run_seq, warm-up state, exchange, gather, LL or ring area or other
 * measurement's state.  *out carries abi, n, reps and path whatever the return code.  CDPROBE_ERR_ARG: null argument,
 * reps > 64, bytes_per_pair > 32 GiB, arguments that differ between processes, or an armed
 * CDPROBE_OPT_ALLREDUCE_PUSH_FAULT whose mode is above 3, whose rank is >= n, whose k is >= n_sizes, whose word is
 * >= size[k] / 8, or whose mode 3 is armed at n == 1 or names the word's owner as receiver; CDPROBE_ERR_STATE: sticky
 * handle. */
CDPROBE_API int cdprobe_allreduce_push(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out);
/* Multicast (NVLS) all-reduce of every rank's source buffer, on every rank at once, through one multicast object that
 * spans the domain: the switch sums and the switch fans out.  For each size of the cdprobe_bwcurve ladder, one untimed
 * warm-up rep and `reps` timed reps.  Each rank has an NVLS area of 2 x s_max bytes (s_max: the ladder's largest
 * size), rounded up to the VMM and multicast granularities, bound into the object at offset 0: its first half is the
 * input, its second the output.  On every call, untimed and before any kernel runs, each rank copies the first s_max
 * bytes of its source buffer into its input half and zeroes its output half.  The size is cut into
 * cdprobe_allreduce_twoshot's chunks of 8 KiB units.  In a rep, rank r reads each word of its own chunk with
 * multimem.ld_reduce .add.u64 through the object, which returns the wrapping 64-bit sum of that word over every
 * member, and stores each summed 16 bytes with one multimem.st into every member's output half at once.  The sums are
 * exact, so the output is cdprobe_allreduce's word for word.  A fenced domain barrier opens the rep, and one closes it
 * after a fence.proxy.alias per thread and a fence.sys per CTA; a rep is timed per rank by %globaltimer from its
 * opening release to its closing release.  After every rep, warm-up included and
 * untimed, each rank reads back every word of its output through its own mapping, compares it with the pattern's sum
 * and overwrites it with 0; row r of *out is as cdprobe_allreduce_twoshot's, path is CDPROBE_ALLREDUCE_PATH_NVLS
 * whatever CDPROBE_OPT_PATH says, and peak_gbps is the algorithm bandwidth, size / ns (bus bandwidth peak_gbps x
 * 2 (n - 1) / n).  The object and the areas are created on the first call that runs, with the probe allocation's
 * handle type (the process hosting rank 0 creates the object and hands it to the others over the rendezvous), and kept
 * until close; if a step fails in any process, every process returns that error, cdprobe_last_error names the step and
 * the CUresult, nothing is kept, and the next call tries again.  When a rank's device reports no multicast support
 * (CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, or a MIG instance), the driver lacks the multicast entry points, or two
 * ranks of the domain share a device (by UUID, across processes), nothing is created and nothing runs: every filled
 * row has measured = 0 and status CDPROBE_ERR_UNSUPPORTED, and the call returns CDPROBE_OK.  The same holds, with
 * cdprobe_last_error naming the CUresult, for a one-rank domain whose driver refuses a multicast object of one device
 * (cuMulticastCreate returns CUDA_ERROR_INVALID_VALUE); that call asks the driver again each time.  Likewise, if any probe
 * mapping of the domain is down, every filled row has the status of the first such cell.  A rank whose kernel passes
 * timeout_ms is CDPROBE_ERR_TIMEOUT with no times and the handle stays usable.  Collective when world_size > 1: every
 * process calls it with the same reps and fills the rows of its own ranks (row_mask); call_seq counts calls of this
 * function.  Needs no run first and touches no result, pattern, source buffer, landing slot, run_seq, warm-up state or
 * other measurement's state.  *out carries abi, n, reps and path whatever the return code.  CDPROBE_ERR_ARG: null
 * argument, reps > 64, bytes_per_pair > 32 GiB, arguments that differ between processes, or an armed
 * CDPROBE_OPT_ALLREDUCE_NVLS_FAULT whose mode is above 1, that sets any of bits 32 to 47, whose k is >= n_sizes or
 * whose word is >= size[k] / 8; CDPROBE_ERR_STATE: sticky handle. */
CDPROBE_API int cdprobe_allreduce_nvls(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out);
/* Copy-engine bandwidth versus transfer size of every cell whose issuer is local to this process, checked word for
 * word: for each size of the cdprobe_bwcurve ladder, one untimed warm-up rep, then `reps` timed reps, each one
 * cudaMemcpyAsync of the first size bytes of a source slice (written only at open, so no run is needed first) on the
 * issuer's stream.  op = CDPROBE_OP_READ pulls: the slice issuer i reads from target j, from j's allocation into block j
 * of i's exchange area.  op = CDPROBE_OP_WRITE pushes: the slice j reads from i, from i's own allocation into block i
 * of j's exchange area.  The exchange area is cdprobe_alltoall's (n x bytes_per_pair per rank, created on the first
 * call of either, collectively, and kept until close; cdprobe_alltoall salts and checks every word it uses, so the two
 * may share it).  The timed part of a rep is queued whole before any of it may start: a stream wait
 * (cuStreamWaitValue64) on a host-mapped ticket word, an event, the copy, an event.  The host then releases the ticket,
 * so the events bracket the copy alone, without the host's enqueue time; ns per rep is their cudaEventElapsedTime,
 * which resolves about 0.5 us, so t0_ns is indicative only.  Once the copy has completed, the untimed checks are queued
 * on the issuer's GPU through its mapping: cdprobe_diagnose's comparison of every destination word with the pattern,
 * cdprobe_bwcurve's (S, X) read of the destination on the issuer's grid and CDPROBE_OPT_PATH data path, and a memset
 * of the destination to 0, so that a copy that does not land in a later rep reads as 0s.  The local ranks of one process are released together; across processes only the
 * domain barrier before each size aligns them.  Every rep, warm-up included, is checked (bad_sizes, bad_words,
 * first_bad, CDPROBE_ERR_INTEGRITY).  The cells run in the tournament's rounds (cdprobe_plan partner table), both ranks
 * of a pair at once, then with a loop-back slice (n == 1 or CDPROBE_FLAG_LOCAL_DIAG) a last round copies the diagonal;
 * a domain barrier opens every round and every size.  A cell runs when the issuer maps the target's probe allocation
 * and exchange area; otherwise nothing is copied (measured = 0, the mapping status).  Nothing is written but the
 * cells' blocks of the exchange area and the issuers' scratch buffers, which grow to hold a diagnosis of
 * bytes_per_pair.  An (S, X) read that passes timeout_ms makes its cell CDPROBE_ERR_TIMEOUT and the handle stays
 * usable; a copy whose closing event has not completed timeout_ms after its release returns CDPROBE_ERR_TIMEOUT and
 * leaves the handle sticky (a copy cannot be aborted).  Collective when world_size > 1: every process calls it with the
 * same op and reps, and fills the rows of its own ranks (row_mask).  Touches no result, pattern, source buffer, landing
 * slot, Ctrl word, run_seq, warm-up state or other measurement's state.  *out carries abi, n, reps and op whatever the
 * return code.  CDPROBE_ERR_ARG: null argument, an op other than CDPROBE_OP_READ or CDPROBE_OP_WRITE, reps > 64,
 * bytes_per_pair > 32 GiB, arguments that differ between processes, or an armed CDPROBE_OPT_MEMCPY_FAULT that names no
 * cell of the domain, a k >= n_sizes or a word >= size[k] / 8, or has a mode above 1; CDPROBE_ERR_TIMEOUT: a copy did
 * not complete (sticky); CDPROBE_ERR_UNSUPPORTED: the driver has no cuStreamWaitValue64; CDPROBE_ERR_CUDA: it
 * refused one (sticky); CDPROBE_ERR_STATE: sticky handle. */
CDPROBE_API int cdprobe_memcpy(cdprobe_t* h, uint32_t op, uint32_t reps, cdprobe_memcpy_t* out);
/* Copy-engine all-to-all across the domain, checked word for word (DESIGN §5p): for each size of the cdprobe_bwcurve
 * ladder, one untimed warm-up rep, then `reps` timed reps, in each of which every cell of cdprobe_memcpy (the same
 * source slice, the same block of the exchange area, the diagonal with a loop-back slice) copies the first size bytes
 * of its slice with cudaMemcpyAsync, all at once.  Each local rank keeps one copy stream per cell it issues, made on
 * the first call and kept until close; its own stream carries the barrier, the joins and the checks.  A rep of rank r,
 * queued whole before the host releases the rep's ticket (cdprobe_memcpy's): its stream waits for the ticket, writes
 * the opening value into line r of every peer's flag lines with cuStreamWriteValue64 through r's mapping and waits
 * (cuStreamWaitValue64, GEQ) for every peer's in its own; event A; each copy stream waits for A, copies between
 * events, and on a push then writes the landed value into line r of the receiver's lines (fenced, so it is ordered
 * after the copy); the stream joins every copy stream and, on a push, waits for every sender's landed value; event B.
 * ns per rep is B - A; copy_ns_median comes from each copy stream's own events (about 0.5 us resolution).  Once every
 * local B has completed, the rank that owns each destination checks it on its own GPU, as cdprobe_memcpy's issuer does:
 * the diagnosis against the pattern, the (S, X) read, the clearing to 0.  The next rep's opening write is queued behind
 * those checks, so no block is copied into before its owner has checked and cleared the last one.  Only the domain
 * barrier before each size is a host collective.  The exchange area is cdprobe_alltoall's and cdprobe_memcpy's. When
 * any probe or exchange-area mapping of the domain is down, nothing runs: every local row and every cell a local rank
 * issues or owns gets the status of the domain's first down cell, row-major, and the call returns CDPROBE_OK.  No
 * kernel runs in the timed window.  Collective when world_size > 1: every process calls it with the same op and reps.
 * Touches no result, pattern, source buffer, landing slot, run_seq, warm-up state or other measurement's lines or
 * areas.  *out carries abi, n, reps and op whatever the return code.  CDPROBE_ERR_ARG: as cdprobe_memcpy, or an armed
 * CDPROBE_OPT_CE_ALLTOALL_FAULT that names no cell of the domain, a k >= n_sizes, a word >= size[k] / 8 (modes 0 and
 * 1), a delay of timeout_ms / 2 or more (mode 2) or a mode above 2; CDPROBE_ERR_UNSUPPORTED (every process): the
 * driver lacks cuStreamWriteValue64 or cuStreamWaitValue64, or some process would hold more streams on one device
 * (each local rank's own and its copy streams) than CUDA_DEVICE_MAX_CONNECTIONS (read at open, default 8) gives
 * hardware queues, so that a stream wait could block a stream sharing its queue (cdprobe_last_error names the need and
 * the limit); CDPROBE_ERR_CUDA: the driver refused a stream memory operation (sticky, the CUresult named);
 * CDPROBE_ERR_TIMEOUT: some rep's B had not completed timeout_ms after its release (sticky; the host writes the awaited
 * values into its own ranks' lines first, so no stream stays blocked); CDPROBE_ERR_STATE: sticky handle. */
CDPROBE_API int cdprobe_ce_alltoall(cdprobe_t* h, uint32_t op, uint32_t reps, cdprobe_ce_alltoall_t* out);
/* The per-link NVLink counters of the last cdprobe_run taken with CDPROBE_OPT_LINK_COUNTERS on: one row per distinct
 * device of this process's ranks (ranks sharing a device share a row), with the payload the run's phase tables moved
 * between devices next to what NVML counted.  The samples bracket probe_ms: the first is taken before its clock
 * starts, the second after it stops (and after the event_timing round trip), so probe_ms, device_ms, kernel_ms and
 * event_ms mean what they mean without the option.  Nothing here judges the numbers: the verdict is unchanged.  A run
 * that fails before its rows are published takes no second sample and leaves the last report in place.  One-sided, not
 * collective.  Before any sampled run: run_seq 0 and every other field 0.  CDPROBE_ERR_ARG: null argument. */
CDPROBE_API int cdprobe_links(cdprobe_t* h, cdprobe_links_t* out);
CDPROBE_API void cdprobe_close(cdprobe_t* h);

/* Host-only helpers (no CUDA): schedule + slice arithmetic; the fd/blob rendezvous self-test. */
CDPROBE_API int cdprobe_plan(uint32_t n, uint64_t bytes, uint32_t mode, uint32_t flags, cdprobe_plan_t* out);
/* strict != 0: getCliqueIDStrict (feature gate CrashOnNVLinkFabricErrors, default on), else the legacy walk. */
CDPROBE_API int cdprobe_topology(uint32_t strict, cdprobe_topology_t* out);
CDPROBE_API int cdprobe_schedule(uint32_t n, uint32_t rank, uint64_t bytes, uint32_t mode, uint32_t ops, uint32_t flags,
                                 uint32_t ctas, uint32_t verify_ctas, cdprobe_schedule_t* out);
CDPROBE_API int cdprobe_rendezvous_selftest(const char* session, uint32_t rank, uint32_t world, uint32_t timeout_ms);
/* The GB/s gate cdprobe_run would apply to reads / writes for this configuration in an n-rank domain (0: bandwidth is
 * not judged — reach-only mode, n == 1).  Host-only arithmetic: lets a caller log or test the threshold without a GPU. */
CDPROBE_API int cdprobe_gate(const cdprobe_config_t* cfg, uint32_t n_total, float* gate_read_gbps, float* gate_write_gbps);

#ifdef __cplusplus
}
#endif
#endif /* CDPROBE_H_ */
