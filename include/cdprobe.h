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
  uint32_t path;                        /* the read data path used (CDPROBE_OPT_PATH) */
  uint64_t call_seq;                    /* 1-based count of cdprobe_allreduce calls on this handle, equal in every
                                           process (0 when the call was refused) */
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
 *   cdprobe_latency, cdprobe_pingpong, cdprobe_atomics, cdprobe_bwcurve, cdprobe_allreduce: diagnostics, benches,
 *   fault injection; the reference has no counterpart (it has no probe, SURVEY.md F1).
 *   cdprobe_diagnose, cdprobe_latency, cdprobe_pingpong, cdprobe_atomics, cdprobe_bwcurve and cdprobe_allreduce are
 *   optional for callers: a daemon binds them with dlsym and works without.
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
#define CDPROBE_OPT_ALLREDUCE_FAULT 19u   /* tests: value = ((rank + 1) << 32) | ((k + 1) << 24) | word arms an off-by-one
                                             in cdprobe_allreduce: in the process that hosts `rank`, timed rep 1 of
                                             size[k] adds 1 to output word `word` (< 2^24) before it is stored and
                                             folded, so exactly that row and size fail the checksum (and the word check
                                             when reps == 1); 0 disarms */
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
 * latency apart, so no time is domain-wide.  Every rep's (S, X) is checked against the pattern's sum, and after the
 * last rep of a size every output word is (bad_sizes, bad_words, CDPROBE_ERR_INTEGRITY).  If any cell of the domain
 * is down (cdprobe_unmap_peer, a failed mapping, MIG), nothing runs: every filled row has measured = 0 and the status
 * of the first such cell, and the call returns CDPROBE_OK.  A rank whose kernel passes timeout_ms is
 * CDPROBE_ERR_TIMEOUT and the handle stays usable.  Collective when world_size > 1: every process calls it with the
 * same reps and fills the rows of its own ranks (row_mask).  The output is bytes_per_pair per rank, so the scratch
 * buffer grows by that much until close (1 GiB at n == 1 with 1 GiB).  Touches no result, pattern, landing slot, Ctrl
 * word, pingpong or atomics line, run_seq, warm-up or bwcurve state.  *out carries abi, n and reps whatever the return
 * code.  CDPROBE_ERR_ARG: null argument, reps > 64, bytes_per_pair > 32 GiB, arguments that differ between processes,
 * or an armed CDPROBE_OPT_ALLREDUCE_FAULT whose rank is >= n, whose k is >= n_sizes or whose word is
 * >= size[k] / 8; CDPROBE_ERR_STATE: sticky handle. */
CDPROBE_API int cdprobe_allreduce(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out);
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
