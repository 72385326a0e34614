"""ctypes mirror of include/cdprobe.h (the structs a cgo shim would see as C.cdprobe_*_t)."""
from __future__ import annotations

import ctypes as C
import os

MAX_GPUS = 16
MAX_PHASES = 64
ABI_VERSION = 2

OK = 0
ERR_ABI, ERR_ARG, ERR_NO_DEVICE, ERR_CUDA, ERR_TIMEOUT = -1, -2, -3, -4, -5
ERR_RENDEZVOUS, ERR_NOMEM, ERR_UNSUPPORTED, ERR_STATE, ERR_INTEGRITY = -6, -7, -8, -9, -10

MODE_REACH_ONLY, MODE_SLICED, MODE_FULL = 0, 1, 2
OP_READ, OP_WRITE = 1, 2
FLAG_FABRIC_HANDLES = 0x01
FLAG_MIG_AWARE = 0x02
FLAG_LOCAL_DIAG = 0x04
FLAG_PATH_LDST = 0x08
FLAG_NO_COOPERATIVE = 0x10
FLAG_OVERLAP_VERIFY = 0x20
FLAG_ALLOW_SAME_DEVICE = 0x40
FLAG_UNIDIRECTIONAL = 0x80
FLAG_SERIAL_VERIFY = 0x100
FLAG_SIMULATE_MIG = 0x200
FLAG_ALL_RANK_BARRIERS = 0x400
FLAG_PAIR_BARRIERS = 0x800

OPT_EVENT_TIMING, OPT_CTAS, OPT_PATH, OPT_TIMEOUT_MS, OPT_OVERLAP_VERIFY, OPT_VERIFY_CTAS = 1, 2, 3, 4, 5, 6
OPT_UNIDIRECTIONAL = 7
OPT_WARMUP, OPT_WARMUP_BYTES, OPT_DEBUG_SKIP_RANK = 8, 9, 10
OPT_CTAS_RANK, OPT_MIN_FRACTION_PPM, OPT_LINK_PEAK_MBPS, OPT_SOLO_RANK, OPT_ALL_RANK_BARRIERS = 11, 12, 13, 14, 15
OPT_PAIR_BARRIERS = 16
OPT_PINGPONG_FAULT = 17
OPT_ATOMICS_FAULT = 18
OPT_ALLREDUCE_FAULT = 19

DIAG_SAMPLES = 16
DIAG_FLIP, DIAG_ZERO, DIAG_DISPLACED, DIAG_STALE, DIAG_FOREIGN = 0, 1, 2, 3, 4
DIAG_KIND_NAMES = ("flip", "zero", "displaced", "stale", "foreign")

LATENCY_DEFAULT_HOPS, LATENCY_DEFAULT_REPS = 1024, 8
LATENCY_MAX_HOPS, LATENCY_MAX_REPS = 1 << 20, 64

PINGPONG_DEFAULT_TRIPS, PINGPONG_DEFAULT_REPS = 256, 8
PINGPONG_MAX_TRIPS, PINGPONG_MAX_REPS = 1 << 16, 64

ATOMIC_FETCH_ADD, ATOMIC_CAS, ATOMIC_CONTENDED = 0, 1, 2
ATOMIC_KIND_NAMES = ("fetch_add", "cas", "contended")
ATOMICS_DEFAULT_OPS, ATOMICS_DEFAULT_REPS = 1024, 8
ATOMICS_MAX_OPS, ATOMICS_MAX_REPS = 1 << 16, 64

BWCURVE_MAX_SIZES = 24
BWCURVE_DEFAULT_REPS, BWCURVE_MAX_REPS = 8, 64
ALLREDUCE_DEFAULT_REPS, ALLREDUCE_MAX_REPS = 8, 64

_N2 = MAX_GPUS * MAX_GPUS


class ConfigT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("n_gpus", C.c_uint32),
        ("ordinals", C.c_int32 * MAX_GPUS),
        ("bytes", C.c_uint64),
        ("mode", C.c_uint32),
        ("ops", C.c_uint32),
        ("timeout_ms", C.c_uint32),
        ("flags", C.c_uint32),
        ("seed", C.c_uint64),
        ("min_fraction", C.c_float),
        ("link_peak_gbps", C.c_float),
        ("ctas", C.c_uint32),
        ("world_size", C.c_uint32),
        ("rank", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("session", C.c_char * 64),
    ]


class ResultT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("n", C.c_uint32),
        ("row_mask", C.c_uint32),
        ("verdict", C.c_uint32),
        ("reach_read", C.c_uint8 * _N2),
        ("reach_write", C.c_uint8 * _N2),
        ("gbps_read", C.c_float * _N2),
        ("gbps_write", C.c_float * _N2),
        ("status", C.c_int32 * _N2),
        ("sum_read", C.c_uint64 * _N2),
        ("xor_read", C.c_uint64 * _N2),
        ("sum_write", C.c_uint64 * _N2),
        ("xor_write", C.c_uint64 * _N2),
        ("bytes_per_pair", C.c_uint64),
        ("run_seq", C.c_uint64),
        ("rounds", C.c_uint32),
        ("phases", C.c_uint32),
        ("launches", C.c_uint32),
        ("aborted", C.c_uint32),
        ("warmed", C.c_uint32),
        ("reserved1", C.c_uint32),
        ("probe_ms", C.c_double),
        ("device_ms", C.c_double * MAX_GPUS),
        ("barrier_us", C.c_double * MAX_GPUS),
        ("event_ms", C.c_double * MAX_GPUS),
        ("min_gbps_read", C.c_float),
        ("min_gbps_write", C.c_float),
        ("gate_gbps_read", C.c_float),
        ("gate_gbps_write", C.c_float),
        ("kernel_ms", C.c_double * MAX_GPUS),
        ("unreachable_pairs", C.c_uint32),
        ("slow_pairs", C.c_uint32),
    ]


class InfoT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("n", C.c_uint32),
        ("n_local", C.c_uint32),
        ("first_local_rank", C.c_uint32),
        ("ordinal", C.c_int32 * MAX_GPUS),
        ("sm_count", C.c_uint32 * MAX_GPUS),
        ("ctas", C.c_uint32 * MAX_GPUS),
        ("mig", C.c_uint32 * MAX_GPUS),
        ("uuid", (C.c_char * 48) * MAX_GPUS),
        ("handle_type", C.c_uint32),
        ("path", C.c_uint32),
        ("bytes_per_pair", C.c_uint64),
        ("alloc_bytes", C.c_uint64),
        ("src_sum", (C.c_uint64 * MAX_GPUS) * MAX_GPUS),
        ("src_xor", (C.c_uint64 * MAX_GPUS) * MAX_GPUS),
        ("n_slices", C.c_uint32),
        ("smem_bytes", C.c_uint32),
        ("open_ms", C.c_double),
        ("fill_ms", C.c_double),
    ]


class PlanT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("n", C.c_uint32),
        ("rounds", C.c_uint32),
        ("n_slots", C.c_uint32),
        ("n_slices", C.c_uint32),
        ("reserved", C.c_uint32),
        ("bytes_per_pair", C.c_uint64),
        ("src_bytes", C.c_uint64),
        ("land_bytes", C.c_uint64),
        ("partner", (C.c_int8 * MAX_GPUS) * MAX_GPUS),
    ]


class TraceT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("n_phases", C.c_uint32),
        ("kind0", C.c_uint8 * MAX_PHASES),
        ("kind1", C.c_uint8 * MAX_PHASES),
        ("peer0", C.c_int8 * MAX_PHASES),
        ("peer1", C.c_int8 * MAX_PHASES),
        ("sync_all", C.c_uint8 * MAX_PHASES),
        ("sync_mask", C.c_uint16 * MAX_PHASES),
        ("post_mask", C.c_uint16 * MAX_PHASES),
        ("t_start", C.c_uint64 * MAX_PHASES),
        ("t_end0", C.c_uint64 * MAX_PHASES),
        ("t_end1", C.c_uint64 * MAX_PHASES),
        ("t_arrive", C.c_uint64 * MAX_PHASES),
    ]


class TopologyT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("n", C.c_uint32),
        ("uuid", (C.c_char * 96) * MAX_GPUS),
        ("pci_bus_id", (C.c_char * 32) * MAX_GPUS),
        ("mig", C.c_uint8 * MAX_GPUS),
        ("links_active", C.c_uint8 * MAX_GPUS),
        ("link_mask", C.c_uint32 * MAX_GPUS),
        ("fabric_state", C.c_uint8 * MAX_GPUS),
        ("clique_id", C.c_char * 96),
        ("clique_error", C.c_char * 160),
    ]


class ScheduleT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("n_phases", C.c_uint32),
        ("peer_mask", C.c_uint32),
        ("reserved", C.c_uint32),
        ("kind", (C.c_uint8 * MAX_PHASES) * 2),
        ("peer", (C.c_int8 * MAX_PHASES) * 2),
        ("slot", (C.c_uint8 * MAX_PHASES) * 2),
        ("writer", (C.c_uint8 * MAX_PHASES) * 2),
        ("cta0", (C.c_uint16 * MAX_PHASES) * 2),
        ("nctas", (C.c_uint16 * MAX_PHASES) * 2),
        ("sync_all", C.c_uint8 * MAX_PHASES),
        ("sync_mask", C.c_uint16 * MAX_PHASES),
        ("post_mask", C.c_uint16 * MAX_PHASES),
        ("wait_barrier", (C.c_uint8 * MAX_PHASES) * 2),
    ]


class DiagSampleT(C.Structure):
    _fields_ = [
        ("offset", C.c_uint64),
        ("expected", C.c_uint64),
        ("observed", C.c_uint64),
        ("word", C.c_uint64),
        ("run_seq", C.c_uint64),
        ("kind", C.c_uint32),
        ("rank", C.c_int32),
    ]


class DiagT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("op", C.c_uint32),
        ("issuer", C.c_uint32),
        ("target", C.c_uint32),
        ("reader", C.c_uint32),
        ("n_samples", C.c_uint32),
        ("run_seq", C.c_uint64),
        ("region_offset", C.c_uint64),
        ("bytes", C.c_uint64),
        ("bad_words", C.c_uint64),
        ("bad_granules", C.c_uint64),
        ("zero_words", C.c_uint64),
        ("first_bad", C.c_uint64),
        ("last_bad", C.c_uint64),
        ("kind_count", C.c_uint64 * 5),
        ("bit_flips", C.c_uint64 * 64),
        ("ms", C.c_double),
        ("sample", DiagSampleT * DIAG_SAMPLES),
    ]


class LatencyT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("n", C.c_uint32),
        ("row_mask", C.c_uint32),
        ("hops", C.c_uint32),
        ("reps", C.c_uint32),
        ("reserved", C.c_uint32),
        ("region_bytes", C.c_uint64),
        ("measured", C.c_uint8 * _N2),
        ("status", C.c_int32 * _N2),
        ("ns_min", C.c_float * _N2),
        ("ns_median", C.c_float * _N2),
        ("ns_max", C.c_float * _N2),
        ("digest", C.c_uint64 * _N2),
        ("ms", C.c_double),
    ]


class PingPongT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("n", C.c_uint32),
        ("row_mask", C.c_uint32),
        ("trips", C.c_uint32),
        ("reps", C.c_uint32),
        ("fenced", C.c_uint32),
        ("call_seq", C.c_uint64),
        ("measured", C.c_uint8 * _N2),
        ("status", C.c_int32 * _N2),
        ("ns_min", C.c_float * _N2),
        ("ns_median", C.c_float * _N2),
        ("ns_max", C.c_float * _N2),
        ("digest", C.c_uint64 * _N2),
        ("ms", C.c_double),
    ]


class AtomicsT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("n", C.c_uint32),
        ("row_mask", C.c_uint32),
        ("kind", C.c_uint32),
        ("ops", C.c_uint32),
        ("reps", C.c_uint32),
        ("lanes", C.c_uint32),
        ("reserved", C.c_uint32),
        ("call_seq", C.c_uint64),
        ("measured", C.c_uint8 * _N2),
        ("native", C.c_uint8 * _N2),
        ("status", C.c_int32 * _N2),
        ("ns_min", C.c_float * _N2),
        ("ns_median", C.c_float * _N2),
        ("ns_max", C.c_float * _N2),
        ("digest", C.c_uint64 * _N2),
        ("ms", C.c_double),
    ]


class BwCurveT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("n", C.c_uint32),
        ("row_mask", C.c_uint32),
        ("reps", C.c_uint32),
        ("n_sizes", C.c_uint32),
        ("path", C.c_uint32),
        ("call_seq", C.c_uint64),
        ("size", C.c_uint64 * BWCURVE_MAX_SIZES),
        ("measured", C.c_uint8 * _N2),
        ("status", C.c_int32 * _N2),
        ("bad_sizes", C.c_uint32 * _N2),
        ("t0_ns", C.c_float * _N2),
        ("peak_gbps", C.c_float * _N2),
        ("half_bytes", C.c_uint64 * _N2),
        ("ns_min", C.c_float * BWCURVE_MAX_SIZES * _N2),
        ("ns_median", C.c_float * BWCURVE_MAX_SIZES * _N2),
        ("ns_max", C.c_float * BWCURVE_MAX_SIZES * _N2),
        ("sum", C.c_uint64 * BWCURVE_MAX_SIZES * _N2),
        ("xr", C.c_uint64 * BWCURVE_MAX_SIZES * _N2),
        ("ms", C.c_double),
    ]


class AllReduceT(C.Structure):
    _fields_ = [
        ("abi", C.c_uint32),
        ("n", C.c_uint32),
        ("row_mask", C.c_uint32),
        ("reps", C.c_uint32),
        ("n_sizes", C.c_uint32),
        ("path", C.c_uint32),
        ("call_seq", C.c_uint64),
        ("size", C.c_uint64 * BWCURVE_MAX_SIZES),
        ("measured", C.c_uint8 * MAX_GPUS),
        ("status", C.c_int32 * MAX_GPUS),
        ("bad_sizes", C.c_uint32 * MAX_GPUS),
        ("t0_ns", C.c_float * MAX_GPUS),
        ("peak_gbps", C.c_float * MAX_GPUS),
        ("half_bytes", C.c_uint64 * MAX_GPUS),
        ("ns_min", C.c_float * BWCURVE_MAX_SIZES * MAX_GPUS),
        ("ns_median", C.c_float * BWCURVE_MAX_SIZES * MAX_GPUS),
        ("ns_max", C.c_float * BWCURVE_MAX_SIZES * MAX_GPUS),
        ("sum", C.c_uint64 * BWCURVE_MAX_SIZES * MAX_GPUS),
        ("xr", C.c_uint64 * BWCURVE_MAX_SIZES * MAX_GPUS),
        ("bad_words", C.c_uint64 * BWCURVE_MAX_SIZES * MAX_GPUS),
        ("first_bad", C.c_uint64 * BWCURVE_MAX_SIZES * MAX_GPUS),
        ("ms", C.c_double),
    ]


def allreduce_fault(rank: int, k: int, word: int) -> int:
    """The CDPROBE_OPT_ALLREDUCE_FAULT value that makes timed rep 1 of size[k] add 1 to output word `word` on `rank`."""
    return ((rank + 1) << 32) | ((k + 1) << 24) | word


def atomics_fault(issuer: int, target: int) -> int:
    """The CDPROBE_OPT_ATOMICS_FAULT value that makes the first op of timed rep 1 of cell (issuer, target) step by 2."""
    return ((issuer + 1) << 16) | (target + 1)


def pingpong_fault(initiator: int, target: int, trip: int) -> int:
    """The CDPROBE_OPT_PINGPONG_FAULT value that arms a skip-ahead echo at `trip` of timed rep 1 of cell
    (initiator, target)."""
    return ((initiator + 1) << 32) | ((target + 1) << 16) | trip


# Every symbol include/cdprobe.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "cdprobe_abi_version": (C.c_uint32, []),
    "cdprobe_strerror": (C.c_char_p, [C.c_int]),
    "cdprobe_last_error": (C.c_char_p, []),
    "cdprobe_open": (C.c_int, [C.POINTER(ConfigT), C.POINTER(C.c_void_p)]),
    "cdprobe_run": (C.c_int, [C.c_void_p, C.POINTER(ResultT)]),
    "cdprobe_gather": (C.c_int, [C.c_void_p, C.POINTER(ResultT)]),
    "cdprobe_info": (C.c_int, [C.c_void_p, C.POINTER(InfoT)]),
    "cdprobe_trace": (C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(TraceT)]),
    "cdprobe_set_option": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint64]),
    "cdprobe_remap_peer": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32]),
    "cdprobe_unmap_peer": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32]),
    "cdprobe_corrupt": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64]),
    "cdprobe_corrupt_landing": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64),
                                          C.POINTER(C.c_uint64)]),
    "cdprobe_ce_copy": (C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_uint32,
                                  C.c_uint64, C.c_uint32, C.POINTER(C.c_double)]),
    "cdprobe_diagnose": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(DiagT)]),
    "cdprobe_latency": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(LatencyT)]),
    "cdprobe_pingpong": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(PingPongT)]),
    "cdprobe_atomics": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(AtomicsT)]),
    "cdprobe_bwcurve": (C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(BwCurveT)]),
    "cdprobe_allreduce": (C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(AllReduceT)]),
    "cdprobe_close": (None, [C.c_void_p]),
    "cdprobe_plan": (C.c_int, [C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(PlanT)]),
    "cdprobe_topology": (C.c_int, [C.c_uint32, C.POINTER(TopologyT)]),
    "cdprobe_schedule": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                   C.c_uint32, C.POINTER(ScheduleT)]),
    "cdprobe_rendezvous_selftest": (C.c_int, [C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32]),
    "cdprobe_gate": (C.c_int, [C.POINTER(ConfigT), C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
}

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libcdprobe.so")
_lib = None


def load_library(path: str | None = None) -> C.CDLL:
    """dlopen libcdprobe.so (lazily, like go-nvml does for NVML) and type every entry point.

    There is no fallback: a missing library is an error, never a silent CPU path.
    """
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise OSError(f"{p} not found: build it with `python k8s-dra-driver-gpu_b200/build.py` (needs nvcc)")
    lib = C.CDLL(p)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export it
        fn.restype = res
        fn.argtypes = args
    if path is None:
        _lib = lib
    return lib
