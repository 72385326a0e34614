"""Host-side mirror of the Go shim ``pkg/fabricprobe`` (SURVEY.md §8b).

Go signature being mirrored (see INTEGRATION.md for the cgo file)::

    type Config struct{ Ordinals []int; Bytes uint64; Mode, Ops, TimeoutMs, Flags uint32; ... }
    type Result struct{ N int; ReachRead, ReachWrite []bool /* N x N row-major */
                        GBpsRead, GBpsWrite []float32; ProbeMs float64; ... }
    func Open(Config) (*Probe, error)
    func (*Probe) Run(ctx) (Result, error)
    func (*Probe) Close()

Caller in the reference tree: ``run()`` in cmd/compute-domain-daemon/main.go:212-347
owns the probe; ``check()`` (main.go:435-459) reads its cached verdict.  Errors
follow the daemon's convention: a Python exception here is a Go ``error`` there;
``ErrUnsupported`` is what the ``!cgo`` stub returns.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
from typing import List, Optional, Sequence

from . import abi


class ProbeError(RuntimeError):
    def __init__(self, code: int, what: str, detail: str = ""):
        self.code = code
        self.detail = detail
        super().__init__(f"{what}: {detail}" if detail else what)


class ErrUnsupported(ProbeError):
    """No CUDA driver / no sm_90 GPU: the probe cannot run and nothing stands in for it."""


@dataclasses.dataclass
class Config:
    ordinals: Optional[Sequence[int]] = None  # None = all visible GPUs
    bytes: int = 1 << 30
    mode: int = abi.MODE_SLICED
    ops: int = abi.OP_READ | abi.OP_WRITE
    timeout_ms: int = 5000
    flags: int = 0
    seed: int = 0
    min_fraction: float = 0.0  # 0 = library default (0.65 of the reference)
    link_peak_gbps: float = 0.0  # 0 = nominal NVLink 4 reference (include/cdprobe.h); > 0 = absolute GB/s
    ctas: int = 0
    world_size: int = 1
    rank: int = 0
    session: str = ""

    def to_c(self) -> abi.ConfigT:
        c = abi.ConfigT()
        c.abi = abi.ABI_VERSION
        if self.ordinals is None:
            c.n_gpus = 0
        else:
            c.n_gpus = len(self.ordinals)
            for i, o in enumerate(self.ordinals):
                c.ordinals[i] = int(o)
        c.bytes = int(self.bytes)
        c.mode = self.mode
        c.ops = self.ops
        c.timeout_ms = self.timeout_ms
        c.flags = self.flags
        c.seed = self.seed
        c.min_fraction = self.min_fraction
        c.link_peak_gbps = self.link_peak_gbps
        c.ctas = self.ctas
        c.world_size = self.world_size
        c.rank = self.rank
        c.session = self.session.encode()[:63]
        return c


def _mat(t, a, keep=None):
    """The n x n matrix [i][j] of a CDPROBE_MAX_GPUS-strided array of result `t`; None where keep(k) is false."""
    return [[a[k] if keep is None or keep(k) else None for k in range(i * abi.MAX_GPUS, i * abi.MAX_GPUS + t.n)]
            for i in range(t.n)]


def _row(t, a, keep=None):
    """The n entries [r] of a CDPROBE_MAX_GPUS-long array of result `t`; None where keep(r) is false."""
    return [a[r] if keep is None or keep(r) else None for r in range(t.n)]


def _sized(t, a):
    """Each entry of the per-size array `a` of result `t`, as a list cut to the ladder's n_sizes."""
    return [list(x)[:t.n_sizes] for x in a]


def _measured(t):
    """keep: entry k of `t` (a cell or a rank) was measured."""
    return lambda k: t.measured[k]


def _timed(t):
    """keep: entry k of `t` (a cell or a rank) was measured and did not pass timeout_ms."""
    return lambda k: t.measured[k] and t.status[k] != abi.ERR_TIMEOUT


def _timed_cells(t) -> dict:
    """The per-cell fields of a Latency, a PingPong or an Atomics.  A cell that was not measured is None in every
    matrix but `status`; a cell that timed out keeps its digest but has no times."""
    timed = _timed(t)
    return dict(measured=_mat(t, [bool(m) for m in t.measured]), status=_mat(t, t.status),
                ns_min=_mat(t, t.ns_min, timed), ns_median=_mat(t, t.ns_median, timed), ns_max=_mat(t, t.ns_max, timed),
                digest=_mat(t, t.digest, _measured(t)), ms=t.ms, raw=t)


def _ladder(t, shape, keep) -> dict:
    """The fields every ladder measurement has, per cell (shape _mat) or per rank (shape _row): `sizes`, `measured`,
    `status`, and where keep, the summary of the medians and the times per size."""
    return dict(sizes=list(t.size)[:t.n_sizes], measured=shape(t, [bool(m) for m in t.measured]),
                status=shape(t, t.status), t0_ns=shape(t, t.t0_ns, keep), peak_gbps=shape(t, t.peak_gbps, keep),
                half_bytes=shape(t, t.half_bytes, keep), ns_min=shape(t, _sized(t, t.ns_min), keep),
                ns_median=shape(t, _sized(t, t.ns_median), keep), ns_max=shape(t, _sized(t, t.ns_max), keep),
                ms=t.ms, raw=t)


def _curve(t, shape) -> dict:
    """The fields a BwCurve, a Memcpy and an AllReduce share: the ladder's and the (S, X) check's, each None but
    `measured` and `status` where the entry was not measured or timed out."""
    timed = _timed(t)
    return dict(_ladder(t, shape, timed), bad_sizes=shape(t, t.bad_sizes, timed),
                sum=shape(t, _sized(t, t.sum), timed), xr=shape(t, _sized(t, t.xr), timed))


def _cell_checks(t) -> dict:
    """The per-cell check fields of an AllToAll and a CeAllToAll, each None but `cell_measured` and `cell_status`
    where the block was not checked or its check timed out."""
    def checked(c):
        return t.cell_measured[c] and t.cell_status[c] != abi.ERR_TIMEOUT

    return dict(cell_measured=_mat(t, [bool(m) for m in t.cell_measured]), cell_status=_mat(t, t.cell_status),
                bad_sizes=_mat(t, t.bad_sizes, checked), bad_words=_mat(t, _sized(t, t.bad_words), checked),
                first_bad=_mat(t, _sized(t, t.first_bad), checked), sum=_mat(t, _sized(t, t.sum), checked),
                xr=_mat(t, _sized(t, t.xr), checked))


@dataclasses.dataclass
class Result:
    n: int
    row_mask: int
    verdict: bool
    reach_read: List[List[int]]
    reach_write: List[List[int]]
    gbps_read: List[List[float]]
    gbps_write: List[List[float]]
    status: List[List[int]]
    sum_read: List[List[int]]
    xor_read: List[List[int]]
    sum_write: List[List[int]]
    xor_write: List[List[int]]
    bytes_per_pair: int
    run_seq: int
    rounds: int
    phases: int
    launches: int
    aborted: bool
    warmed: bool
    probe_ms: float
    device_ms: List[float]
    barrier_us: List[float]
    event_ms: List[float]
    min_gbps_read: float
    min_gbps_write: float
    gate_gbps_read: float = 0.0
    gate_gbps_write: float = 0.0
    unreachable_pairs: int = 0
    slow_pairs: int = 0
    kernel_ms: List[float] = dataclasses.field(default_factory=list)
    raw: abi.ResultT = dataclasses.field(repr=False, default=None)

    @property
    def reach(self) -> List[List[int]]:
        """reach_read AND reach_write — what is compared with the NVML oracle (SURVEY §8c)."""
        return [[a & b for a, b in zip(ra, rb)] for ra, rb in zip(self.reach_read, self.reach_write)]

    @staticmethod
    def from_c(r: abi.ResultT) -> "Result":
        n = r.n
        return Result(
            n=n,
            row_mask=r.row_mask,
            verdict=bool(r.verdict),
            reach_read=_mat(r, r.reach_read),
            reach_write=_mat(r, r.reach_write),
            gbps_read=_mat(r, r.gbps_read),
            gbps_write=_mat(r, r.gbps_write),
            status=_mat(r, r.status),
            sum_read=_mat(r, r.sum_read),
            xor_read=_mat(r, r.xor_read),
            sum_write=_mat(r, r.sum_write),
            xor_write=_mat(r, r.xor_write),
            bytes_per_pair=r.bytes_per_pair,
            run_seq=r.run_seq,
            rounds=r.rounds,
            phases=r.phases,
            launches=r.launches,
            aborted=bool(r.aborted),
            warmed=bool(r.warmed),
            probe_ms=r.probe_ms,
            device_ms=list(r.device_ms)[:n],
            barrier_us=list(r.barrier_us)[:n],
            event_ms=list(r.event_ms)[:n],
            min_gbps_read=r.min_gbps_read,
            min_gbps_write=r.min_gbps_write,
            gate_gbps_read=r.gate_gbps_read,
            gate_gbps_write=r.gate_gbps_write,
            unreachable_pairs=r.unreachable_pairs,
            slow_pairs=r.slow_pairs,
            kernel_ms=list(r.kernel_ms)[:n],
            raw=r,
        )


@dataclasses.dataclass
class Diagnosis:
    """What cdprobe_diagnose found in one cell's region: exact counts, the classes of the bad words, the bit-flip
    histogram of FLIP words and the lowest-offset bad words (dicts with kind names)."""
    op: str                   # "read" or "write"
    issuer: int
    target: int
    reader: int
    run_seq: int
    region_offset: int
    bytes: int
    bad_words: int
    bad_granules: int
    zero_words: int
    first_bad: Optional[int]  # byte offset; None when the region is clean
    last_bad: Optional[int]
    kinds: dict               # {"flip": n, "zero": n, "displaced": n, "stale": n, "foreign": n}
    bit_flips: List[int]      # [64]
    ms: float
    samples: List[dict]
    raw: abi.DiagT = dataclasses.field(repr=False, default=None)

    @property
    def words(self) -> int:
        return self.bytes // 8

    @staticmethod
    def from_c(d: abi.DiagT) -> "Diagnosis":
        clean = d.bad_words == 0
        return Diagnosis(
            op={abi.OP_READ: "read", abi.OP_WRITE: "write"}.get(d.op, str(d.op)),
            issuer=d.issuer, target=d.target, reader=d.reader, run_seq=d.run_seq,
            region_offset=d.region_offset, bytes=d.bytes, bad_words=d.bad_words, bad_granules=d.bad_granules,
            zero_words=d.zero_words, first_bad=None if clean else d.first_bad, last_bad=None if clean else d.last_bad,
            kinds={name: d.kind_count[k] for k, name in enumerate(abi.DIAG_KIND_NAMES)},
            bit_flips=list(d.bit_flips), ms=d.ms,
            samples=[{"offset": s.offset, "expected": s.expected, "observed": s.observed, "word": s.word,
                      "run_seq": s.run_seq, "kind": abi.DIAG_KIND_NAMES[s.kind], "rank": s.rank}
                     for s in d.sample[:d.n_samples]],
            raw=d,
        )


@dataclasses.dataclass
class Latency:
    """What cdprobe_latency measured: n x n matrices [issuer][target] of ns per dependent 8-byte load (min, median and
    max over the timed reps) and the digest of the loaded words.  A cell that was not chased (a row of another
    process, a mapping that is down, the diagonal without a loop-back slice) is None in every matrix but `status`;
    a chase that passed timeout_ms has a digest but no times."""
    n: int
    row_mask: int
    hops: int
    reps: int
    region_bytes: int
    measured: List[List[bool]]
    status: List[List[int]]     # 0 ok; ERR_INTEGRITY; ERR_TIMEOUT; else the mapping's status
    ns_min: List[List[Optional[float]]]
    ns_median: List[List[Optional[float]]]
    ns_max: List[List[Optional[float]]]
    digest: List[List[Optional[int]]]
    ms: float
    raw: abi.LatencyT = dataclasses.field(repr=False, default=None)

    @staticmethod
    def from_c(t: abi.LatencyT) -> "Latency":
        return Latency(n=t.n, row_mask=t.row_mask, hops=t.hops, reps=t.reps, region_bytes=t.region_bytes,
                       **_timed_cells(t))


@dataclasses.dataclass
class PingPong:
    """What cdprobe_pingpong measured: n x n matrices [initiator][target] of ns per signal round trip (min, median and
    max over the timed reps) and the digest of the echo words the initiator received.  A cell that did not run (a row
    of another process, the diagonal, a pair whose mapping is down) is None in every matrix but `status`; a cell that
    passed timeout_ms has a digest but no times."""
    n: int
    row_mask: int
    trips: int
    reps: int
    fenced: bool
    call_seq: int
    measured: List[List[bool]]
    status: List[List[int]]     # 0 ok; ERR_INTEGRITY; ERR_TIMEOUT; else the pair's mapping status
    ns_min: List[List[Optional[float]]]
    ns_median: List[List[Optional[float]]]
    ns_max: List[List[Optional[float]]]
    digest: List[List[Optional[int]]]
    ms: float
    raw: abi.PingPongT = dataclasses.field(repr=False, default=None)

    @staticmethod
    def from_c(t: abi.PingPongT) -> "PingPong":
        return PingPong(n=t.n, row_mask=t.row_mask, trips=t.trips, reps=t.reps, fenced=bool(t.fenced),
                        call_seq=t.call_seq, **_timed_cells(t))


@dataclasses.dataclass
class Atomics:
    """What cdprobe_atomics measured: n x n matrices [issuer][target] of ns per system-scope atomic on the cell's own
    word in the target's memory (min, median and max over the timed reps) and the digest of the values the atomics
    returned.  `native` is 1 (same device, or CUDA reports native atomics), 0 (CUDA reports none: not run) or 2 (the
    target's device is not visible in this process) for the local rows, None elsewhere.  A cell that did not run is
    None in every matrix but `status` and `native`; a cell that passed timeout_ms has a digest but no times."""
    n: int
    row_mask: int
    kind: int
    ops: int
    reps: int
    lanes: int
    call_seq: int
    native: List[List[Optional[int]]]
    measured: List[List[bool]]
    status: List[List[int]]     # 0 ok; ERR_INTEGRITY; ERR_TIMEOUT; ERR_UNSUPPORTED; else the mapping's status
    ns_min: List[List[Optional[float]]]
    ns_median: List[List[Optional[float]]]
    ns_max: List[List[Optional[float]]]
    digest: List[List[Optional[int]]]
    ms: float
    raw: abi.AtomicsT = dataclasses.field(repr=False, default=None)

    @staticmethod
    def from_c(t: abi.AtomicsT) -> "Atomics":
        return Atomics(n=t.n, row_mask=t.row_mask, kind=t.kind, ops=t.ops, reps=t.reps, lanes=t.lanes,
                       call_seq=t.call_seq,
                       native=_mat(t, t.native, lambda k: t.row_mask >> (k // abi.MAX_GPUS) & 1),
                       **_timed_cells(t))


@dataclasses.dataclass
class BwCurve:
    """What cdprobe_bwcurve measured: per cell [issuer][target], ns per rep (min, median and max over the timed reps)
    of reading each size of the ladder `sizes` from the source slice the issuer reads, the (S, X) of the last timed
    rep, the sizes whose reads did not match the pattern (`bad_sizes`, bit k for sizes[k]) and the summary of the
    medians: t0_ns (the smallest size), peak_gbps and half_bytes.  Per-size values are lists over `sizes`.  A cell
    that did not run is None everywhere but `status`; a cell that passed timeout_ms has no times."""
    n: int
    row_mask: int
    reps: int
    path: int
    call_seq: int
    sizes: List[int]
    measured: List[List[bool]]
    status: List[List[int]]     # 0 ok; ERR_INTEGRITY; ERR_TIMEOUT; else the mapping's status
    bad_sizes: List[List[Optional[int]]]
    t0_ns: List[List[Optional[float]]]
    peak_gbps: List[List[Optional[float]]]
    half_bytes: List[List[Optional[int]]]
    ns_min: List[List[Optional[List[float]]]]
    ns_median: List[List[Optional[List[float]]]]
    ns_max: List[List[Optional[List[float]]]]
    sum: List[List[Optional[List[int]]]]
    xr: List[List[Optional[List[int]]]]
    ms: float
    raw: abi.BwCurveT = dataclasses.field(repr=False, default=None)

    @staticmethod
    def from_c(t: abi.BwCurveT) -> "BwCurve":
        return BwCurve(n=t.n, row_mask=t.row_mask, reps=t.reps, path=t.path, call_seq=t.call_seq, **_curve(t, _mat))


@dataclasses.dataclass
class AllReduce:
    """What cdprobe_allreduce measured: per rank r, ns per rep (min, median and max over the timed reps) of the one-shot
    all-reduce of each size of the ladder `sizes`, the (S, X) of the output the last timed rep stored, the word check
    of that output (`bad_words`, and `first_bad`, the byte offset of the first bad word or U64_MAX), the sizes that
    failed either check (`bad_sizes`, bit k for sizes[k]) and the summary of the medians: t0_ns (the smallest size),
    peak_gbps (algorithm bandwidth: size / ns; each rank's ingress is (n - 1) x that) and half_bytes.  Per-size values
    are lists over `sizes`, and every list is indexed by rank.  A rank that did not run is None everywhere but
    `status`; a rank that passed timeout_ms has no times."""
    n: int
    row_mask: int
    reps: int
    path: int
    call_seq: int
    sizes: List[int]
    measured: List[bool]
    status: List[int]     # 0 ok; ERR_INTEGRITY; ERR_TIMEOUT; else the mapping status of the domain's first cell down
    bad_sizes: List[Optional[int]]
    t0_ns: List[Optional[float]]
    peak_gbps: List[Optional[float]]
    half_bytes: List[Optional[int]]
    ns_min: List[Optional[List[float]]]
    ns_median: List[Optional[List[float]]]
    ns_max: List[Optional[List[float]]]
    sum: List[Optional[List[int]]]
    xr: List[Optional[List[int]]]
    bad_words: List[Optional[List[int]]]
    first_bad: List[Optional[List[int]]]
    ms: float
    raw: abi.AllReduceT = dataclasses.field(repr=False, default=None)

    @staticmethod
    def from_c(t: abi.AllReduceT) -> "AllReduce":
        timed = _timed(t)
        return AllReduce(n=t.n, row_mask=t.row_mask, reps=t.reps, path=t.path, call_seq=t.call_seq,
                         bad_words=_row(t, _sized(t, t.bad_words), timed),
                         first_bad=_row(t, _sized(t, t.first_bad), timed), **_curve(t, _row))


@dataclasses.dataclass
class AllToAll:
    """What cdprobe_alltoall measured.  Per rank r, as the sender: `blocks` pushed per rep, ns per rep (min, median and
    max over the timed reps) of each size of the ladder `sizes`, and the summary of the medians: t0_ns (the smallest
    size), peak_gbps (egress: blocks x size / ns) and half_bytes.  Per cell [s][d] (sender, receiver), as the receiver
    checked it: `cell_status`, the sizes that delivered a bad word (`bad_sizes`, bit k for sizes[k]), `bad_words` and
    `first_bad` (the byte offset of the lowest bad word, or U64_MAX) per size, and the (S, X) of the block in the last
    timed rep.  Per-size values are lists over `sizes`.  A rank that did not run, or timed out, is None everywhere but
    `measured` and `status`; a cell its receiver did not check is None everywhere but `cell_measured` and
    `cell_status`."""
    n: int
    row_mask: int
    reps: int
    path: int
    call_seq: int
    area_bytes: int
    sizes: List[int]
    measured: List[bool]
    status: List[int]     # 0 ok; ERR_TIMEOUT
    blocks: List[Optional[int]]
    t0_ns: List[Optional[float]]
    peak_gbps: List[Optional[float]]
    half_bytes: List[Optional[int]]
    ns_min: List[Optional[List[float]]]
    ns_median: List[Optional[List[float]]]
    ns_max: List[Optional[List[float]]]
    cell_measured: List[List[bool]]
    cell_status: List[List[int]]  # 0 ok; ERR_INTEGRITY; ERR_TIMEOUT; else the sender's mapping status of the receiver
    bad_sizes: List[List[Optional[int]]]
    bad_words: List[List[Optional[List[int]]]]
    first_bad: List[List[Optional[List[int]]]]
    sum: List[List[Optional[List[int]]]]
    xr: List[List[Optional[List[int]]]]
    ms: float
    raw: abi.AllToAllT = dataclasses.field(repr=False, default=None)

    @staticmethod
    def from_c(t: abi.AllToAllT) -> "AllToAll":
        return AllToAll(n=t.n, row_mask=t.row_mask, reps=t.reps, path=t.path, call_seq=t.call_seq,
                        area_bytes=t.area_bytes, blocks=_row(t, t.blocks, _measured(t)), **_ladder(t, _row, _timed(t)),
                        **_cell_checks(t))


@dataclasses.dataclass
class Memcpy:
    """What cdprobe_memcpy measured: per cell [issuer][target], ns per copy-engine copy (min, median and max over the
    timed reps, by CUDA events) of each size of the ladder `sizes`, pulled from the target (op OP_READ) or pushed to it
    (OP_WRITE), the word check of what landed (`bad_words` over every rep, and `first_bad`, the byte offset of the
    lowest bad word or U64_MAX), the (S, X) of the last timed rep's destination, the sizes that failed either check
    (`bad_sizes`, bit k for sizes[k]) and the summary of the medians: t0_ns (the smallest size; events resolve about
    0.5 us), peak_gbps and half_bytes.  Per-size values are lists over `sizes`.  A cell that did not run is None
    everywhere but `status`; a cell whose (S, X) read passed timeout_ms has no times."""
    n: int
    row_mask: int
    reps: int
    op: int
    call_seq: int
    area_bytes: int
    sizes: List[int]
    measured: List[List[bool]]
    status: List[List[int]]     # 0 ok; ERR_INTEGRITY; ERR_TIMEOUT; else the issuer's mapping status
    bad_sizes: List[List[Optional[int]]]
    t0_ns: List[List[Optional[float]]]
    peak_gbps: List[List[Optional[float]]]
    half_bytes: List[List[Optional[int]]]
    ns_min: List[List[Optional[List[float]]]]
    ns_median: List[List[Optional[List[float]]]]
    ns_max: List[List[Optional[List[float]]]]
    sum: List[List[Optional[List[int]]]]
    xr: List[List[Optional[List[int]]]]
    bad_words: List[List[Optional[List[int]]]]
    first_bad: List[List[Optional[List[int]]]]
    ms: float
    raw: abi.MemcpyT = dataclasses.field(repr=False, default=None)

    @staticmethod
    def from_c(t: abi.MemcpyT) -> "Memcpy":
        timed = _timed(t)
        return Memcpy(n=t.n, row_mask=t.row_mask, reps=t.reps, op=t.op, call_seq=t.call_seq, area_bytes=t.area_bytes,
                      bad_words=_mat(t, _sized(t, t.bad_words), timed),
                      first_bad=_mat(t, _sized(t, t.first_bad), timed), **_curve(t, _mat))


@dataclasses.dataclass
class CeAllToAll:
    """What cdprobe_ce_alltoall measured.  Per rank r: `blocks` it copies per rep (the cells it issues), ns per rep
    (min, median and max over the timed reps, from its release until its own copies are complete and every block
    addressed to it has landed) of each size of the ladder `sizes`, and the summary of the medians: t0_ns (the smallest
    size), peak_gbps (blocks x size / ns) and half_bytes.  Per cell [issuer][target]: `copy_ns_median`, the median of
    its copy stream's own timing per size, filled by the issuer's process; and, as the block's owner checked it (the
    issuer on a pull, the target on a push), `cell_status`, the sizes that failed a check (`bad_sizes`, bit k for
    sizes[k]), `bad_words` and `first_bad` (the byte offset of the lowest bad word, or U64_MAX) per size, and the (S, X)
    of the block in the last timed rep.  Per-size values are lists over `sizes`.  A rank that did not run is None
    everywhere but `measured` and `status`; a cell whose owner did not check it is None in the check fields, and one
    whose issuer is not local has no `copy_ns_median`."""
    n: int
    row_mask: int
    reps: int
    op: int
    call_seq: int
    area_bytes: int
    sizes: List[int]
    measured: List[bool]
    status: List[int]     # 0 ok; else the status of the domain's first down mapping
    blocks: List[Optional[int]]
    t0_ns: List[Optional[float]]
    peak_gbps: List[Optional[float]]
    half_bytes: List[Optional[int]]
    ns_min: List[Optional[List[float]]]
    ns_median: List[Optional[List[float]]]
    ns_max: List[Optional[List[float]]]
    cell_measured: List[List[bool]]
    cell_status: List[List[int]]  # 0 ok; ERR_INTEGRITY; ERR_TIMEOUT; else the status of the first down mapping
    bad_sizes: List[List[Optional[int]]]
    copy_ns_median: List[List[Optional[List[float]]]]
    bad_words: List[List[Optional[List[int]]]]
    first_bad: List[List[Optional[List[int]]]]
    sum: List[List[Optional[List[int]]]]
    xr: List[List[Optional[List[int]]]]
    ms: float
    raw: abi.CeAllToAllT = dataclasses.field(repr=False, default=None)

    @staticmethod
    def from_c(t: abi.CeAllToAllT) -> "CeAllToAll":
        measured = _measured(t)

        def issued(c):
            # rank s issues a cell to every peer, and to itself only with a loop-back slice (then it copies n blocks)
            s, d = divmod(c, abi.MAX_GPUS)
            return t.measured[s] and (s != d or t.blocks[s] == t.n)

        return CeAllToAll(n=t.n, row_mask=t.row_mask, reps=t.reps, op=t.op, call_seq=t.call_seq,
                          area_bytes=t.area_bytes, blocks=_row(t, t.blocks, measured), **_ladder(t, _row, measured),
                          copy_ns_median=_mat(t, _sized(t, t.copy_ns_median), issued), **_cell_checks(t))


@dataclasses.dataclass
class Links:
    """What cdprobe_links reported: per distinct local device, the per-link NVLink counter deltas NVML gave over the
    last run taken with abi.OPT_LINK_COUNTERS on, next to the payload that run's plan moved between devices.  Each
    device is a dict: status (0, abi.ERR_UNSUPPORTED or an nvmlReturn_t), rank_mask, uuid, link_mask, lost_mask,
    error_mask, expected_tx_kib, expected_rx_kib, and per link (lists of 18) tx_kib, rx_kib, errors ({"replay",
    "recovery", "crc"}), failed_fields (abi.LINK_FIELD_* bits) and remote_bus_id.  run_seq 0: no sampled run yet."""
    n_devices: int
    run_seq: int
    sample_ms: float
    devices: List[dict]
    raw: abi.LinksT = dataclasses.field(repr=False, default=None)

    @staticmethod
    def from_c(t: abi.LinksT) -> "Links":
        L = abi.NVLINK_MAX_LINKS
        return Links(n_devices=t.n_devices, run_seq=t.run_seq, sample_ms=t.sample_ms, raw=t, devices=[
            {"status": d.status, "rank_mask": d.rank_mask, "uuid": d.uuid.decode(), "link_mask": d.link_mask,
             "lost_mask": d.lost_mask, "error_mask": d.error_mask, "expected_tx_kib": d.expected_tx_kib,
             "expected_rx_kib": d.expected_rx_kib, "tx_kib": list(d.tx_kib), "rx_kib": list(d.rx_kib),
             "errors": [dict(zip(abi.LINK_ERROR_NAMES, d.errors[l])) for l in range(L)],
             "failed_fields": list(d.failed_fields),
             "remote_bus_id": [d.remote_bus_id[l].value.decode() for l in range(L)]}
            for d in t.dev[:t.n_devices]])


def _raise(lib, rc: int, what: str):
    msg = lib.cdprobe_strerror(rc).decode()
    detail = lib.cdprobe_last_error().decode()
    cls = ErrUnsupported if rc in (abi.ERR_NO_DEVICE, abi.ERR_UNSUPPORTED) else ProbeError
    raise cls(rc, f"{what}: {msg}", detail)


def _check(lib, rc: int, what: str):
    if rc != abi.OK:
        _raise(lib, rc, what)


class Probe:
    """One probe domain handle (not thread-safe, like the C handle)."""

    def __init__(self, cfg: Config):
        self._lib = abi.load_library()
        self._h = C.c_void_p()
        self.cfg = cfg
        c = cfg.to_c()
        rc = self._lib.cdprobe_open(C.byref(c), C.byref(self._h))
        if rc != abi.OK:
            self._h = C.c_void_p()
            _raise(self._lib, rc, "cdprobe_open")

    def _call(self, fn: str, out_type, *args):
        """Entry point `fn` called with the handle, `args` and a new `out_type` to fill: (return code, the out struct
        as the library left it)."""
        out = out_type()
        return getattr(self._lib, fn)(self._h, *args, C.byref(out)), out

    def _decode(self, fn: str, result_type, call):
        """The (return code, out struct) `call` of entry point `fn` decoded as a `result_type`; a ProbeError named
        after `fn` when the code is not OK."""
        rc, out = call
        _check(self._lib, rc, fn)
        return result_type.from_c(out)

    # -- Go: (*Probe).Run -------------------------------------------------------------
    def Run(self, gather: bool = False, allow_timeout: bool = False) -> Result:
        r = abi.ResultT()
        rc = self._lib.cdprobe_run(self._h, C.byref(r))
        if rc != abi.OK and not (allow_timeout and rc == abi.ERR_TIMEOUT):
            _raise(self._lib, rc, "cdprobe_run")
        if gather:
            _check(self._lib, self._lib.cdprobe_gather(self._h, C.byref(r)), "cdprobe_gather")
        return Result.from_c(r)

    def run_raw(self, out: abi.ResultT) -> int:
        """The bare ABI call (bench.py times this)."""
        return self._lib.cdprobe_run(self._h, C.byref(out))

    def Info(self) -> abi.InfoT:
        i = abi.InfoT()
        _check(self._lib, self._lib.cdprobe_info(self._h, C.byref(i)), "cdprobe_info")
        return i

    def Trace(self, local: int = 0):
        """Per-phase timeline of the last run: list of dicts (ns relative to the first barrier release)."""
        t = abi.TraceT()
        _check(self._lib, self._lib.cdprobe_trace(self._h, local, C.byref(t)), "cdprobe_trace")
        names = {0: "-", 1: "read", 2: "write", 3: "verify", 4: "warm"}
        return [{"job0": names[t.kind0[p]], "peer0": t.peer0[p], "job1": names[t.kind1[p]], "peer1": t.peer1[p],
                 "sync_all": int(t.sync_all[p]), "sync_mask": int(t.sync_mask[p]), "post_mask": int(t.post_mask[p]), "t_start": t.t_start[p], "t_end0": t.t_end0[p], "t_end1": t.t_end1[p],
                 "t_arrive": t.t_arrive[p]} for p in range(t.n_phases)]

    def SetOption(self, option: int, value: int) -> None:
        _check(self._lib, self._lib.cdprobe_set_option(self._h, option, value), "cdprobe_set_option")

    def UnmapPeer(self, local: int, peer: int) -> None:
        _check(self._lib, self._lib.cdprobe_unmap_peer(self._h, local, peer), "cdprobe_unmap_peer")

    def RemapPeer(self, local: int, peer: int) -> None:
        _check(self._lib, self._lib.cdprobe_remap_peer(self._h, local, peer), "cdprobe_remap_peer")

    def CeCopy(self, copies, push: bool = True, nbytes: int = 0, reps: int = 4):
        """Copy-engine reference on the probe's buffers: `copies` = [(local rank, peer rank), ...] run concurrently;
        returns [(ms for `reps` copies, GB/s), ...].  Not part of a probe: the same-box ceiling quoted beside it."""
        k = len(copies)
        loc = (C.c_uint32 * k)(*[c[0] for c in copies])
        peer = (C.c_uint32 * k)(*[c[1] for c in copies])
        ms = (C.c_double * k)()
        _check(self._lib, self._lib.cdprobe_ce_copy(self._h, k, loc, peer, 1 if push else 0, nbytes, reps, ms),
               "cdprobe_ce_copy")
        info = self.Info()
        pl = plan(info.n, self.cfg.bytes, self.cfg.mode, self.cfg.flags)
        nb = min(x for x in (nbytes or pl.src_bytes, pl.src_bytes, pl.land_bytes))
        return [(ms[i], nb * reps / (ms[i] * 1e-3) / 1e9 if ms[i] > 0 else 0.0) for i in range(k)]

    def Corrupt(self, local: int, byte_offset: int, xor_mask: int) -> None:
        _check(self._lib, self._lib.cdprobe_corrupt(self._h, local, byte_offset, xor_mask), "cdprobe_corrupt")

    def CorruptLanding(self, local: int, target: int, faults) -> None:
        """Test-only fault in transit: on every Run until disarmed, xor each (word index, mask) of `faults` into
        the landing slot local rank `local` writes in `target`, after the write and before the verify.  [] disarms."""
        _check(self._lib, self.corrupt_landing_raw(local, target, faults), "cdprobe_corrupt_landing")

    def corrupt_landing_raw(self, local: int, target: int, faults) -> int:
        """The bare ABI call: its return code."""
        k = len(faults)
        word = (C.c_uint64 * max(k, 1))(*[int(w) for w, _ in faults])
        mask = (C.c_uint64 * max(k, 1))(*[int(m) for _, m in faults])
        return self._lib.cdprobe_corrupt_landing(self._h, local, target, k, word, mask)

    def Diagnose(self, op, issuer: int, target: int, reader: Optional[int] = None) -> Diagnosis:
        """Go: (*Probe).Diagnose.  Re-reads cell (op, issuer, target) of the last Run on `reader`'s GPU (default: the
        issuer, i.e. through the fabric; the target reads it at rest) and diffs it against the pattern.
        op: abi.OP_READ / abi.OP_WRITE or "read" / "write"."""
        op = {"read": abi.OP_READ, "write": abi.OP_WRITE}.get(op, op)
        reader = issuer if reader is None else reader
        return self._decode("cdprobe_diagnose", Diagnosis, self.diagnose_raw(op, issuer, target, reader))

    def diagnose_raw(self, op: int, issuer: int, target: int, reader: int):
        """The bare ABI call: (return code, abi.DiagT as the library left it)."""
        return self._call("cdprobe_diagnose", abi.DiagT, op, issuer, target, reader)

    def Latency(self, hops: int = 0, reps: int = 0) -> Latency:
        """Go: (*Probe).Latency.  Dependent-load latency of every cell whose issuer is local (0: 1024 hops, 8 timed
        reps).  Needs no Run first and disturbs none."""
        return self._decode("cdprobe_latency", Latency, self.latency_raw(hops, reps))

    def latency_raw(self, hops: int, reps: int):
        """The bare ABI call: (return code, abi.LatencyT as the library left it)."""
        return self._call("cdprobe_latency", abi.LatencyT, hops, reps)

    def PingPong(self, trips: int = 0, reps: int = 0, fenced: bool = False) -> PingPong:
        """Go: (*Probe).PingPong.  Signal round trip of every off-diagonal cell over the tournament's pairs (0: 256
        round trips, 8 timed reps); fenced: a fence.sys before every store.  Collective when world_size > 1.  Needs no
        Run first and disturbs none."""
        return self._decode("cdprobe_pingpong", PingPong, self.pingpong_raw(trips, reps, 1 if fenced else 0))

    def pingpong_raw(self, trips: int, reps: int, fenced: int):
        """The bare ABI call: (return code, abi.PingPongT as the library left it)."""
        return self._call("cdprobe_pingpong", abi.PingPongT, trips, reps, fenced)

    def Atomics(self, kind: int, ops: int = 0, reps: int = 0) -> Atomics:
        """Go: (*Probe).Atomics.  Remote atomics of every cell whose issuer is local (kind: abi.ATOMIC_*; 0: 1024 ops
        per lane, 8 timed reps).  One-sided, not collective.  Needs no Run first and disturbs none."""
        return self._decode("cdprobe_atomics", Atomics, self.atomics_raw(kind, ops, reps))

    def atomics_raw(self, kind: int, ops: int, reps: int):
        """The bare ABI call: (return code, abi.AtomicsT as the library left it)."""
        return self._call("cdprobe_atomics", abi.AtomicsT, kind, ops, reps)

    def BwCurve(self, reps: int = 0) -> BwCurve:
        """Go: (*Probe).BwCurve.  Bandwidth versus transfer size of every cell whose issuer is local, on the probe's
        read path and grid (0: 8 timed reps per size).  Collective when world_size > 1.  Needs no Run first and
        disturbs none."""
        return self._decode("cdprobe_bwcurve", BwCurve, self.bwcurve_raw(reps))

    def bwcurve_raw(self, reps: int):
        """The bare ABI call: (return code, abi.BwCurveT as the library left it)."""
        return self._call("cdprobe_bwcurve", abi.BwCurveT, reps)

    def AllReduce(self, reps: int = 0) -> AllReduce:
        """Go: (*Probe).AllReduce.  One-shot all-reduce of every rank's source buffer on every rank at once, at each
        size of the bwcurve ladder, on the probe's read path and grid (0: 8 timed reps per size).  Collective when
        world_size > 1.  Needs no Run first and disturbs none."""
        return self._decode("cdprobe_allreduce", AllReduce, self.allreduce_raw(reps))

    def allreduce_raw(self, reps: int):
        """The bare ABI call: (return code, abi.AllReduceT as the library left it)."""
        return self._call("cdprobe_allreduce", abi.AllReduceT, reps)

    def AllReduceTwoShot(self, reps: int = 0) -> AllReduce:
        """Go: (*Probe).AllReduceTwoShot.  Two-shot all-reduce (reduce-scatter, then a pushed all-gather) of every
        rank's source buffer on every rank at once, at each size of the bwcurve ladder, on the probe's read path and
        grid (0: 8 timed reps per size).  The result is an AllReduce whose bad_words and first_bad cover every rep;
        the nccl-tests bus bandwidth is peak_gbps x 2 (n - 1) / n.  Collective when world_size > 1.  Needs no Run first
        and disturbs none."""
        return self._decode("cdprobe_allreduce_twoshot", AllReduce, self.allreduce_twoshot_raw(reps))

    def allreduce_twoshot_raw(self, reps: int):
        """The bare ABI call: (return code, abi.AllReduceT as the library left it)."""
        return self._call("cdprobe_allreduce_twoshot", abi.AllReduceT, reps)

    def AllReduceLL(self, reps: int = 0) -> AllReduce:
        """Go: (*Probe).AllReduceLL.  Low-latency all-reduce of every rank's source buffer on every rank at once:
        flag-carrying 16-byte packets pushed to every peer, no barrier or fence per rep, at each size of the LL ladder
        (the bwcurve ladder up to 1 MiB), on the probe's grids (0: 8 timed reps per size).  A rep is timed from the end
        of the rank's previous rep; path is abi.ALLREDUCE_PATH_LL.  Collective when world_size > 1.  Needs no Run
        first and disturbs none."""
        return self._decode("cdprobe_allreduce_ll", AllReduce, self.allreduce_ll_raw(reps))

    def allreduce_ll_raw(self, reps: int):
        """The bare ABI call: (return code, abi.AllReduceT as the library left it)."""
        return self._call("cdprobe_allreduce_ll", abi.AllReduceT, reps)

    def AllReduceRing(self, reps: int = 0) -> AllReduce:
        """Go: (*Probe).AllReduceRing.  Ring all-reduce of every rank's source buffer on every rank at once: each
        8 KiB unit is passed to the next rank under its own flag, 2 (n - 1) steps of reduce-scatter and all-gather
        with no barrier or fence between them, at each size of the bwcurve ladder, on the probe's grids (0: 8 timed
        reps per size).  A rep is timed from its opening barrier to the moment the rank's output is complete; path is
        abi.ALLREDUCE_PATH_RING.  Collective when world_size > 1.  Needs no Run first and disturbs none."""
        return self._decode("cdprobe_allreduce_ring", AllReduce, self.allreduce_ring_raw(reps))

    def allreduce_ring_raw(self, reps: int):
        """The bare ABI call: (return code, abi.AllReduceT as the library left it)."""
        return self._call("cdprobe_allreduce_ring", abi.AllReduceT, reps)

    def AllReducePush(self, reps: int = 0) -> AllReduce:
        """Go: (*Probe).AllReducePush.  Push all-reduce of every rank's source buffer on every rank at once, every byte
        moved as a write: each rank reduces every 8 KiB unit of its input into the unit's owner (bulk reductions on the
        TMA path, red.global per word on ld/st), then each owner pushes its finished chunk to every peer, at each size
        of the bwcurve ladder, on the probe's data path and grids (0: 8 timed reps per size).  A rep is timed from its
        opening to its closing barrier; path is the handle's.  Collective when world_size > 1.  Needs no Run first and
        disturbs none."""
        return self._decode("cdprobe_allreduce_push", AllReduce, self.allreduce_push_raw(reps))

    def allreduce_push_raw(self, reps: int):
        """The bare ABI call: (return code, abi.AllReduceT as the library left it)."""
        return self._call("cdprobe_allreduce_push", abi.AllReduceT, reps)

    def AllReduceNVLS(self, reps: int = 0) -> AllReduce:
        """Go: (*Probe).AllReduceNVLS.  Multicast (NVLS) all-reduce of every rank's source buffer on every rank at once:
        each rank sums its chunk of 8 KiB units with multimem.ld_reduce through one multicast object that spans the
        domain and stores each sum to every rank with one multimem.st, at each size of the bwcurve ladder (0: 8 timed
        reps per size).  A rep is timed from its opening to its closing barrier; path is ALLREDUCE_PATH_NVLS.  Rows are
        ERR_UNSUPPORTED, with nothing run, where the devices, the driver or a shared device rule multicast out.
        Collective when world_size > 1.  Needs no Run first and disturbs none."""
        return self._decode("cdprobe_allreduce_nvls", AllReduce, self.allreduce_nvls_raw(reps))

    def allreduce_nvls_raw(self, reps: int):
        """The bare ABI call: (return code, abi.AllReduceT as the library left it)."""
        return self._call("cdprobe_allreduce_nvls", abi.AllReduceT, reps)

    def AllToAll(self, reps: int = 0) -> AllToAll:
        """Go: (*Probe).AllToAll.  One-shot all-to-all: every rank pushes a block to every peer at once, at each size of
        the bwcurve ladder, on the probe's write path and grid, and every receiver checks every word (0: 8 timed reps
        per size).  Collective when world_size > 1.  Needs no Run first and disturbs none."""
        return self._decode("cdprobe_alltoall", AllToAll, self.alltoall_raw(reps))

    def alltoall_raw(self, reps: int):
        """The bare ABI call: (return code, abi.AllToAllT as the library left it)."""
        return self._call("cdprobe_alltoall", abi.AllToAllT, reps)

    def Memcpy(self, op: int, reps: int = 0) -> Memcpy:
        """Go: (*Probe).Memcpy.  Copy-engine bandwidth versus transfer size of every cell whose issuer is local:
        cudaMemcpyAsync of each size of the bwcurve ladder from the target into the issuer's exchange area (op
        abi.OP_READ, a pull) or from the issuer into the target's (abi.OP_WRITE, a push), each copy timed by CUDA events
        and every landed word checked (0: 8 timed reps per size).  Collective when world_size > 1.  Needs no Run first
        and disturbs none."""
        return self._decode("cdprobe_memcpy", Memcpy, self.memcpy_raw(op, reps))

    def memcpy_raw(self, op: int, reps: int):
        """The bare ABI call: (return code, abi.MemcpyT as the library left it)."""
        return self._call("cdprobe_memcpy", abi.MemcpyT, op, reps)

    def CeAllToAll(self, op: int, reps: int = 0) -> CeAllToAll:
        """Go: (*Probe).CeAllToAll.  Copy-engine all-to-all: in every rep every cell of Memcpy copies its block at
        once, each on a copy stream of its own, pulled (op abi.OP_READ) or pushed (abi.OP_WRITE), with the ranks
        signalling each other by stream memory operations, at each size of the bwcurve ladder; the owner of every block
        checks every word (0: 8 timed reps per size).  Collective when world_size > 1.  Needs no Run first and disturbs
        none."""
        return self._decode("cdprobe_ce_alltoall", CeAllToAll, self.ce_alltoall_raw(op, reps))

    def ce_alltoall_raw(self, op: int, reps: int):
        """The bare ABI call: (return code, abi.CeAllToAllT as the library left it)."""
        return self._call("cdprobe_ce_alltoall", abi.CeAllToAllT, op, reps)

    def Links(self) -> Links:
        """Go: (*Probe).Links.  The per-link NVLink counters of the last Run taken with abi.OPT_LINK_COUNTERS on, one
        entry per distinct local device.  One-sided, not collective."""
        return self._decode("cdprobe_links", Links, self._call("cdprobe_links", abi.LinksT))

    def Close(self) -> None:
        if self._h:
            self._lib.cdprobe_close(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.Close()

    def __del__(self):
        try:
            self.Close()
        except Exception:
            pass


def Open(cfg: Config) -> Probe:
    return Probe(cfg)


def topology(strict: bool = True) -> abi.TopologyT:
    """internal/common topology enumeration (NVML only, no CUDA)."""
    lib = abi.load_library()
    t = abi.TopologyT()
    _check(lib, lib.cdprobe_topology(1 if strict else 0, C.byref(t)), "cdprobe_topology")
    return t


def gate(cfg: Config, n_total: int):
    """(read, write) GB/s threshold the verdict of an n_total-rank domain with this config applies (host-only)."""
    lib = abi.load_library()
    r, w = C.c_float(), C.c_float()
    c = cfg.to_c()
    _check(lib, lib.cdprobe_gate(C.byref(c), n_total, C.byref(r), C.byref(w)), "cdprobe_gate")
    return r.value, w.value


def plan(n: int, nbytes: int, mode: int, flags: int = 0) -> abi.PlanT:
    lib = abi.load_library()
    p = abi.PlanT()
    _check(lib, lib.cdprobe_plan(n, nbytes, mode, flags, C.byref(p)), "cdprobe_plan")
    return p
