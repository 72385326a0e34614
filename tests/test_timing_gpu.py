"""The probe's numbers, not only its bytes: every rate, time and verdict field is checked against the raw stamps of
the run's own trace, an independent clock (CUDA events around each launch), the HBM ceiling, and a plain restatement
of the verdict (tests/verdict_ref.py).

- a. Rates and times equal the raw stamps exactly: gbps = float32(bpp / (t_end0 - t_start)) of the phase that
  carries the cell, device_ms = the last arrival, barrier_us = the gaps between phases; and the stamps are ordered.
- b. CUDA events bracket the kernel: device_ms <= kernel_ms <= event_ms (+ clock slack), event_ms <= probe_ms.
- c. Nothing beats HBM: the 1 GiB loop-back's rates stay under the H100 SXM data-sheet bandwidth.
- d. The verdict rules hold on real results (gate nobody meets, corrupt slice, torn mapping, MIG, diagonal, ops).
- e. cdprobe_gather merges counts, minima and verdicts of two processes as the restatement says.
- f. The on-demand measurements (latency, pingpong, atomics) normalise per hop / trip / op and fit in their call.

Several ranks share GPU 0 where a test needs N > 1, so the file runs on one H100.  The one-sided bounds in (b), (c)
and (f) only ever tighten if other contexts share the device: they can stretch event and host times, never shrink them.
"""
import subprocess
import textwrap
import time

import numpy as np
import pytest

import verdict_ref
from conftest import ROOT
from harness import run_children

pytestmark = pytest.mark.gpu

SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE: several ranks on one device
LOCAL_DIAG = 0x04
SIMULATE_MIG = 0x200

# cudaEventElapsedTime resolves about 0.5 us (CUDA Runtime API reference) and %globaltimer is a different clock;
# kernel_ms, measured inside the kernel, may exceed the events around it by no more than that disagreement.
EVENT_SLACK_MS = 0.002
# NVIDIA H100 SXM data sheet: 3.35 TB/s of HBM3.  A hard ceiling for any rate the loop-back reports.
HBM_DATASHEET_GBPS = 3350.0
# The write is stamped done when its stores have left the SMs; up to the 50 MB of L2 may still hold the last of them
# (5 % of 1 GiB), and the source read can start on lines still in L2.  Measured on an H100 80GB HBM3 at 400 W
# (profiles/h100_bench_n1.json): 3049 / 3175 GB/s per job, 3.17 TB/s for the pass, all under 1.0 x the data sheet.
HBM_MARGIN = 1.10
# Per-rep counts of the on-demand measurements: at C the fixed cost of a rep (its start and end stamps, the atom.exch
# that opens an atomics rep, the first trip's handshake) is under 1 % of the rep; 8C repeats the same op 8x longer.
ONDEMAND_C = 2048
ONDEMAND_REPS = 4
# Median per op at C and at 8C agree within this: the 1 % fixed cost plus the spread of a median of 4 reps on a device
# other contexts may share.  A per-rep count applied wrongly is off by a factor of 8 or more.
NORMALISATION_TOL = 0.10
# 64 KiB: the L2-resident region of the latency normalisation (the H100's L2 is 50 MB).
L2_REGION_BYTES = 64 << 10

N1_SIZES = [128, 8192 + 128, 1 << 20, 64 << 20, 1 << 30]
N1_SIZE_IDS = ["128B", "8KiB+128", "1MiB", "64MiB", "1GiB"]
PATHS = [0, 1, 2]
PATH_IDS = ["tma", "ldst", "ldst256"]
SAME_DEVICE_BYTES = 2 << 20


def card():
    """Name and power limit of GPU 0 (read-only query), for failure messages that carry absolute numbers."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown card"
    except (OSError, subprocess.SubprocessError):
        return "unknown card"


def traces_of(p):
    info = p.Info()
    return {info.first_local_rank + li: p.Trace(li) for li in range(info.n_local)}


def f32(x):
    return float(np.float32(x))


# ------------------------------------------------------------------ a. rates and times equal the stamps ----
def is_streamed_pass(tr):
    """The N = 1 loop-back pass: [write self] [read self || verify self], run without barriers."""
    return (len(tr) == 2 and tr[0]["job0"] == "write" and tr[0]["job1"] == "-" and tr[1]["job0"] == "read"
            and tr[1]["job1"] == "verify")


def check_stamps(res, traces):
    """gbps, device_ms and barrier_us of every local rank are the arithmetic of its trace's stamps, exactly, and the
    stamps are in the order the schedule runs them."""
    assert not res.aborted
    bpp = res.bytes_per_pair
    for li, (g, tr) in enumerate(sorted(traces.items())):
        carried = set()
        for p, ph in enumerate(tr):
            if ph["job0"] not in ("read", "write"):
                continue
            cell = (ph["job0"], ph["peer0"])
            assert cell not in carried, (g, cell)  # one phase carries each cell
            carried.add(cell)
            dt = ph["t_end0"] - ph["t_start"]
            want = f32(bpp / dt) if dt > 0 else 0.0
            got = getattr(res, "gbps_" + ph["job0"])[g][ph["peer0"]]
            assert got == want, (g, p, cell, got, want, ph)
        assert res.device_ms[li] == tr[-1]["t_arrive"] / 1e6, (g, res.device_ms[li], tr[-1])
        bar_ns = 0.0
        for ph, nx in zip(tr, tr[1:]):
            bar_ns += float(max(0, nx["t_start"] - ph["t_arrive"]))
        assert res.barrier_us[li] == bar_ns / 1e3, (g, res.barrier_us[li], bar_ns)
        if is_streamed_pass(tr):
            w, rv = tr
            assert w["t_start"] <= rv["t_start"], tr
            assert w["t_start"] <= w["t_end0"] == w["t_arrive"], tr  # the write's end closes phase 0
            assert rv["t_start"] <= rv["t_end0"] <= rv["t_arrive"], tr
            assert w["t_end0"] <= rv["t_end1"] <= rv["t_arrive"], tr  # no verify ends before the last write landed
        else:
            for p, ph in enumerate(tr):
                for jb in ("0", "1"):
                    if ph["job" + jb] != "-" and ph["t_end" + jb] > 0:
                        assert ph["t_start"] <= ph["t_end" + jb] <= ph["t_arrive"], (g, p, jb, ph)
                assert ph["t_start"] <= ph["t_arrive"], (g, p, ph)
                if p + 1 < len(tr):
                    assert ph["t_arrive"] <= tr[p + 1]["t_start"], (g, p, ph, tr[p + 1])


def check_events(res, n_local, wall_ms):
    """With CDPROBE_OPT_EVENT_TIMING: the CUDA events around each launch bracket the kernel's own clock, and the
    host clock brackets both.  probe_ms stops when the last row is published, which is before the kernels retire and
    their closing events fire (a rank launched first on a shared device retires a few us later), so the events are
    bounded by the wall clock of the whole call, which reads them back; probe_ms bounds the in-kernel clock."""
    for li in range(n_local):
        assert res.event_ms[li] > 0, li
        assert res.device_ms[li] <= res.kernel_ms[li] <= res.event_ms[li] + EVENT_SLACK_MS, \
            (li, res.device_ms[li], res.kernel_ms[li], res.event_ms[li])
        assert res.kernel_ms[li] <= res.probe_ms <= wall_ms, (li, res.kernel_ms[li], res.probe_ms, wall_ms)
        assert res.event_ms[li] <= wall_ms, (li, res.event_ms[li], wall_ms)


def run_and_check(pkg, p, ops, loopback, gate, n_local):
    """One run without and one with event timing: both checked against their stamps and the verdict restatement."""
    for timing in (0, 1):
        p.SetOption(pkg.abi.OPT_EVENT_TIMING, timing)
        t0 = time.perf_counter()
        res = p.Run()
        wall_ms = (time.perf_counter() - t0) * 1e3
        traces = traces_of(p)
        check_stamps(res, traces)
        verdict_ref.check(res, traces, ops, loopback, gate)
        if timing:
            check_events(res, n_local, wall_ms)
        else:
            assert all(e == 0 for e in res.event_ms)
            assert all(k <= res.probe_ms <= wall_ms for k in res.kernel_ms[:n_local])


@pytest.mark.parametrize("path", PATHS, ids=PATH_IDS)
@pytest.mark.parametrize("nbytes", N1_SIZES, ids=N1_SIZE_IDS)
def test_single_gpu_stamps_events_and_verdict(pkg, nbytes, path):
    cfg = pkg.Config(ordinals=[0], bytes=nbytes)
    with pkg.Open(cfg) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        run_and_check(pkg, p, 3, True, pkg.gate(cfg, 1), 1)
        assert is_streamed_pass(p.Trace(0))


SCHEDULES = {
    "default": (0, {}),
    "unidirectional": (0x80, {}),
    "serial-verify": (0x100, {}),
    "overlap-verify-3": (0x20, {"OPT_VERIFY_CTAS": 3}),
    "local-diag": (LOCAL_DIAG, {}),
    "all-rank-barriers": (0, {"OPT_ALL_RANK_BARRIERS": 1}),
    "pair-barriers": (0, {"OPT_PAIR_BARRIERS": 1}),
}


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("n", [2, 3, 5, 8])
def test_same_device_stamps_events_and_verdict(pkg, n, schedule):
    flags, opts = SCHEDULES[schedule]
    cfg = pkg.Config(ordinals=[0] * n, bytes=SAME_DEVICE_BYTES, flags=SAME | flags, ctas=8, timeout_ms=20000)
    with pkg.Open(cfg) as p:
        for name, value in opts.items():
            p.SetOption(getattr(pkg.abi, name), value)
        run_and_check(pkg, p, 3, bool(flags & LOCAL_DIAG), pkg.gate(cfg, n), n)


@pytest.mark.parametrize("ops", [1, 2], ids=["read", "write"])
@pytest.mark.parametrize("n", [1, 4])
def test_one_op_stamps_events_and_verdict(pkg, n, ops):
    cfg = (pkg.Config(ordinals=[0], bytes=1 << 20, ops=ops) if n == 1 else
           pkg.Config(ordinals=[0] * n, bytes=SAME_DEVICE_BYTES, ops=ops, flags=SAME, ctas=8, timeout_ms=20000))
    with pkg.Open(cfg) as p:
        run_and_check(pkg, p, ops, n == 1, pkg.gate(cfg, n), n)
        res = p.Run()
        other = res.gbps_write if ops == 1 else res.gbps_read
        assert all(x == 0 for row in other for x in row)  # the op that did not run has no rate


# ------------------------------------------------------------------------------- c. nothing beats HBM ----
@pytest.mark.parametrize("path", PATHS, ids=PATH_IDS)
def test_loopback_rates_stay_under_hbm(pkg, path):
    ceiling = HBM_MARGIN * HBM_DATASHEET_GBPS
    with pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 30)) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        p.Run()  # warm-up
        r = p.Run()
        assert r.verdict
        bpp = r.bytes_per_pair
        assert bpp == 1 << 30
        pass_gbps = 3 * bpp / r.kernel_ms[0] / 1e6  # read + write + verify of 1 GiB each, bytes per ms -> GB/s
        what = (f"{card()}: read {r.gbps_read[0][0]:.0f}, write {r.gbps_write[0][0]:.0f}, pass {pass_gbps:.0f} GB/s "
                f"over kernel_ms {r.kernel_ms[0]:.4f}; ceiling {ceiling:.0f} GB/s")
        assert 0 < r.gbps_read[0][0] <= ceiling, what
        assert 0 < r.gbps_write[0][0] <= ceiling, what
        assert 0 < pass_gbps <= ceiling, what


# ---------------------------------------------------------------------- d. the verdict on real results ----
UNMEETABLE = dict(min_fraction=0.99, link_peak_gbps=1e6)  # 990 TB/s per pair


def open_same(pkg, n, flags=0, nbytes=1 << 20, **kw):
    cfg = pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME | flags, ctas=8, timeout_ms=20000, **kw)
    return cfg, pkg.Open(cfg)


def test_verdict_gate_nobody_meets(pkg):
    n = 3
    cfg, p = open_same(pkg, n, **UNMEETABLE)
    with p:
        r = p.Run()
        want = verdict_ref.check(r, traces_of(p), 3, False, pkg.gate(cfg, n))
        assert want["slow_pairs"] == n * (n - 1) and want["unreachable_pairs"] == 0 and not want["verdict"]


def test_verdict_corrupt_slice_is_unreachable_not_slow(pkg):
    n = 4
    cfg, p = open_same(pkg, n, **UNMEETABLE)
    with p:
        bpp = p.Info().bytes_per_pair
        p.Corrupt(0, bpp + 64, 0xFF)  # slice 1 of rank 0's source: what rank 2 reads
        r = p.Run()
        assert r.reach_read[2][0] == 0 and r.reach_write[2][0] == 1
        want = verdict_ref.check(r, traces_of(p), 3, False, pkg.gate(cfg, n))
        assert want["unreachable_pairs"] == 1 and want["slow_pairs"] == n * (n - 1) - 1


def test_verdict_unmapped_peer(pkg):
    n = 4
    cfg, p = open_same(pkg, n)
    with p:
        p.UnmapPeer(1, 2)
        r = p.Run()
        want = verdict_ref.check(r, traces_of(p), 3, False, pkg.gate(cfg, n))
        assert want["unreachable_pairs"] == 2 and not want["verdict"]


def test_verdict_simulated_mig(pkg):
    n = 4
    cfg, p = open_same(pkg, n, SIMULATE_MIG | LOCAL_DIAG)
    with p:
        r = p.Run()
        want = verdict_ref.check(r, traces_of(p), 3, True, pkg.gate(cfg, n))
        assert want["verdict"] and want["unreachable_pairs"] == 0 and want["slow_pairs"] == 0


def test_verdict_local_diag_is_reported_not_gated(pkg):
    n = 4
    cfg, p = open_same(pkg, n, LOCAL_DIAG, min_fraction=1.0, link_peak_gbps=1e-3)  # gate = link_peak_gbps
    with p:
        r = p.Run()
        assert all(r.gbps_read[i][i] > 0 and r.gbps_write[i][i] > 0 for i in range(n))
        want = verdict_ref.check(r, traces_of(p), 3, True, pkg.gate(cfg, n))
        assert want["verdict"]
        # a gate between the slowest diagonal cell and the slowest off-diagonal one, where the rates allow it: the
        # diagonal under the gate is neither slow nor the minimum
        diag = min(min(r.gbps_read[i][i], r.gbps_write[i][i]) for i in range(n))
        off = min(min(r.gbps_read[i][j], r.gbps_write[i][j]) for i in range(n) for j in range(n) if i != j)
        if diag < off:
            mbps = int((diag * off) ** 0.5 * 1e3)
            p.SetOption(pkg.abi.OPT_LINK_PEAK_MBPS, mbps)
            cfg.link_peak_gbps = mbps / 1e3
            r = p.Run()
            verdict_ref.check(r, traces_of(p), 3, True, pkg.gate(cfg, n))


@pytest.mark.parametrize("ops", [1, 2, 3])
def test_verdict_single_gpu_ops(pkg, ops):
    cfg = pkg.Config(ordinals=[0], bytes=1 << 20, ops=ops)
    with pkg.Open(cfg) as p:
        r = p.Run()
        want = verdict_ref.check(r, traces_of(p), ops, True, pkg.gate(cfg, 1))
        assert want["verdict"] and r.gate_gbps_read == 0 and r.gate_gbps_write == 0


# ------------------------------------------------------------------------------------ e. gather ----
CHILD = textwrap.dedent(
    """
    import ctypes, dataclasses, json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world, nbytes, flags, ctas = sys.argv[1], *map(int, sys.argv[2:7])
    min_fraction, link_peak, corrupt = float(sys.argv[7]), float(sys.argv[8]), int(sys.argv[9])
    cfg = m.Config(ordinals=[0], bytes=nbytes, world_size=world, rank=rank, session=session, flags=flags, ctas=ctas,
                   timeout_ms=30000, min_fraction=min_fraction, link_peak_gbps=link_peak)

    def fields(res):
        return {k: v for k, v in dataclasses.asdict(res).items() if k != "raw"}

    runs = []
    with m.Open(cfg) as p:
        for run in range(2):
            if run == 1 and corrupt and rank == 0:
                p.Corrupt(0, 64, 0xFF)  # slice 0 of rank 0's source: what rank 1 reads
            r = m.abi.ResultT()
            assert p.run_raw(r) == m.abi.OK
            pre = fields(m.Result.from_c(m.abi.ResultT.from_buffer_copy(r)))
            assert p._lib.cdprobe_gather(p._h, ctypes.byref(r)) == m.abi.OK
            runs.append({"pre": pre, "post": fields(m.Result.from_c(r)), "trace": p.Trace(0)})
    print("RESULT " + json.dumps({"runs": runs, "gate": m.gate(cfg, world)}))
    """
) % ROOT

# fields that cdprobe_gather makes equal in every process (the per-local-rank times stay each process's own)
GATHERED = ("n", "row_mask", "verdict", "reach_read", "reach_write", "gbps_read", "gbps_write", "status", "sum_read",
            "xor_read", "sum_write", "xor_write", "bytes_per_pair", "run_seq", "aborted", "min_gbps_read",
            "min_gbps_write", "gate_gbps_read", "gate_gbps_write", "unreachable_pairs", "slow_pairs", "probe_ms")
ROW_FIELDS = ("reach_read", "reach_write", "gbps_read", "gbps_write", "status", "sum_read", "xor_read", "sum_write",
              "xor_write")


class SimpleResult:
    """A Result rebuilt from the child's JSON: the attributes verdict_ref reads."""

    def __init__(self, d):
        self.__dict__.update(d)


def run_two_processes(nbytes, min_fraction, link_peak, corrupt):
    return run_children(CHILD, 2, nbytes, 64, 8, min_fraction, link_peak, int(corrupt), timeout=300)


@pytest.mark.parametrize("case", ["healthy", "gate-nobody-meets", "corrupt-slice"])
def test_gather_merges_two_processes(pkg, case):
    nbytes = 1 << 20
    if case == "gate-nobody-meets":
        outs = run_two_processes(nbytes, UNMEETABLE["min_fraction"], UNMEETABLE["link_peak_gbps"], False)
    else:
        outs = run_two_processes(nbytes, 0.0, 1e-3, case == "corrupt-slice")  # a gate every pair meets
    gate = tuple(outs[0]["gate"])
    assert tuple(outs[1]["gate"]) == gate
    for run in range(2):
        pre = [o["runs"][run]["pre"] for o in outs]
        post = [o["runs"][run]["post"] for o in outs]
        traces = {rank: o["runs"][run]["trace"] for rank, o in enumerate(outs)}
        for rank in range(2):
            assert pre[rank]["row_mask"] == 1 << rank
            verdict_ref.check(SimpleResult(pre[rank]), {rank: traces[rank]}, 3, False, gate)
            for f in ROW_FIELDS:  # the gathered rows are their owners' rows
                assert post[0][f][rank] == post[1][f][rank] == pre[rank][f][rank], (run, rank, f)
        for f in GATHERED:
            assert post[0][f] == post[1][f], (run, f, post[0][f], post[1][f])
        want = verdict_ref.check(SimpleResult(post[0]), traces, 3, False, gate)
        assert post[0]["row_mask"] == 0b11
        assert want["unreachable_pairs"] == sum(p["unreachable_pairs"] for p in pre)
        assert want["slow_pairs"] == sum(p["slow_pairs"] for p in pre)
        assert want["verdict"] == all(p["verdict"] for p in pre)
        for op in ("read", "write"):
            assert post[0]["min_gbps_" + op] == min(p["min_gbps_" + op] for p in pre)
        if case == "healthy" or (case == "corrupt-slice" and run == 0):
            assert want["verdict"] and want["unreachable_pairs"] == want["slow_pairs"] == 0
        elif case == "gate-nobody-meets":
            assert not want["verdict"] and want["slow_pairs"] == 2 and want["unreachable_pairs"] == 0
        else:
            assert post[0]["reach_read"][1][0] == 0 and want["unreachable_pairs"] == 1
            assert not post[0]["verdict"] and not post[1]["verdict"]


# ---------------------------------------------------------------------- f. on-demand measurements ----
def timed_call(fn, **kw):
    t0 = time.perf_counter()
    out = fn(**kw)
    wall_ms = (time.perf_counter() - t0) * 1e3
    assert 0 < out.ms <= wall_ms, (out.ms, wall_ms)
    return out


def check_fits_in_call(m, per_rep, what):
    """Every measured cell's fastest rep, times the rep count, fits in the host wall clock of the call."""
    for i in range(m.n):
        for j in range(m.n):
            if not m.measured[i][j]:
                continue
            assert m.status[i][j] == 0, (what, i, j, m.status[i][j])
            busy_ms = m.reps * per_rep * m.ns_min[i][j] / 1e6
            assert busy_ms <= m.ms, (what, i, j, f"{m.reps} x {per_rep} x {m.ns_min[i][j]} ns > {m.ms} ms", card())


def check_normalised(small, large, i, j, what):
    ratio = large.ns_median[i][j] / small.ns_median[i][j]
    assert abs(ratio - 1) <= NORMALISATION_TOL, (what, small.ns_median[i][j], large.ns_median[i][j], card())


def test_latency_per_hop(pkg):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=L2_REGION_BYTES)) as p:
        runs = [timed_call(p.Latency, hops=h, reps=ONDEMAND_REPS) for h in (ONDEMAND_C, 8 * ONDEMAND_C)]
        for lat in runs:
            assert lat.region_bytes == L2_REGION_BYTES and lat.measured[0][0]
            check_fits_in_call(lat, lat.hops, "latency")  # per_rep: hops (summarize in cdprobe_latency)
        check_normalised(*runs, 0, 0, "latency")


@pytest.mark.parametrize("fenced", [False, True], ids=["plain", "fenced"])
def test_pingpong_per_trip(pkg, fenced):
    _, p = open_same(pkg, 2)
    with p:
        runs = [timed_call(p.PingPong, trips=t, reps=ONDEMAND_REPS, fenced=fenced) for t in (ONDEMAND_C, 8 * ONDEMAND_C)]
        for pp in runs:
            assert pp.measured[0][1] and pp.measured[1][0]
            check_fits_in_call(pp, pp.trips, "pingpong")  # per_rep: trips (summarize in cdprobe_pingpong)
        for i, j in ((0, 1), (1, 0)):
            check_normalised(*runs, i, j, "pingpong")


@pytest.mark.parametrize("kind", [0, 1, 2], ids=["fetch_add", "cas", "contended"])
def test_atomics_per_op(pkg, kind):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 20)) as p:
        runs = [timed_call(p.Atomics, kind=kind, ops=o, reps=ONDEMAND_REPS) for o in (ONDEMAND_C, 8 * ONDEMAND_C)]
        for at in runs:
            assert at.measured[0][0] and at.lanes == (32 if kind == 2 else 1)
            check_fits_in_call(at, at.lanes * at.ops, "atomics")  # per_rep: lanes x ops (summarize in cdprobe_atomics)
        check_normalised(*runs, 0, 0, "atomics")
