"""What every on-demand measurement does when it refuses a call: the return code, the exact cdprobe_last_error() text,
an output that holds the ABI version and the prologue fields the call fills before it refuses (everything else zero),
and a call number that a refusal does not advance.  Where one call has two reasons to refuse, the one that wins is
fixed: pingpong reports an invalid armed fault instead of its argument error, while atomics, the three all-reduces
and all-to-all report the argument error; memcpy and the copy-engine all-to-all refuse their reps, and the copy-engine
all-to-all reports its reps over its op, its op over its armed fault, and all three over its hardware queues.  Two
processes refuse together: the one with invalid arguments gets its own message, the other is told another process was
at fault, and arguments that differ refuse both; a process without the hardware queues for the copy-engine all-to-all
names its need and its limit, and the other is told another process cannot run it."""
import ctypes as C
import json
import os
import subprocess
import sys
import textwrap
import uuid

import pytest

import allreduce_ll_ref
import bwcurve_ref
from conftest import ROOT

pytestmark = pytest.mark.gpu

SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
MODE_SLICED = 1
ERR_ARG = -2
N, NBYTES = 2, 1 << 20

ARGS_LATENCY = "hops must be at most 1 << 20 and reps at most 64"
ARGS_PINGPONG = "trips must be at most 1 << 16, reps at most 64 and fenced 0 or 1"
ARGS_ATOMICS = "kind must be a CDPROBE_ATOMIC_*, ops at most 1 << 16 and reps at most 64"
ARGS_REPS = "reps must be at most 64"
FAULT_PINGPONG_CELL = "the armed pingpong fault names no off-diagonal cell"
FAULT_PINGPONG_TRIP = "the armed pingpong fault's trip must be below trips - 1, and below trips - 2 when reps is 1"
FAULT_ATOMICS = "the armed atomics fault names no cell of this domain"
FAULT_ALLREDUCE = "the armed all-reduce fault names no rank, size or output word of this call"
FAULT_TWOSHOT = "the armed two-shot all-reduce fault names no receiver, size or output word of this call"
FAULT_LL = "the armed LL all-reduce fault names no packet, size or delay of this call"
FAULT_ALLTOALL = "the armed all-to-all fault names no cell, size or word of this call"
ARGS_OP = "op must be CDPROBE_OP_READ or CDPROBE_OP_WRITE"
FAULT_CE_ALLTOALL = ("the armed copy-engine all-to-all fault names no cell, size, word or delay of this call, or has a "
                     "mode above 2")
QUEUES_OTHER = ("cdprobe_ce_alltoall: another process cannot run it (no stream memory operations, or more streams than "
                "CUDA_DEVICE_MAX_CONNECTIONS)")
ERR_UNSUPPORTED = -8


@pytest.fixture(scope="module")
def probe(pkg):
    with pkg.Open(pkg.Config(ordinals=[0] * N, bytes=NBYTES, mode=MODE_SLICED, flags=SAME, ctas=8,
                             timeout_ms=20000)) as p:
        yield p


def bpp(pkg):
    return pkg.plan(N, NBYTES, MODE_SLICED).bytes_per_pair


def expect(cls, **fields):
    t = cls()
    C.memset(C.byref(t), 0, C.sizeof(t))
    t.abi = 2
    for k, v in fields.items():
        setattr(t, k, v)
    return bytes(t)


def check_refused(p, rc, got, message, want):
    assert rc == ERR_ARG
    assert p._lib.cdprobe_last_error().decode() == message
    assert bytes(got) == want


# ---- latency: not collective, no call number -------------------------------------------------------------------------

@pytest.mark.parametrize("hops, reps", [(1 << 20 | 1, 2), (64, 65), (1 << 21, 1 << 31)], ids=["hops", "reps", "both"])
def test_latency_refuses_its_arguments(pkg, probe, hops, reps):
    a = pkg.abi
    rc, t = probe.latency_raw(hops, reps)
    check_refused(probe, rc, t, ARGS_LATENCY,
                  expect(a.LatencyT, n=N, hops=hops, reps=reps, region_bytes=bpp(pkg)))
    rc, t = probe.latency_raw(64, 1)
    assert rc == 0 and t.measured[1] and t.status[1] == 0


# ---- pingpong --------------------------------------------------------------------------------------------------------

def arm(p, fault):
    """Arms (option, value) when given; returns a function that disarms it."""
    if fault is not None:
        p.SetOption(*fault)
    return lambda: fault is not None and p.SetOption(fault[0], 0)


def pingpong_refusal(pkg, p, trips, reps, fenced, message, fault=None):
    seq = p.PingPong(trips=64, reps=1).call_seq
    disarm = arm(p, fault)
    rc, t = p.pingpong_raw(trips, reps, fenced)
    want = expect(pkg.abi.PingPongT, n=N, trips=trips or 256, reps=reps or 8, fenced=fenced)
    check_refused(p, rc, t, message, want)
    disarm()
    assert p.PingPong(trips=64, reps=1).call_seq == seq + 1


@pytest.mark.parametrize("trips, reps, fenced", [(1 << 16 | 1, 2, 0), (64, 65, 0), (64, 2, 2)],
                         ids=["trips", "reps", "fenced"])
def test_pingpong_refuses_its_arguments(pkg, probe, trips, reps, fenced):
    pingpong_refusal(pkg, probe, trips, reps, fenced, ARGS_PINGPONG)


@pytest.mark.parametrize("fault, trips, reps, message", [
    ((0, 0, 0), 64, 2, FAULT_PINGPONG_CELL),
    ((0, 2, 0), 64, 2, FAULT_PINGPONG_CELL),
    ((2, 0, 0), 64, 2, FAULT_PINGPONG_CELL),
    ((0, 1, 63), 64, 2, FAULT_PINGPONG_TRIP),
    ((1, 0, 62), 64, 1, FAULT_PINGPONG_TRIP),
], ids=["diagonal", "target", "initiator", "trip", "trip-one-rep"])
def test_pingpong_refuses_an_armed_fault(pkg, probe, fault, trips, reps, message):
    a = pkg.abi
    pingpong_refusal(pkg, probe, trips, reps, 0, message, (a.OPT_PINGPONG_FAULT, a.pingpong_fault(*fault)))


def test_pingpong_reports_an_invalid_fault_over_its_arguments(pkg, probe):
    a = pkg.abi
    pingpong_refusal(pkg, probe, 64, 65, 0, FAULT_PINGPONG_CELL, (a.OPT_PINGPONG_FAULT, a.pingpong_fault(0, 0, 0)))
    # a fault that is valid for these trips leaves the argument error in place
    pingpong_refusal(pkg, probe, 64, 65, 0, ARGS_PINGPONG, (a.OPT_PINGPONG_FAULT, a.pingpong_fault(0, 1, 3)))


# ---- atomics: not collective -----------------------------------------------------------------------------------------

def atomics_refusal(pkg, p, kind, ops, reps, message, fault=None):
    a = pkg.abi
    seq = p.Atomics(a.ATOMIC_FETCH_ADD, ops=64, reps=1).call_seq
    disarm = arm(p, fault)
    rc, t = p.atomics_raw(kind, ops, reps)
    want = expect(a.AtomicsT, n=N, kind=kind, ops=ops or 1024, reps=reps or 8,
                  lanes=32 if kind == a.ATOMIC_CONTENDED else 1)
    check_refused(p, rc, t, message, want)
    disarm()
    assert p.Atomics(a.ATOMIC_FETCH_ADD, ops=64, reps=1).call_seq == seq + 1


@pytest.mark.parametrize("kind, ops, reps", [(3, 64, 2), (2, 1 << 16 | 1, 2), (0, 64, 65)], ids=["kind", "ops", "reps"])
def test_atomics_refuses_its_arguments(pkg, probe, kind, ops, reps):
    atomics_refusal(pkg, probe, kind, ops, reps, ARGS_ATOMICS)


@pytest.mark.parametrize("fault", [(0, 0), (2, 0), (0, 2)], ids=["diagonal", "issuer", "target"])
def test_atomics_refuses_an_armed_fault(pkg, probe, fault):
    a = pkg.abi
    atomics_refusal(pkg, probe, a.ATOMIC_CAS, 64, 2, FAULT_ATOMICS, (a.OPT_ATOMICS_FAULT, a.atomics_fault(*fault)))


def test_atomics_reports_its_arguments_over_an_invalid_fault(pkg, probe):
    a = pkg.abi
    atomics_refusal(pkg, probe, a.ATOMIC_FETCH_ADD, 64, 65, ARGS_ATOMICS, (a.OPT_ATOMICS_FAULT, a.atomics_fault(0, 0)))


# ---- bwcurve, the all-reduces and all-to-all: the size ladder --------------------------------------------------------

LADDER_CALLS = ["bwcurve", "allreduce", "allreduce_twoshot", "allreduce_ll", "alltoall"]


def ladder_refusal(pkg, p, what, reps, message, fault=None):
    a = pkg.abi
    call = {"bwcurve": p.BwCurve, "allreduce": p.AllReduce, "allreduce_twoshot": p.AllReduceTwoShot,
            "allreduce_ll": p.AllReduceLL, "alltoall": p.AllToAll}[what]
    raw = getattr(p, what + "_raw")
    cls = {"bwcurve": a.BwCurveT, "alltoall": a.AllToAllT}.get(what, a.AllReduceT)
    path = a.ALLREDUCE_PATH_LL if what == "allreduce_ll" else 0
    seq = call(reps=1).call_seq
    disarm = arm(p, fault)
    rc, t = raw(reps)
    check_refused(p, rc, t, message, expect(cls, n=N, reps=reps or 8, path=path))
    disarm()
    assert call(reps=1).call_seq == seq + 1


@pytest.mark.parametrize("what", LADDER_CALLS)
def test_ladder_calls_refuse_their_reps(pkg, probe, what):
    ladder_refusal(pkg, probe, what, 65, ARGS_REPS)
    ladder_refusal(pkg, probe, what, 1 << 31, ARGS_REPS)


def test_allreduce_refuses_an_armed_fault(pkg, probe):
    a = pkg.abi
    sizes = bwcurve_ref.ladder(bpp(pkg))
    for fault in (a.allreduce_fault(N, 0, 0), a.allreduce_fault(0, len(sizes), 0),
                  a.allreduce_fault(0, 0, sizes[0] // 8), (1 << 24) | 5, (1 << 32) | 5):
        ladder_refusal(pkg, probe, "allreduce", 2, FAULT_ALLREDUCE, (a.OPT_ALLREDUCE_FAULT, fault))


def test_allreduce_twoshot_refuses_an_armed_fault(pkg, probe):
    a = pkg.abi
    sizes = bwcurve_ref.ladder(bpp(pkg))
    for fault in (a.allreduce_twoshot_fault(N, 0, 0), a.allreduce_twoshot_fault(0, len(sizes), 0),
                  a.allreduce_twoshot_fault(0, 0, sizes[0] // 8), (1 << 24) | 5, (1 << 32) | 5,
                  (1 << 49) | a.allreduce_twoshot_fault(0, 0, 0), (1 << 63) | a.allreduce_twoshot_fault(1, 1, 1)):
        ladder_refusal(pkg, probe, "allreduce_twoshot", 2, FAULT_TWOSHOT, (a.OPT_ALLREDUCE_TWOSHOT_FAULT, fault))


def test_allreduce_ll_refuses_an_armed_fault(pkg, probe):
    """On LL's own ladder; a delay of 10 s is half the handle's 20 s timeout, which LL refuses."""
    a = pkg.abi
    sizes = allreduce_ll_ref.ladder(bpp(pkg))
    for fault in (a.allreduce_ll_fault(N, 0, 0, 0), a.allreduce_ll_fault(0, N, 0, 0),
                  a.allreduce_ll_fault(0, 1, len(sizes), 0), a.allreduce_ll_fault(0, 1, 0, sizes[0] // 8),
                  a.allreduce_ll_fault(1, 1, 0, 0), a.allreduce_ll_fault(0, 1, 0, 10_000_000, mode=1),
                  (2 << 48) | a.allreduce_ll_fault(0, 1, 0, 0), (1 << 63) | a.allreduce_ll_fault(0, 1, 0, 0),
                  (1 << 24) | 5):
        ladder_refusal(pkg, probe, "allreduce_ll", 2, FAULT_LL, (a.OPT_ALLREDUCE_LL_FAULT, fault))


def test_alltoall_refuses_an_armed_fault(pkg, probe):
    a = pkg.abi
    sizes = bwcurve_ref.ladder(bpp(pkg))
    for fault in (a.alltoall_fault(0, 0, 0, 0), a.alltoall_fault(N, 0, 0, 0), a.alltoall_fault(0, N, 0, 0),
                  a.alltoall_fault(0, 1, len(sizes), 0), a.alltoall_fault(1, 0, 0, sizes[0] // 8)):
        ladder_refusal(pkg, probe, "alltoall", 2, FAULT_ALLTOALL, (a.OPT_ALLTOALL_FAULT, fault))


@pytest.mark.parametrize("what", LADDER_CALLS[1:])
def test_ladder_calls_report_their_reps_over_an_invalid_fault(pkg, probe, what):
    a = pkg.abi
    fault = {"allreduce": (a.OPT_ALLREDUCE_FAULT, a.allreduce_fault(N, 0, 0)),
             "allreduce_twoshot": (a.OPT_ALLREDUCE_TWOSHOT_FAULT, a.allreduce_twoshot_fault(N, 0, 0)),
             "allreduce_ll": (a.OPT_ALLREDUCE_LL_FAULT, a.allreduce_ll_fault(N, 0, 0, 0)),
             "alltoall": (a.OPT_ALLTOALL_FAULT, a.alltoall_fault(0, 0, 0, 0))}[what]
    ladder_refusal(pkg, probe, what, 65, ARGS_REPS, fault)


# ---- memcpy and the copy-engine all-to-all: an op and the size ladder ------------------------------------------------

def op_ladder_refusal(pkg, p, what, op, reps, message, fault=None):
    """cdprobe_memcpy or cdprobe_ce_alltoall refused with `message`: the prologue holds n, reps and op, the call number
    does not advance, and the next valid call runs."""
    a = pkg.abi
    call, raw, cls = {"memcpy": (p.Memcpy, p.memcpy_raw, a.MemcpyT),
                      "ce_alltoall": (p.CeAllToAll, p.ce_alltoall_raw, a.CeAllToAllT)}[what]
    seq = call(a.OP_READ, reps=1).call_seq
    disarm = arm(p, fault)
    rc, t = raw(op, reps)
    check_refused(p, rc, t, message, expect(cls, n=N, reps=reps or 8, op=op))
    disarm()
    assert call(a.OP_WRITE, reps=1).call_seq == seq + 1


@pytest.mark.parametrize("what", ["memcpy", "ce_alltoall"])
def test_memcpy_and_ce_alltoall_refuse_their_reps(pkg, probe, what):
    for op in (pkg.abi.OP_READ, pkg.abi.OP_WRITE):
        op_ladder_refusal(pkg, probe, what, op, 65, ARGS_REPS)
    op_ladder_refusal(pkg, probe, what, pkg.abi.OP_WRITE, 1 << 31, ARGS_REPS)


def test_ce_alltoall_refuses_its_op_and_an_armed_fault_in_that_order(pkg, probe):
    a = pkg.abi
    sizes = bwcurve_ref.ladder(bpp(pkg))
    for op in (0, 3, 4):
        op_ladder_refusal(pkg, probe, "ce_alltoall", op, 2, ARGS_OP)
    for fault in (a.ce_alltoall_fault(0, 0, 0, 0), a.ce_alltoall_fault(N, 0, 0, 0), a.ce_alltoall_fault(0, N, 0, 0),
                  a.ce_alltoall_fault(0, 1, len(sizes), 0), a.ce_alltoall_fault(1, 0, 0, sizes[0] // 8),
                  a.ce_alltoall_fault(1, 0, 0, sizes[0] // 8, mode=1), a.ce_alltoall_fault(0, 1, 0, 10_000_000, mode=2),
                  (3 << 48) | a.ce_alltoall_fault(0, 1, 0, 0), (1 << 32) | (1 << 24), (1 << 40) | (1 << 24)):
        op_ladder_refusal(pkg, probe, "ce_alltoall", a.OP_READ, 2, FAULT_CE_ALLTOALL, (a.OPT_CE_ALLTOALL_FAULT, fault))
    bad = (a.OPT_CE_ALLTOALL_FAULT, a.ce_alltoall_fault(0, 0, 0, 0))
    op_ladder_refusal(pkg, probe, "ce_alltoall", 3, 2, ARGS_OP, bad)  # the op over the fault
    op_ladder_refusal(pkg, probe, "ce_alltoall", 3, 65, ARGS_REPS, bad)  # the reps over both


# ---- two processes ---------------------------------------------------------------------------------------------------

CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank = sys.argv[1], int(sys.argv[2])
    cfg = m.Config(ordinals=[0], bytes=1 << 20, world_size=2, rank=rank, session=session, flags=0x40, ctas=8,
                   timeout_ms=30000)
    out = {}
    with m.Open(cfg) as p:
        lib = p._lib
        calls = {"pingpong": lambda reps: p.pingpong_raw(64, reps, 0), "bwcurve": p.bwcurve_raw,
                 "allreduce": p.allreduce_raw, "allreduce_twoshot": p.allreduce_twoshot_raw,
                 "allreduce_ll": p.allreduce_ll_raw, "alltoall": p.alltoall_raw}
        for name, call in calls.items():
            got = []
            for reps in (65 if rank == 0 else 2, 2 + rank, 2):  # invalid in one process, then different, then alike
                rc, t = call(reps)
                got.append({"rc": rc, "error": lib.cdprobe_last_error().decode(), "call_seq": t.call_seq})
            out[name] = got
    print("RESULT " + json.dumps(out))
    """
) % ROOT


def run_processes(world):
    """Runs CHILD in `world` processes of one domain; any still running when the time is up is killed."""
    session = f"refuse-{uuid.uuid4().hex[:12]}"
    procs = [subprocess.Popen([sys.executable, "-c", CHILD, session, str(r)], stdout=subprocess.PIPE,
                              stderr=subprocess.PIPE, text=True) for r in range(world)]
    outs = []
    try:
        for pr in procs:
            so, se = pr.communicate(timeout=600)
            assert pr.returncode == 0, se[-2000:]
            outs.append(json.loads([l for l in so.splitlines() if l.startswith("RESULT ")][-1][7:]))
    finally:
        for pr in procs:
            if pr.poll() is None:
                pr.kill()
                pr.wait()
    return outs


def test_two_processes_refuse_together():
    outs = run_processes(2)
    for rank, o in enumerate(outs):
        for name in ["pingpong"] + LADDER_CALLS:
            fn = "cdprobe_" + name
            own = ARGS_PINGPONG if name == "pingpong" else ARGS_REPS
            bad, differ, ok = o[name]
            assert bad == {"rc": ERR_ARG, "call_seq": 0,
                           "error": own if rank == 0 else f"another process called {fn} with invalid arguments"}
            assert differ == {"rc": ERR_ARG, "call_seq": 0,
                              "error": f"{fn} is collective: every process must call it with the same arguments"}
            assert ok == {"rc": 0, "error": "", "call_seq": 1}, (rank, name)


QUEUES_CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank = sys.argv[1], int(sys.argv[2])
    cfg = m.Config(ordinals=[0] * 3, bytes=1 << 20, world_size=2, rank=rank, session=session, flags=0x50, ctas=8,
                   timeout_ms=30000)
    out = []
    with m.Open(cfg) as p:
        lib = p._lib
        for op, reps in ((m.abi.OP_WRITE, 65), (m.abi.OP_READ, 2), (m.abi.OP_WRITE, 1)):
            rc, t = p.ce_alltoall_raw(op, reps)
            out.append({"rc": rc, "error": lib.cdprobe_last_error().decode(), "call_seq": t.call_seq,
                        "measured": sum(t.measured)})
        mc = p.Memcpy(m.abi.OP_WRITE, reps=1)
        out.append({"call_seq": mc.call_seq, "row_mask": mc.row_mask,
                    "clean": all(mc.status[g][j] == 0 and mc.bad_sizes[g][j] == 0 for g in range(6) for j in range(6)
                                 if mc.row_mask >> g & 1 and g != j),
                    "measured": sum(mc.measured[g][j] for g in range(6) for j in range(6))})
    print("RESULT " + json.dumps(out))
    """
) % ROOT


def test_a_process_without_the_queues_refuses_the_copy_engine_alltoall_in_both():
    """Two processes of three ranks each on one device (n = 6): each needs 18 hardware queues.  Process 0 has 8,
    process 1 has 32.  Invalid reps are refused first in both, with their own text; then process 0 names its need and
    its limit and process 1 is told another process cannot run it.  Nothing advances, and memcpy then runs clean."""
    session = f"refuse-q-{uuid.uuid4().hex[:12]}"
    procs = [subprocess.Popen([sys.executable, "-c", QUEUES_CHILD, session, str(r)], stdout=subprocess.PIPE,
                              stderr=subprocess.PIPE, text=True,
                              env=dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS=str(limit)))
             for r, limit in enumerate((8, 32))]
    outs = []
    try:
        for pr in procs:
            so, se = pr.communicate(timeout=600)
            assert pr.returncode == 0, se[-2000:]
            outs.append(json.loads([l for l in so.splitlines() if l.startswith("RESULT ")][-1][7:]))
    finally:
        for pr in procs:
            if pr.poll() is None:
                pr.kill()
                pr.wait()
    own = "cdprobe_ce_alltoall: needs 18 queues on ordinal 0, CUDA_DEVICE_MAX_CONNECTIONS allows 8"
    for rank, o in enumerate(outs):
        reps, first, second, mc = o
        assert reps == {"rc": ERR_ARG, "error": ARGS_REPS, "call_seq": 0, "measured": 0}, (rank, reps)
        for got in (first, second):
            assert got == {"rc": ERR_UNSUPPORTED, "error": own if rank == 0 else QUEUES_OTHER, "call_seq": 0,
                           "measured": 0}, (rank, got)
        assert mc == {"call_seq": 1, "row_mask": 0b111 << (3 * rank), "clean": True, "measured": 3 * 5}, (rank, mc)
