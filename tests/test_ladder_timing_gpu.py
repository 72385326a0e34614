"""Where the ladder measurements' times come from: every rep window against the HBM traffic it must hold, the call it
runs in, and the slowest rank of a barrier-closed collective.

- Floor.  With reps = 1 a rank's one timed rep per size is exact (min = median = max).  At every size of 512 MiB and
  more, the slowest rank's rep plus 20 us must reach tests/ladder_traffic.py's floor: the rep's unique bytes, less
  what L2 can hold, at the data-sheet HBM rate.  N = 1 on all three data paths for bwcurve, the one-shot, two-shot and
  push all-reduces and the all-to-all; the ring, both ops of memcpy and both ops of the CE all-to-all have one path.
  N = 2 and 4 ranks on one device for the collectives.  A window that closes before the rep's work (a t_end stamped
  after the opening barrier, a two-shot or push rep closed at its first barrier) falls far below it.
- Windows fit in the call.  With reps = 3, (min, median, max) are exactly the three timed reps, which run one after
  another on each rank: their sum over every size (and every cell a rank issues, which run in rounds one after
  another) is at most the call's own `ms`, which is at most this test's perf_counter around the call.  Every summary
  is the restatement of its medians, at scale `blocks` for the two all-to-alls.  N = 1 and 3, every measurement above
  and the LL all-reduce.
- The rep spans the slowest rank, for the push all-reduce, whose closing domain barrier stamps t_end: with one rank on
  a single CTA, every rank's rep is as long as that one's (the two-shot has the same test).  The one-shot, bwcurve and
  the all-to-all close a rank's window at its own last CTA stamp, so the floor covers them instead.

Every bound is one-sided: other contexts on the card can only stretch a window or a call, never shrink one.  Each test
first checks the device's free memory by arithmetic and skips, naming both figures, when it is short.  The CE
all-to-all runs in a child process with CUDA_DEVICE_MAX_CONNECTIONS=32, as its own tests do."""
import json
import textwrap
import time

import pytest

import alltoall_ref
import bwcurve_ref
import ladder_traffic as lt
from conftest import ROOT
from harness import run_children
from test_timing_gpu import card

pytestmark = pytest.mark.gpu

GIB = 1 << 30
MIB = 1 << 20
FLOOR_FROM = 512 * MIB  # sizes that cannot stay in the 50 MB L2
SLACK_NS = 20_000       # the spread of the ranks' releases, and the clock's resolution
SAME = 0x40 | 0x10      # ALLOW_SAME_DEVICE | NO_COOPERATIVE
MODE_SLICED = 1
VMM = 2 << 20
HEADROOM = 4 * GIB
SPARE = 64 << 20
PATHS = (0, 1, 2)       # TMA, 16-byte ld/st, 32-byte ld/st
OPS = (lt.OP_READ, lt.OP_WRITE)

# name: (Probe method, whether it takes an op, whether it reports cells [issuer][target] rather than ranks)
CALLS = {"bwcurve": ("BwCurve", False, True), "allreduce": ("AllReduce", False, False),
         "twoshot": ("AllReduceTwoShot", False, False), "ring": ("AllReduceRing", False, False),
         "push": ("AllReducePush", False, False), "ll": ("AllReduceLL", False, False),
         "alltoall": ("AllToAll", False, False), "memcpy": ("Memcpy", True, True)}
ON_PATH = ("bwcurve", "allreduce", "twoshot", "push", "alltoall")


def round_up(v, a):
    return -(-v // a) * a


def guard(pkg, n, nbytes, flags=0):
    """Skip unless the device has, per rank, its probe allocation, room for n + 4 blocks of bytes_per_pair (the
    exchange area, the gather, ring and push areas and the one-shot's output) and SPARE, plus HEADROOM free."""
    import torch

    pl = pkg.plan(n, nbytes, MODE_SLICED, flags)
    per_rank = VMM + round_up(pl.src_bytes, VMM) + round_up(pl.land_bytes, VMM)
    need = n * (per_rank + (n + 4) * round_up(pl.bytes_per_pair, VMM) + SPARE)
    free, _ = torch.cuda.mem_get_info(0)
    if free < need + HEADROOM:
        pytest.skip(f"needs {need} bytes plus {HEADROOM} spare on the device; {free} free")


def config(pkg, n, bpp, flags=0):
    return pkg.Config(ordinals=[0] * n, bytes=bpp * max(n - 1, 1), mode=MODE_SLICED,
                      flags=(SAME if n > 1 else 0) | flags, ctas=16 if n > 1 else 0, timeout_ms=120000)


def open_bpp(pkg, n, bpp, flags=0):
    guard(pkg, n, bpp * max(n - 1, 1), flags)
    p = pkg.Open(config(pkg, n, bpp, flags))
    assert p.Info().bytes_per_pair == bpp
    return p


def rows(name, m):
    """{rank or cell: (ns_min, ns_median, ns_max) per size} of every entry that ran."""
    out = {}
    if CALLS.get(name, (None, False, False))[2]:
        for i, row in enumerate(m.ns_min):
            for j, v in enumerate(row):
                if v is not None:
                    out[(i, j)] = (v, m.ns_median[i][j], m.ns_max[i][j])
    else:
        for r, v in enumerate(m.ns_min):
            if v is not None:
                out[r] = (v, m.ns_median[r], m.ns_max[r])
    return out


def call(p, name, reps, op=None):
    meth, takes_op, _ = CALLS[name]
    t = time.perf_counter()
    m = getattr(p, meth)(op, reps) if takes_op else getattr(p, meth)(reps=reps)
    return m, (time.perf_counter() - t) * 1e3


CE_CHILD = textwrap.dedent(
    """
    import json, sys, time
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    n, bpp, reps = int(sys.argv[4]), int(sys.argv[5]), int(sys.argv[6])
    cfg = m.Config(ordinals=[0] * n, bytes=bpp * max(n - 1, 1), mode=1, flags=0x50 if n > 1 else 0,
                   ctas=16 if n > 1 else 0, timeout_ms=120000)
    out = []
    with m.Open(cfg) as p:
        for op in (m.abi.OP_READ, m.abi.OP_WRITE):
            t0 = time.perf_counter()
            c = p.CeAllToAll(op, reps)
            wall_ms = (time.perf_counter() - t0) * 1e3
            out.append({"wall_ms": wall_ms, **{k: getattr(c, k) for k in (
                "n", "op", "reps", "sizes", "ms", "measured", "status", "blocks", "t0_ns", "peak_gbps", "half_bytes",
                "ns_min", "ns_median", "ns_max")}})
    print("RESULT " + json.dumps(out))
    """
) % ROOT


def ce_calls(pkg, monkeypatch, n, bpp, reps):
    """Both ops of cdprobe_ce_alltoall on n ranks of one device, in a child process with 32 hardware queues."""
    guard(pkg, n, bpp * max(n - 1, 1))
    monkeypatch.setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    return run_children(CE_CHILD, 1, n, bpp, reps)[0]


def margins(tag, name, n, sizes, per_rank, op=lt.OP_READ):
    """Asserts the floor at every size of FLOOR_FROM or more: the slowest rank's one timed rep, plus SLACK_NS, reaches
    floor_ns of the rep's unique bytes.  Prints each size's ns over the floor."""
    for k, s in enumerate(sizes):
        if s < FLOOR_FROM:
            continue
        floor = lt.floor_ns(lt.unique_bytes(name, n, s, op))
        slowest = max(t[k] for t in per_rank)
        print(f"FLOOR {json.dumps({'what': tag, 'n': n, 'size': s, 'ns': slowest, 'floor_ns': floor})}")
        assert slowest + SLACK_NS >= floor, (f"{card()}: {tag} n={n} size={s}: slowest rep {slowest} ns + {SLACK_NS} "
                                             f"< floor {floor:.0f} ns")


def check_floor(p, name, n, tag, op=None):
    m, _ = call(p, name, 1, op)
    got = rows(name, m)
    assert got, (tag, "nothing ran")
    for key, (lo, med, hi) in got.items():
        assert lo == med == hi, (tag, key)  # one timed rep
    margins(tag, name, n, m.sizes, [med for _, med, _ in got.values()], op or lt.OP_READ)


# ---- floor ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", PATHS)
def test_floor_n1_on_each_path(pkg, path):
    with open_bpp(pkg, 1, GIB) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        for name in ON_PATH:
            check_floor(p, name, 1, f"{name} path {path}")
        if path == 0:
            check_floor(p, "ring", 1, "ring")
            for op in OPS:
                check_floor(p, "memcpy", 1, f"memcpy op {op}", op)


@pytest.mark.parametrize("n", [1, 2, 4])
def test_floor_ce_alltoall(pkg, monkeypatch, n):
    bpp = GIB if n == 1 else 512 * MIB
    for c in ce_calls(pkg, monkeypatch, n, bpp, 1):
        per_rank = [c["ns_median"][r] for r in range(n)]
        assert all(c["ns_max"][r] == c["ns_median"][r] for r in range(n))
        margins(f"ce_alltoall op {c['op']}", "ce_alltoall", n, c["sizes"], per_rank, c["op"])


@pytest.mark.parametrize("n", [2, 4])
@pytest.mark.parametrize("name", ["allreduce", "twoshot", "ring", "push", "alltoall"])
def test_floor_ranks_sharing_a_device(pkg, name, n):
    with open_bpp(pkg, n, 512 * MIB) as p:
        check_floor(p, name, n, name)


# ---- windows fit in the call ------------------------------------------------------------------------------------------
def check_windows(name, m, wall_ms, tag, blocks=None):
    got = rows(name, m) if not isinstance(m, dict) else {r: (m["ns_min"][r], m["ns_median"][r], m["ns_max"][r])
                                                            for r in range(m["n"])}
    ms = m["ms"] if isinstance(m, dict) else m.ms
    sizes = m["sizes"] if isinstance(m, dict) else m.sizes
    assert got, (tag, "nothing ran")
    per_rank = {}
    for key, (lo, med, hi) in got.items():
        assert all(0 < a <= b <= c for a, b, c in zip(lo, med, hi)), (tag, key)
        rank = key[0] if isinstance(key, tuple) else key
        per_rank[rank] = per_rank.get(rank, 0.0) + sum(lo) + sum(med) + sum(hi)
    for rank, busy_ns in per_rank.items():
        assert busy_ns / 1e6 <= ms, f"{card()}: {tag} rank {rank}: three reps of every size {busy_ns:.0f} ns > {ms} ms"
    assert ms <= wall_ms, f"{card()}: {tag}: ms {ms} > {wall_ms} ms around the call"
    if isinstance(m, dict):
        return
    for key, (_, med, _) in got.items():
        want = (alltoall_ref.summary(sizes, med, m.blocks[key]) if name == "alltoall"
                else bwcurve_ref.summary(sizes, med))
        if CALLS[name][2]:
            i, j = key
            have = (m.t0_ns[i][j], m.peak_gbps[i][j], m.half_bytes[i][j])
        else:
            have = (m.t0_ns[key], m.peak_gbps[key], m.half_bytes[key])
        assert have == want, (tag, key)


@pytest.mark.parametrize("n", [1, 3])
def test_windows_fit_in_the_call(pkg, n):
    bpp = 64 * MIB
    with open_bpp(pkg, n, bpp) as p:
        for name in ("bwcurve", "allreduce", "twoshot", "ring", "push", "ll", "alltoall"):
            m, wall = call(p, name, 3)
            assert m.reps == 3
            check_windows(name, m, wall, f"{name} n={n}")
        for op in OPS:
            m, wall = call(p, "memcpy", 3, op)
            check_windows("memcpy", m, wall, f"memcpy op {op} n={n}")


@pytest.mark.parametrize("n", [1, 3])
def test_ce_windows_fit_in_the_call(pkg, monkeypatch, n):
    for c in ce_calls(pkg, monkeypatch, n, 64 * MIB, 3):
        check_windows("ce_alltoall", c, c["wall_ms"], f"ce_alltoall op {c['op']} n={n}")
        for r in range(n):
            assert (c["t0_ns"][r], c["peak_gbps"][r], c["half_bytes"][r]) == \
                alltoall_ref.summary(c["sizes"], c["ns_median"][r], c["blocks"][r]), (c["op"], r)


# ---- the rep spans the slowest rank -----------------------------------------------------------------------------------
def test_push_rep_spans_the_slowest_rank(pkg):
    """A push rep ends at the closing release, when every rank's all-gather is in: with one rank on a single CTA the
    other ranks' reps take as long as its own."""
    n = 3
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=1 << 20, mode=MODE_SLICED, flags=SAME, ctas=8,
                             timeout_ms=20000)) as p:
        p.SetOption(pkg.abi.OPT_CTAS_RANK, (1 << 16) | 1)
        ar = p.AllReducePush(reps=4)
        big = len(ar.sizes) - 1
        slow = ar.ns_median[0][big]
        for r in (1, 2):
            assert ar.ns_median[r][big] >= 0.5 * slow, (card(), r, ar.ns_median[r][big], slow)
