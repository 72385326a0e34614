"""cdprobe_memcpy on the GPU: every cell of every domain shape lands every word of every size, pulled and pushed, with
the (S, X) of the pattern; an armed fault fails exactly its cell and size, and the clearing check makes the next call
clean; a mapping that is down stops only its cell; MIG copies nothing; the call needs no run and disturbs none; the
times are ordered and bounded; two processes agree; and nothing leaks.  Several ranks share one device where a test
needs N > 1."""
import os
import textwrap

import pytest

import memcpy_ref as ref
from conftest import ROOT
from harness import run_children

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
LOCAL_DIAG = 0x4
SIMULATE_MIG = 0x200
MODE_REACH, MODE_SLICED, MODE_FULL = 0, 1, 2
OPS = (ref.OP_READ, ref.OP_WRITE)
ERR_ARG, ERR_UNSUPPORTED, ERR_STATE, ERR_INTEGRITY = -2, -8, -9, -10
U64_MAX = (1 << 64) - 1
GIB = 1 << 30
HBM_GBPS = 3350.0  # H100 SXM data sheet


def open_same(pkg, n, flags=0, nbytes=1 << 20, mode=MODE_SLICED):
    return pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, mode=mode, flags=SAME | flags,
                               ctas=8 if n <= 8 else 4, timeout_ms=20000))


def assert_cell_clean(mc, oracle, g, j, mode):
    c = ref.cell(mc.n, mc.sizes[-1], mode, mc.op, g, j)
    assert mc.measured[g][j] and mc.status[g][j] == 0 and mc.bad_sizes[g][j] == 0, \
        (g, j, mc.status[g][j], mc.bad_sizes[g][j])
    k = len(mc.sizes)
    assert mc.bad_words[g][j] == [0] * k and mc.first_bad[g][j] == [U64_MAX] * k, (g, j)
    assert list(zip(mc.sum[g][j], mc.xr[g][j])) == ref.expected(oracle, SEED, c, mc.sizes), (g, j)


def assert_cell_timed(mc, g, j, copied=True):
    """copied: every timed rep copied (a dropped copy leaves two events back to back, which may time as 0)."""
    for k, s in enumerate(mc.sizes):
        assert (0 < mc.ns_min[g][j][k] or not copied) and 0 <= mc.ns_min[g][j][k] <= mc.ns_median[g][j][k] <= \
            mc.ns_max[g][j][k], (g, j, s)
    assert (mc.t0_ns[g][j], mc.peak_gbps[g][j], mc.half_bytes[g][j]) == ref.summary(mc.sizes, mc.ns_median[g][j])


def assert_all_clean(mc, oracle, bpp, mode, diag):
    assert mc.sizes == ref.ladder(bpp)
    for g in range(mc.n):
        for j in range(mc.n):
            if g != j or diag:
                assert_cell_clean(mc, oracle, g, j, mode)
                assert_cell_timed(mc, g, j)
            else:
                assert not mc.measured[g][j] and mc.sum[g][j] is None
    # one rep at a time on each issuer's stream, and the issuers of one device copy at once: at least the medians of
    # the busiest issuer fit in the call
    assert max(sum(sum(mc.ns_median[g][j]) for j in range(mc.n) if mc.measured[g][j]) for g in range(mc.n)) / 1e6 \
        <= mc.ms


@pytest.mark.parametrize("op", OPS, ids=["pull", "push"])
@pytest.mark.parametrize("nbytes", [4 << 20, GIB], ids=["4MiB", "1GiB"])
def test_single_rank_loop_back_every_size_clean(pkg, oracle, nbytes, op):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, timeout_ms=20000)) as p:
        mc = p.Memcpy(op)
        assert (mc.n, mc.row_mask, mc.reps, mc.op, mc.call_seq) == (1, 1, 8, op, 1)
        assert mc.area_bytes == (nbytes + (2 << 20) - 1) // (2 << 20) * (2 << 20)
        assert_all_clean(mc, oracle, nbytes, MODE_SLICED, True)
        assert sum(mc.ns_median[0][0]) / 1e6 <= mc.ms
        if nbytes == GIB:
            # a device-local copy reads and writes every byte, so it moves at most half the HBM rate
            assert nbytes / mc.ns_median[0][0][-1] <= 1.1 * HBM_GBPS / 2, mc.ns_median[0][0][-1]
        mc2 = p.Memcpy(op, reps=3)
        assert (mc2.reps, mc2.call_seq) == (3, 2)
        assert_all_clean(mc2, oracle, nbytes, MODE_SLICED, True)


@pytest.mark.parametrize("mode", [MODE_SLICED, MODE_FULL, MODE_REACH], ids=["sliced", "full", "reach"])
@pytest.mark.parametrize("n", [2, 3, 4, 5, 8, 16])
def test_same_device_every_cell_clean(pkg, oracle, n, mode):
    nbytes = 1 << 20
    for flags in (0, LOCAL_DIAG):
        with open_same(pkg, n, flags=flags, nbytes=nbytes, mode=mode) as p:
            bpp = pkg.plan(n, nbytes, mode, flags).bytes_per_pair
            for call, op in enumerate(OPS, 1):
                mc = p.Memcpy(op, reps=2)
                assert (mc.n, mc.row_mask, mc.reps, mc.op, mc.call_seq) == (n, (1 << n) - 1, 2, op, call)
                assert_all_clean(mc, oracle, bpp, mode, bool(flags))


@pytest.mark.parametrize("op", OPS, ids=["pull", "push"])
@pytest.mark.parametrize("mode", [0, 1], ids=["flip", "drop"])
def test_an_armed_fault_fails_exactly_its_cell_and_size(pkg, oracle, mode, op):
    n, nbytes = 3, 1 << 20
    a = pkg.abi
    with open_same(pkg, n, nbytes=nbytes) as p:
        bpp = pkg.plan(n, nbytes, MODE_SLICED).bytes_per_pair
        sizes = ref.ladder(bpp)
        for (i, j, k, word) in ((2, 0, 3, sizes[3] // 8 - 5), (0, 1, len(sizes) - 1, 1234)):
            p.SetOption(a.OPT_MEMCPY_FAULT, a.memcpy_fault(i, j, k, word, mode))
            for reps in (2, 1):
                mc = p.Memcpy(op, reps=reps)
                for g in range(n):
                    for d in range(n):
                        if g == d:
                            continue
                        assert_cell_timed(mc, g, d, copied=mode == 0 or (g, d) != (i, j))
                        if (g, d) != (i, j):
                            assert_cell_clean(mc, oracle, g, d, MODE_SLICED)
                            continue
                        assert mc.status[g][d] == ERR_INTEGRITY and mc.bad_sizes[g][d] == 1 << k
                        for q in range(len(sizes)):
                            bad = (1 if mode == 0 else sizes[q] // 8) if q == k else 0
                            first = (8 * word if mode == 0 else 0) if q == k else U64_MAX
                            assert (mc.bad_words[g][d][q], mc.first_bad[g][d][q]) == (bad, first), (reps, q)
                            if q != k or reps > 1:  # the fault is in timed rep 1; the folded rep is the last
                                c = ref.cell(n, bpp, MODE_SLICED, op, g, d)
                                assert (mc.sum[g][d][q], mc.xr[g][d][q]) == ref.expected(oracle, SEED, c, [sizes[q]])[0]
            # disarmed, the very next call is clean: the check cleared what the faulty rep left
            p.SetOption(a.OPT_MEMCPY_FAULT, 0)
            assert_all_clean(p.Memcpy(op, reps=1), oracle, bpp, MODE_SLICED, False)
        # arming that names no cell, size or word of the call, or a mode above 1, is refused and changes nothing
        seq = p.Memcpy(op, reps=1).call_seq
        for bad in (a.memcpy_fault(n, 0, 0, 0), a.memcpy_fault(1, 1, 0, 0), a.memcpy_fault(0, 1, len(sizes), 0),
                    a.memcpy_fault(0, 1, 0, sizes[0] // 8), (2 << 48) | (1 << 40) | (2 << 32) | (1 << 24),
                    (1 << 40) | (1 << 24), (1 << 63) | (1 << 40) | (2 << 32) | (1 << 24)):
            p.SetOption(a.OPT_MEMCPY_FAULT, bad)
            rc, t = p.memcpy_raw(op, 2)
            assert rc == ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0
            assert (t.abi, t.n, t.reps, t.op) == (2, n, 2, op)
        p.SetOption(a.OPT_MEMCPY_FAULT, 0)
        mc = p.Memcpy(op, reps=2)
        assert mc.call_seq == seq + 1
        assert_all_clean(mc, oracle, bpp, MODE_SLICED, False)


@pytest.mark.parametrize("op", OPS, ids=["pull", "push"])
def test_a_mapping_that_is_down_stops_only_its_cell(pkg, oracle, op):
    n, nbytes = 4, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        bpp = pkg.plan(n, nbytes, MODE_SLICED).bytes_per_pair
        assert_all_clean(p.Memcpy(op, reps=2), oracle, bpp, MODE_SLICED, False)  # the area exists before the unmap
        p.UnmapPeer(2, 1)
        mc = p.Memcpy(op, reps=2)
        for g in range(n):
            for d in range(n):
                if g == d:
                    continue
                if (g, d) == (2, 1):
                    assert not mc.measured[g][d] and mc.status[g][d] == ERR_STATE
                    assert mc.sum[g][d] is None and mc.raw.sum[g * 16 + d][0] == 0
                else:
                    assert_cell_clean(mc, oracle, g, d, MODE_SLICED)
        p.RemapPeer(2, 1)
        assert_all_clean(p.Memcpy(op, reps=2), oracle, bpp, MODE_SLICED, False)


def test_simulated_mig_copies_nothing(pkg):
    n = 2
    with open_same(pkg, n, flags=SIMULATE_MIG) as p:
        for call, op in enumerate(OPS, 1):
            mc = p.Memcpy(op, reps=2)
            assert mc.call_seq == call and mc.ms < 5000
            for g in range(n):
                for d in range(n):
                    assert not mc.measured[g][d] and mc.ns_median[g][d] is None
            assert mc.status[0][1] == ERR_UNSUPPORTED and mc.status[1][0] == ERR_UNSUPPORTED


def test_argument_errors_fill_the_output(pkg, oracle):
    a = pkg.abi
    with open_same(pkg, 2) as p:
        for op, reps in ((0, 0), (3, 2), (a.OP_READ | a.OP_WRITE, 1), (a.OP_READ, a.MEMCPY_MAX_REPS + 1)):
            rc, t = p.memcpy_raw(op, reps)
            assert rc == ERR_ARG and (t.abi, t.n, t.reps, t.op, t.call_seq, t.row_mask, t.n_sizes) == \
                (2, 2, reps or 8, op, 0, 0, 0)
            assert sum(t.measured) == 0
        with pytest.raises(pkg.ProbeError):
            p.Memcpy(a.OP_WRITE, 1 << 31)
        mc = p.Memcpy(a.OP_WRITE, reps=a.MEMCPY_MAX_REPS)  # the handle stays usable
        assert mc.call_seq == 1
        assert_all_clean(mc, oracle, 1 << 20, MODE_SLICED, False)


def test_callable_before_the_first_run_and_disturbs_nothing(pkg, oracle):
    n, nbytes = 2, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        assert_all_clean(p.Memcpy(ref.OP_READ, reps=2), oracle, nbytes, MODE_SLICED, False)
        r1 = p.Run()
        assert r1.reach == [[1] * n for _ in range(n)] and not r1.aborted
        diags = {(op, i, j): p.Diagnose(op, i, j) for i, j in ((0, 1), (1, 0)) for op in ("read", "write")}
        for op in OPS:
            assert_all_clean(p.Memcpy(op, reps=2), oracle, nbytes, MODE_SLICED, False)
        for key, d in diags.items():
            d2 = p.Diagnose(*key)
            assert (d2.bad_words, d2.run_seq, d2.region_offset, d2.kinds) == \
                (d.bad_words, d.run_seq, d.region_offset, d.kinds), key
            assert d2.bad_words == 0 and d2.run_seq == r1.run_seq
        # the all-to-all shares the exchange area: each is clean after the other, over the same area
        aa = p.AllToAll(reps=2)
        assert all(aa.cell_status[s][d] == 0 and aa.bad_sizes[s][d] == 0 for s in range(n) for d in range(n) if s != d)
        mc = p.Memcpy(ref.OP_WRITE, reps=2)
        assert mc.area_bytes == aa.area_bytes
        assert_all_clean(mc, oracle, nbytes, MODE_SLICED, False)
        aa2 = p.AllToAll(reps=2)
        assert all(aa2.cell_status[s][d] == 0 and aa2.bad_sizes[s][d] == 0 for s in range(n) for d in range(n) if s != d)
        r2 = p.Run()
        assert r2.run_seq == r1.run_seq + 1 and r2.reach == r1.reach and not r2.aborted
        assert (r2.sum_read, r2.xor_read) == (r1.sum_read, r1.xor_read)
        words = r2.bytes_per_pair // 8
        for i, j in ((0, 1), (1, 0)):
            assert (r2.sum_write[i][j], r2.xor_write[i][j]) == oracle.write_checksum(SEED, i, j, r2.run_seq, words)


def test_alltoall_first_then_memcpy(pkg, oracle):
    n, nbytes = 3, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        aa = p.AllToAll(reps=2)
        bpp = pkg.plan(n, nbytes, MODE_SLICED).bytes_per_pair
        for op in OPS:
            mc = p.Memcpy(op, reps=2)
            assert mc.area_bytes == aa.area_bytes
            assert_all_clean(mc, oracle, bpp, MODE_SLICED, False)


def test_no_leak(pkg):
    import torch
    nbytes = 64 << 20
    torch.cuda.init()
    free0 = torch.cuda.mem_get_info(0)[0]
    fds0 = len(os.listdir("/proc/self/fd"))
    for _ in range(3):
        with open_same(pkg, 2, nbytes=nbytes) as p:
            p.Memcpy(ref.OP_READ, reps=1)
            free1 = torch.cuda.mem_get_info(0)[0]
            p.Memcpy(ref.OP_WRITE, reps=1)
            assert torch.cuda.mem_get_info(0)[0] == free1
        assert torch.cuda.mem_get_info(0)[0] == free0
    assert len(os.listdir("/proc/self/fd")) == fds0


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world, n_local = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
    flags = 0x40 | (0x10 if n_local > 1 else 0)
    cfg = m.Config(ordinals=[0] * n_local, bytes=1 << 20, world_size=world, rank=rank, session=session, flags=flags,
                   ctas=8, timeout_ms=30000)

    def dump(mc):
        return {k: getattr(mc, k) for k in ("row_mask", "measured", "status", "bad_words", "first_bad", "sum", "xr",
                                            "ns_min", "sizes", "call_seq", "reps", "op", "bad_sizes")}

    with m.Open(cfg) as p:
        out = {"calls": [dump(p.Memcpy(m.abi.OP_READ, reps=2)), dump(p.Memcpy(m.abi.OP_WRITE, reps=3))]}
        rc, t = p.memcpy_raw(m.abi.OP_READ, 2 + rank)  # the processes disagree
        out["mismatch"] = {"rc": rc, "call_seq": t.call_seq, "measured": sum(t.measured)}
        r = p.Run(gather=True)
        out["run"] = {"reach": r.reach, "aborted": r.aborted}
    print("RESULT " + json.dumps(out))
    """
) % ROOT


@pytest.mark.parametrize("n_local", [1, 2], ids=["2x1", "2x2"])
def test_two_processes_agree_and_fill_their_own_rows(pkg, oracle, n_local):
    world = 2
    n = world * n_local
    outs = run_children(CHILD, world, n_local)
    bpp = pkg.plan(n, 1 << 20, MODE_SLICED).bytes_per_pair
    sizes = ref.ladder(bpp)
    for rank, o in enumerate(outs):
        mine = set(range(rank * n_local, (rank + 1) * n_local))
        assert [c["call_seq"] for c in o["calls"]] == [1, 2]
        assert o["mismatch"] == {"rc": ERR_ARG, "call_seq": 0, "measured": 0}
        for c in o["calls"]:
            assert c["row_mask"] == sum(1 << r for r in mine) and c["sizes"] == sizes
            for g in range(n):
                for d in range(n):
                    if g == d:
                        continue
                    assert c["measured"][g][d] == (g in mine), (g, d)
                    if g not in mine:
                        assert c["sum"][g][d] is None
                        continue
                    cell = ref.cell(n, bpp, MODE_SLICED, c["op"], g, d)
                    assert c["status"][g][d] == 0 and c["bad_words"][g][d] == [0] * len(sizes)
                    assert all(t > 0 for t in c["ns_min"][g][d])
                    assert [[x, y] for x, y in zip(c["sum"][g][d], c["xr"][g][d])] == \
                        [list(e) for e in ref.expected(oracle, SEED, cell, sizes)]
        assert o["run"]["reach"] == [[1] * n for _ in range(n)] and not o["run"]["aborted"]
