"""cdprobe_alltoall on the GPU: every cell of every domain shape delivers every word of every size, with the (S, X) of
the pattern; an armed fault fails exactly its cell and size, also across processes; a mapping that is down stops only
its cell; MIG launches nothing; the call needs no run and disturbs none; the times are ordered and bounded; and the
exchange area leaks nothing.  Several ranks share one device where a test needs N > 1, with CTA counts that let their
grids be resident together (every rank waits for its peers at each rep)."""
import textwrap

import pytest

import alltoall_ref as ref
from conftest import ROOT
from harness import run_children

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
LOCAL_DIAG = 0x4
SIMULATE_MIG = 0x200
MODE_REACH, MODE_SLICED, MODE_FULL = 0, 1, 2
ERR_ARG, ERR_UNSUPPORTED, ERR_STATE, ERR_INTEGRITY = -2, -8, -9, -10
U64_MAX = (1 << 64) - 1
GIB = 1 << 30
REF_MAX = 64 << 20  # blocks up to this get their (S, X) from the numpy reference; larger ones from the oracle


def open_same(pkg, n, flags=0, nbytes=1 << 20, mode=MODE_SLICED):
    return pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, mode=mode, flags=SAME | flags,
                               ctas=8 if n <= 8 else 4, timeout_ms=20000))


def want(oracle, i, j, aa):
    out = []
    for k, s in enumerate(aa.sizes):
        seq = ref.alltoall_seq(aa.call_seq, k, aa.reps)
        out.append(ref.checksum(ref.block_words(SEED, i, j, aa.call_seq, k, aa.reps, s // 8)) if s <= REF_MAX
                   else oracle.write_checksum(SEED, i, j, seq, s // 8))
    return out


def assert_cell_clean(aa, oracle, i, j):
    assert aa.cell_measured[i][j] and aa.cell_status[i][j] == 0 and aa.bad_sizes[i][j] == 0, \
        (i, j, aa.cell_status[i][j], aa.bad_sizes[i][j])
    assert aa.bad_words[i][j] == [0] * len(aa.sizes) and aa.first_bad[i][j] == [U64_MAX] * len(aa.sizes), (i, j)
    assert [(s, x) for s, x in zip(aa.sum[i][j], aa.xr[i][j])] == want(oracle, i, j, aa), (i, j)


def assert_rank_timed(aa, r):
    assert aa.measured[r] and aa.status[r] == 0, (r, aa.status[r])
    for k, s in enumerate(aa.sizes):
        assert 0 < aa.ns_min[r][k] <= aa.ns_median[r][k] <= aa.ns_max[r][k], (r, s)
    assert (aa.t0_ns[r], aa.peak_gbps[r], aa.half_bytes[r]) == ref.summary(aa.sizes, aa.ns_median[r], aa.blocks[r])
    busy = sum(aa.reps * t for t in aa.ns_min[r])  # a rank's timed reps run one after another inside the call
    assert busy / 1e6 <= aa.ms, (r, busy, aa.ms)


def assert_all_clean(aa, oracle, bpp, diag):
    assert aa.sizes == ref.ladder(bpp)
    for i in range(aa.n):
        assert_rank_timed(aa, i)
        assert aa.blocks[i] == aa.n - 1 + (1 if diag else 0), i
        for j in range(aa.n):
            if i != j or diag:
                assert_cell_clean(aa, oracle, i, j)
            else:
                assert not aa.cell_measured[i][j]


@pytest.mark.parametrize("path", [0, 1, 2], ids=["tma", "ldst16", "ldst32"])
@pytest.mark.parametrize("nbytes", [4 << 20, GIB], ids=["4MiB", "1GiB"])
def test_single_rank_every_size_clean(pkg, oracle, nbytes, path):
    """At N = 1 the one block is the loop-back block: a write curve of local HBM."""
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, timeout_ms=20000)) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        aa = p.AllToAll()
        assert (aa.n, aa.row_mask, aa.reps, aa.path, aa.call_seq) == (1, 1, 8, path, 1)
        assert aa.area_bytes == (nbytes + (2 << 20) - 1) // (2 << 20) * (2 << 20)
        assert_all_clean(aa, oracle, nbytes, True)
        aa2 = p.AllToAll(reps=3)
        assert (aa2.reps, aa2.call_seq) == (3, 2)
        assert_all_clean(aa2, oracle, nbytes, True)


@pytest.mark.parametrize("mode", [MODE_SLICED, MODE_FULL, MODE_REACH], ids=["sliced", "full", "reach"])
@pytest.mark.parametrize("n", [2, 3, 4, 5, 8, 16])
def test_same_device_every_cell_clean(pkg, oracle, n, mode):
    nbytes = 1 << 20
    with open_same(pkg, n, nbytes=nbytes, mode=mode) as p:
        bpp = pkg.plan(n, nbytes, mode).bytes_per_pair
        aa = p.AllToAll(reps=2)
        assert (aa.n, aa.row_mask, aa.reps, aa.call_seq) == (n, (1 << n) - 1, 2, 1)
        assert_all_clean(aa, oracle, bpp, False)
        assert p.AllToAll(reps=1).call_seq == 2


@pytest.mark.parametrize("n", [1, 3])
def test_local_diag_adds_the_diagonal_block(pkg, oracle, n):
    with open_same(pkg, n, flags=LOCAL_DIAG) as p:
        bpp = pkg.plan(n, 1 << 20, MODE_SLICED, LOCAL_DIAG).bytes_per_pair
        assert_all_clean(p.AllToAll(reps=2), oracle, bpp, True)


@pytest.mark.parametrize("path", [0, 1, 2], ids=["tma", "ldst16", "ldst32"])
def test_an_armed_fault_fails_exactly_its_cell_and_size(pkg, oracle, path):
    n, nbytes = 3, 1 << 20
    a = pkg.abi
    with open_same(pkg, n, nbytes=nbytes) as p:
        p.SetOption(a.OPT_PATH, path)
        bpp = pkg.plan(n, nbytes, MODE_SLICED).bytes_per_pair
        sizes = ref.ladder(bpp)
        for (i, j, k, word) in ((2, 0, 3, sizes[3] // 8 - 5), (0, 1, len(sizes) - 1, 1234)):
            p.SetOption(a.OPT_ALLTOALL_FAULT, a.alltoall_fault(i, j, k, word))
            for reps in (2, 1):
                aa = p.AllToAll(reps=reps)
                for s in range(n):
                    assert_rank_timed(aa, s)
                    for d in range(n):
                        if s == d:
                            continue
                        if (s, d) != (i, j):
                            assert_cell_clean(aa, oracle, s, d)
                            continue
                        assert aa.cell_status[s][d] == ERR_INTEGRITY and aa.bad_sizes[s][d] == 1 << k
                        for q in range(len(sizes)):
                            assert aa.bad_words[s][d][q] == (1 if q == k else 0), (reps, q)
                            assert aa.first_bad[s][d][q] == (8 * word if q == k else U64_MAX), (reps, q)
                            if q != k or reps > 1:  # the fault is in timed rep 1; the folded rep is the last
                                assert (aa.sum[s][d][q], aa.xr[s][d][q]) == want(oracle, s, d, aa)[q]
        # arming that names no cell, size or word of the call is refused, and refusing changes nothing
        seq = aa.call_seq
        for bad in (a.alltoall_fault(n, 0, 0, 0), a.alltoall_fault(1, 1, 0, 0), a.alltoall_fault(0, 1, len(sizes), 0),
                    a.alltoall_fault(0, 1, 0, sizes[0] // 8), (1 << 32) | (1 << 24), (1 << 40) | (1 << 24)):
            p.SetOption(a.OPT_ALLTOALL_FAULT, bad)
            rc, t = p.alltoall_raw(2)
            assert rc == ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0 and (t.abi, t.n, t.reps) == (2, n, 2)
        p.SetOption(a.OPT_ALLTOALL_FAULT, 0)
        aa = p.AllToAll(reps=2)
        assert aa.call_seq == seq + 1
        assert_all_clean(aa, oracle, bpp, False)


def test_a_mapping_that_is_down_stops_only_its_cell(pkg, oracle):
    n, nbytes = 4, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        bpp = pkg.plan(n, nbytes, MODE_SLICED).bytes_per_pair
        assert_all_clean(p.AllToAll(reps=2), oracle, bpp, False)  # the area exists before the unmap
        p.UnmapPeer(2, 1)
        aa = p.AllToAll(reps=2)
        for s in range(n):
            assert_rank_timed(aa, s)
            assert aa.blocks[s] == (n - 2 if s == 2 else n - 1)
            for d in range(n):
                if s == d:
                    continue
                if (s, d) == (2, 1):
                    assert not aa.cell_measured[s][d] and aa.cell_status[s][d] == ERR_STATE
                    assert aa.sum[s][d] is None and aa.raw.sum[s * 16 + d][0] == 0
                else:
                    assert_cell_clean(aa, oracle, s, d)
        p.RemapPeer(2, 1)
        assert_all_clean(p.AllToAll(reps=2), oracle, bpp, False)


def test_unmapped_before_the_area_exists(pkg, oracle):
    n = 3
    with open_same(pkg, n) as p:
        p.UnmapPeer(0, 2)
        aa = p.AllToAll(reps=2)
        assert not aa.cell_measured[0][2] and aa.cell_status[0][2] == ERR_STATE
        assert_cell_clean(aa, oracle, 2, 0)
        assert_cell_clean(aa, oracle, 1, 2)


def test_simulated_mig_launches_nothing(pkg):
    n = 2
    with open_same(pkg, n, flags=SIMULATE_MIG) as p:
        aa = p.AllToAll(reps=2)
        assert aa.call_seq == 1 and aa.ms < 5000
        for r in range(n):
            assert not aa.measured[r] and aa.ns_median[r] is None
        assert not aa.cell_measured[0][1] and aa.cell_status[0][1] == ERR_UNSUPPORTED
        assert aa.cell_status[1][0] == ERR_UNSUPPORTED


def test_argument_errors_fill_the_output(pkg, oracle):
    a = pkg.abi
    with open_same(pkg, 2) as p:
        rc, t = p.alltoall_raw(a.ALLTOALL_MAX_REPS + 1)
        assert rc == ERR_ARG and (t.abi, t.n, t.reps, t.call_seq, t.row_mask, t.n_sizes) == (2, 2, 65, 0, 0, 0)
        assert sum(t.measured) == 0 and sum(t.cell_measured) == 0
        with pytest.raises(pkg.ProbeError):
            p.AllToAll(1 << 31)
        aa = p.AllToAll(reps=a.ALLTOALL_MAX_REPS)  # the handle stays usable
        assert aa.call_seq == 1
        assert_all_clean(aa, oracle, 1 << 20, False)


def test_callable_before_the_first_run_and_disturbs_nothing(pkg, oracle):
    n, nbytes = 2, 1 << 20
    a = pkg.abi
    with open_same(pkg, n, nbytes=nbytes) as p:
        assert_all_clean(p.AllToAll(reps=2), oracle, nbytes, False)
        r1 = p.Run()
        assert r1.reach == [[1] * n for _ in range(n)] and not r1.aborted
        diags = {(op, i, j): p.Diagnose(op, i, j) for i, j in ((0, 1), (1, 0)) for op in ("read", "write")}
        pp = p.PingPong(trips=64, reps=2)
        at = p.Atomics(a.ATOMIC_FETCH_ADD, ops=64, reps=2)
        bw = p.BwCurve(reps=2)
        ar = p.AllReduce(reps=2)
        aa = p.AllToAll(reps=2)
        assert aa.call_seq == 2
        assert_all_clean(aa, oracle, nbytes, False)
        for key, d in diags.items():
            d2 = p.Diagnose(*key)
            assert (d2.bad_words, d2.run_seq, d2.region_offset, d2.kinds) == \
                (d.bad_words, d.run_seq, d.region_offset, d.kinds), key
            assert d2.bad_words == 0 and d2.run_seq == r1.run_seq
        assert p.BwCurve(reps=2).call_seq == bw.call_seq + 1
        assert p.AllReduce(reps=2).call_seq == ar.call_seq + 1
        assert p.PingPong(trips=64, reps=2).call_seq == pp.call_seq + 1
        assert p.Atomics(a.ATOMIC_FETCH_ADD, ops=64, reps=2).call_seq == at.call_seq + 1
        r2 = p.Run()
        assert r2.run_seq == r1.run_seq + 1 and r2.reach == r1.reach and not r2.aborted
        assert (r2.sum_read, r2.xor_read) == (r1.sum_read, r1.xor_read)
        words = r2.bytes_per_pair // 8
        for i, j in ((0, 1), (1, 0)):
            assert (r2.sum_write[i][j], r2.xor_write[i][j]) == oracle.write_checksum(SEED, i, j, r2.run_seq, words)


def test_no_leak(pkg):
    import torch
    nbytes = 64 << 20
    torch.cuda.init()
    free0 = torch.cuda.mem_get_info(0)[0]
    with open_same(pkg, 2, nbytes=nbytes) as p:
        p.AllToAll(reps=1)
        free1 = torch.cuda.mem_get_info(0)[0]
        p.AllToAll(reps=1)
        assert torch.cuda.mem_get_info(0)[0] == free1
    assert torch.cuda.mem_get_info(0)[0] == free0


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world, n_local, fault = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), sys.argv[5]
    flags = 0x40 | (0x10 if n_local > 1 else 0)
    cfg = m.Config(ordinals=[0] * n_local, bytes=1 << 20, world_size=world, rank=rank, session=session, flags=flags,
                   ctas=8, timeout_ms=30000)

    def dump(aa):
        return {k: getattr(aa, k) for k in ("row_mask", "measured", "status", "blocks", "cell_measured", "cell_status",
                                            "bad_words", "first_bad", "sum", "xr", "ns_min", "sizes", "call_seq",
                                            "reps", "bad_sizes")}

    with m.Open(cfg) as p:
        if fault != "none":
            p.SetOption(m.abi.OPT_ALLTOALL_FAULT, int(fault))
        out = {"calls": [dump(p.AllToAll(reps=2)), dump(p.AllToAll(reps=3))]}
        rc, t = p.alltoall_raw(2 + rank)  # the processes disagree
        out["mismatch"] = {"rc": rc, "call_seq": t.call_seq, "measured": sum(t.measured)}
        r = p.Run(gather=True)
        out["run"] = {"reach": r.reach, "aborted": r.aborted}
    print("RESULT " + json.dumps(out))
    """
) % ROOT


@pytest.mark.parametrize("n_local", [1, 2], ids=["2x1", "2x2"])
def test_two_processes_agree_and_fill_their_own_entries(pkg, oracle, n_local):
    """Both processes drive GPU 0.  With two ranks per process, a fault is armed on a cell from process 0's second rank
    to process 1's first, so the sender and the receiver are in different processes."""
    world = 2
    n = world * n_local
    fi, fj, fk, fw = (1, 2, 2, 77) if n_local == 2 else (0, 1, 2, 77)
    outs = run_children(CHILD, world, n_local, pkg.abi.alltoall_fault(fi, fj, fk, fw))
    sizes = ref.ladder(pkg.plan(n, 1 << 20, MODE_SLICED).bytes_per_pair)
    for rank, o in enumerate(outs):
        mine = set(range(rank * n_local, (rank + 1) * n_local))
        assert [c["call_seq"] for c in o["calls"]] == [1, 2]
        assert o["mismatch"] == {"rc": ERR_ARG, "call_seq": 0, "measured": 0}
        for c in o["calls"]:
            assert c["row_mask"] == sum(1 << r for r in mine) and c["sizes"] == sizes
            for r in range(n):
                assert c["measured"][r] == (r in mine), r
                if r in mine:
                    assert c["status"][r] == 0 and c["blocks"][r] == n - 1 and all(t > 0 for t in c["ns_min"][r])
            for s in range(n):
                for d in range(n):
                    if s == d:
                        continue
                    assert c["cell_measured"][s][d] == (d in mine), (s, d)
                    if d not in mine:
                        assert c["sum"][s][d] is None
                        continue
                    expect = ref.expected(SEED, s, d, c["call_seq"], c["reps"], sizes)
                    if (s, d) == (fi, fj):
                        assert c["cell_status"][s][d] == ERR_INTEGRITY and c["bad_sizes"][s][d] == 1 << fk
                        assert c["bad_words"][s][d] == [1 if q == fk else 0 for q in range(len(sizes))]
                        assert c["first_bad"][s][d][fk] == 8 * fw
                    else:
                        assert c["cell_status"][s][d] == 0 and c["bad_words"][s][d] == [0] * len(sizes)
                        assert [[x, y] for x, y in zip(c["sum"][s][d], c["xr"][s][d])] == [list(e) for e in expect]
        assert o["run"]["reach"] == [[1] * n for _ in range(n)] and not o["run"]["aborted"]
