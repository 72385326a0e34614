"""cdprobe_allreduce_twoshot on the GPU: every row's output at every size is the pattern's sum, word for word and in
(S, X), and equals the one-shot's on the same handle; tiny ladders where some ranks own no unit, and small or unequal
grids; a word corrupted at rest fails exactly the sizes that cover it in every row; an armed fault fails only its
receiver's row and size, and a dropped unit reads as 0s (the per-rep clear); a mapping that is down stops every rank
without waiting; two processes agree; the call needs no run and disturbs none; the times are ordered and bounded.
Several ranks share one device where a test needs N > 1, with CTA counts that let their grids be resident together
(every rank waits for every other at each rep).  No test drives a kernel past its deadline."""
import functools
import textwrap

import numpy as np
import pytest

import allreduce_ref
import allreduce_twoshot_ref as ref
import word_ref
from conftest import ROOT
from harness import run_children
from test_allreduce_gpu import assert_hbm_floor

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
SIMULATE_MIG = 0x200
MODE_REACH, MODE_SLICED, MODE_FULL = 0, 1, 2
ERR_ARG, ERR_UNSUPPORTED, ERR_STATE, ERR_INTEGRITY = -2, -8, -9, -10
U64_MAX = word_ref.U64_MAX
GIB = 1 << 30
REF_MAX = 64 << 20  # sizes up to this get their (S, X) from the numpy reference; larger ones (N = 1) from the oracle
PATHS = (0, 1, 2)   # TMA, 16-byte ld/st, 32-byte ld/st
EDGE_BPP = 57 * 8192 + 384  # a partial last unit in a partial last granule: ladder 4096 ... 262144, 467328


def open_same(pkg, n, flags=0, nbytes=1 << 20, mode=MODE_SLICED, ctas=None):
    return pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, mode=mode, flags=(SAME if n > 1 else 0) | flags,
                               ctas=ctas or (8 if n <= 8 else 4), timeout_ms=20000))


def open_bpp(pkg, n, bpp):
    """A handle whose bytes_per_pair is bpp (sliced mode: bytes / peers)."""
    p = open_same(pkg, n, nbytes=bpp * max(n - 1, 1), ctas=8)
    assert p.Info().bytes_per_pair == bpp
    return p


@functools.lru_cache(maxsize=None)
def src(rank, n_words):
    w = word_ref.src_words(SEED, rank, 0, n_words)
    w.setflags(write=False)
    return w


def check(ar, n, bpp, reps, corrupt=None, fault=None):
    """Every row at every size, from the words at rest: corrupt {(rank, word): mask} is xored into the sources, and
    fault (receiver, k, word, drop) acts in timed rep 1 only.  bad_words count every rep, warm-up included; (S, X) is
    the last timed rep's."""
    corrupt = corrupt or {}
    sizes = allreduce_ref.ladder(bpp)
    assert ar.sizes == sizes and ar.reps == reps and ar.n == n
    W = bpp // 8
    clean = sum(src(j, W) for j in range(n))
    at_rest = clean.copy()
    for (j, w), m in corrupt.items():
        orig = int(src(j, W)[w])
        at_rest[w] = np.uint64((int(at_rest[w]) - orig + (orig ^ m)) % (1 << 64))
    for r in range(n):
        bits = 0
        for k, s in enumerate(sizes):
            rep_words = at_rest[:s // 8].copy()  # what every rep but the faulted one reads back
            bad = np.flatnonzero(rep_words != clean[:s // 8])
            n_bad, first = (reps + 1) * len(bad), [int(bad[0])] if len(bad) else []
            last = rep_words
            if fault is not None and (r, k) == fault[:2]:
                hit = rep_words.copy()
                u0 = fault[2] // ref.UNIT_WORDS * ref.UNIT_WORDS
                if fault[3]:
                    hit[u0:u0 + ref.unit_words(s, fault[2])] = 0
                else:
                    hit[fault[2]] ^= np.uint64(1)
                hbad = np.flatnonzero(hit != clean[:s // 8])
                n_bad += len(hbad) - len(bad)
                first += [int(hbad[0])] if len(hbad) else []
                bits |= 1 << k
                if reps == 1:
                    last = hit
            if len(bad):
                bits |= 1 << k
            ctx = (r, s, fault)
            assert (ar.sum[r][k], ar.xr[r][k]) == allreduce_ref.checksum(last), ctx
            assert ar.bad_words[r][k] == n_bad, (ctx, ar.bad_words[r][k], n_bad)
            assert ar.first_bad[r][k] == (8 * min(first) if first else U64_MAX), (ctx, ar.first_bad[r][k])
            assert 0 < ar.ns_min[r][k] <= ar.ns_median[r][k] <= ar.ns_max[r][k], ctx
        assert ar.measured[r] and ar.bad_sizes[r] == bits, (r, ar.bad_sizes[r], bits)
        assert ar.status[r] == (ERR_INTEGRITY if bits else 0), r
        assert (ar.t0_ns[r], ar.peak_gbps[r], ar.half_bytes[r]) == allreduce_ref.summary(sizes, ar.ns_median[r])
    assert_fits_in_call(ar)
    return ar


def want(oracle, n, sizes):
    small = tuple(s for s in sizes if s <= REF_MAX)
    got = dict(zip(small, allreduce_ref.expected(SEED, n, small))) if small else {}
    for s in sizes:
        if s not in got:
            assert n == 1, "only the single-rank output is checked against the oracle beyond REF_MAX"
            got[s] = oracle.src_checksum(SEED, 0, 0, s // 8)
    return [got[s] for s in sizes]


def assert_fits_in_call(ar):
    """A rank's timed reps run one after another inside the call, so their least times must fit its wall clock."""
    for r in range(ar.n):
        if ar.ns_min[r]:
            assert sum(ar.reps * t for t in ar.ns_min[r]) / 1e6 <= ar.ms, r
            assert max(ar.ns_median[r]) / 1e6 <= ar.ms


def assert_all_clean(ar, oracle, bpp):
    assert ar.sizes == allreduce_ref.ladder(bpp)
    expect = want(oracle, ar.n, ar.sizes)
    for r in range(ar.n):
        assert ar.measured[r] and ar.status[r] == 0 and ar.bad_sizes[r] == 0, (r, ar.status[r], ar.bad_sizes[r])
        assert [(s, x) for s, x in zip(ar.sum[r], ar.xr[r])] == expect, r
        assert ar.bad_words[r] == [0] * len(ar.sizes) and ar.first_bad[r] == [U64_MAX] * len(ar.sizes), r
        for k in range(len(ar.sizes)):
            assert 0 < ar.ns_min[r][k] <= ar.ns_median[r][k] <= ar.ns_max[r][k], (r, k)
        assert (ar.t0_ns[r], ar.peak_gbps[r], ar.half_bytes[r]) == allreduce_ref.summary(ar.sizes, ar.ns_median[r])
    assert_fits_in_call(ar)


@pytest.mark.parametrize("path", PATHS, ids=["tma", "ldst16", "ldst32"])
@pytest.mark.parametrize("nbytes", [4 << 20, GIB], ids=["4MiB", "1GiB"])
def test_single_rank_every_size_clean(pkg, oracle, nbytes, path):
    """At N = 1 the rank owns every unit and its output is a copy of its own prefix: a 1 GiB rep reads 1 GiB and
    stores 1 GiB through HBM, so it takes no less than 2 GiB need at the data sheet's bandwidth."""
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, timeout_ms=20000)) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        ar = p.AllReduceTwoShot()
        assert (ar.n, ar.row_mask, ar.reps, ar.path, ar.call_seq) == (1, 1, 8, path, 1)
        assert_all_clean(ar, oracle, nbytes)
        ar2 = p.AllReduceTwoShot(reps=3)
        assert (ar2.reps, ar2.call_seq) == (3, 2)
        assert_all_clean(ar2, oracle, nbytes)
        if nbytes == GIB:
            for r in (ar, ar2):
                assert_hbm_floor(r, 2 * GIB)


@pytest.mark.parametrize("mode", [MODE_SLICED, MODE_FULL, MODE_REACH], ids=["sliced", "full", "reach"])
@pytest.mark.parametrize("n", [2, 3, 4, 5, 8, 16])
def test_same_device_every_row_clean_and_equal_to_the_one_shot(pkg, oracle, n, mode):
    with open_same(pkg, n, mode=mode) as p:
        bpp = pkg.plan(n, 1 << 20, mode).bytes_per_pair
        for path in PATHS:
            p.SetOption(pkg.abi.OPT_PATH, path)
            ts = p.AllReduceTwoShot(reps=2)
            assert (ts.n, ts.row_mask, ts.reps, ts.path, ts.call_seq) == (n, (1 << n) - 1, 2, path, path + 1)
            assert_all_clean(ts, oracle, bpp)
            one = p.AllReduce(reps=2)
            assert one.call_seq == path + 1
            assert (ts.sum, ts.xr, ts.status) == (one.sum, one.xr, one.status)


@pytest.mark.parametrize("bpp", [128, 4224, 16512, 24704])
@pytest.mark.parametrize("n", [3, 5])
def test_tiny_ladders_where_ranks_own_no_unit(pkg, n, bpp):
    """From 128 bytes: the smallest sizes have fewer units than ranks, so some ranks reduce nothing and still join
    every barrier; a partial unit is a 128-byte TMA copy or 4 of 32 lanes on the 32-byte path."""
    with open_bpp(pkg, n, bpp) as p:
        assert ref.units(allreduce_ref.ladder(bpp)[0]) < n
        for path in PATHS:
            p.SetOption(pkg.abi.OPT_PATH, path)
            check(p.AllReduceTwoShot(reps=1), n, bpp, 1)
            check(p.AllReduceTwoShot(reps=2), n, bpp, 2)


GRIDS = [("ctas", 1), ("ctas", 2), ("ctas", 3), ("ctas", 7), ("rank", (1, 8, 3))]


@pytest.mark.parametrize("grid", GRIDS, ids=[f"{g[0]}{'-'.join(map(str, g[1])) if g[0] == 'rank' else g[1]}"
                                             for g in GRIDS])
def test_grids_and_faults_at_the_edges(pkg, grid):
    """On every path: an XOR fault whose receiver is the rank that reduces the word, one on the last word of the last,
    partial unit (in the last rank's chunk), a dropped unit, and a clean call between them."""
    a = pkg.abi
    n, bpp = 3, EDGE_BPP
    sizes = allreduce_ref.ladder(bpp)
    last, W = len(sizes) - 1, bpp // 8
    with open_bpp(pkg, n, bpp) as p:
        if grid[0] == "ctas":
            p.SetOption(a.OPT_CTAS, grid[1])
        else:
            for li, c in enumerate(grid[1]):
                p.SetOption(a.OPT_CTAS_RANK, ((li + 1) << 16) | c)
        info = p.Info()
        assert [info.ctas[li] for li in range(n)] == (list(grid[1]) if grid[0] == "rank" else [grid[1]] * n)
        mid = 5 * 1024 + 77
        faults = [(ref.owner(sizes[4], n, mid), 4, mid, False),  # receiver == reducer
                  (0, last, W - 1, False),                          # the last rank's partial last unit
                  (1, last - 1, mid, True)]                         # a dropped unit
        assert ref.owner(sizes[last], n, W - 1) == n - 1 and faults[2][0] != ref.owner(sizes[last - 1], n, mid)
        for path in PATHS:
            p.SetOption(a.OPT_PATH, path)
            check(p.AllReduceTwoShot(reps=1), n, bpp, 1)
            for f in faults:
                p.SetOption(a.OPT_ALLREDUCE_TWOSHOT_FAULT, a.allreduce_twoshot_fault(*f))
                check(p.AllReduceTwoShot(reps=1), n, bpp, 1, fault=f)
            p.SetOption(a.OPT_ALLREDUCE_TWOSHOT_FAULT, 0)


def test_a_dropped_unit_reads_as_zeros_because_every_rep_clears_the_output(pkg):
    """The warm-up delivers the unit, timed rep 1 drops it to the receiver, rep 2 delivers it again.  The receiver
    finds every word of the unit bad in rep 1 only because the check after the warm-up overwrote it with 0; without
    that clear it would still hold the warm-up's identical sums and pass."""
    a = pkg.abi
    n, bpp = 4, 1 << 20
    sizes = allreduce_ref.ladder(bpp)
    with open_bpp(pkg, n, bpp) as p:
        for path in PATHS:
            p.SetOption(a.OPT_PATH, path)
            for recv, k, word in ((2, len(sizes) - 1, 3 * 1024 + 5), (0, 2, 1000), (3, 0, 0)):
                f = (recv, k, word, True)
                p.SetOption(a.OPT_ALLREDUCE_TWOSHOT_FAULT, a.allreduce_twoshot_fault(*f))
                ar = check(p.AllReduceTwoShot(reps=2), n, bpp, 2, fault=f)
                u0 = word // ref.UNIT_WORDS * ref.UNIT_WORDS
                assert ar.bad_words[recv][k] == ref.unit_words(sizes[k], word) and ar.first_bad[recv][k] == 8 * u0
                assert ar.bad_sizes[recv] == 1 << k and ar.status[recv] == ERR_INTEGRITY
            p.SetOption(a.OPT_ALLREDUCE_TWOSHOT_FAULT, 0)
            check(p.AllReduceTwoShot(reps=2), n, bpp, 2)


def test_a_corrupt_word_fails_exactly_the_sizes_that_cover_it_in_every_row(pkg):
    n, bpp = 3, EDGE_BPP
    W = bpp // 8
    with open_bpp(pkg, n, bpp) as p:
        for path in PATHS:
            p.SetOption(pkg.abi.OPT_PATH, path)
            for j, w in ((2, 5), (0, 40000), (1, W - 1)):
                p.Corrupt(j, 8 * w, 1 << 17)
                check(p.AllReduceTwoShot(reps=2), n, bpp, 2, corrupt={(j, w): 1 << 17})
                p.Corrupt(j, 8 * w, 1 << 17)  # restore
            check(p.AllReduceTwoShot(reps=1), n, bpp, 1)


def test_an_armed_fault_that_names_nothing_is_refused(pkg, oracle):
    a = pkg.abi
    n = 3
    with open_same(pkg, n) as p:
        bpp = pkg.plan(n, 1 << 20, MODE_SLICED).bytes_per_pair
        sizes = allreduce_ref.ladder(bpp)
        ar = p.AllReduceTwoShot(reps=2)
        for bad in (a.allreduce_twoshot_fault(n, 0, 0), a.allreduce_twoshot_fault(0, len(sizes), 0),
                    a.allreduce_twoshot_fault(0, 0, sizes[0] // 8), (1 << 24) | 5, (1 << 32) | 5,
                    (1 << 49) | a.allreduce_twoshot_fault(0, 0, 0), (1 << 63) | a.allreduce_twoshot_fault(1, 1, 1)):
            p.SetOption(a.OPT_ALLREDUCE_TWOSHOT_FAULT, bad)
            rc, t = p.allreduce_twoshot_raw(2)
            assert rc == ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0, hex(bad)
        p.SetOption(a.OPT_ALLREDUCE_TWOSHOT_FAULT, 0)
        ar2 = p.AllReduceTwoShot(reps=2)
        assert ar2.call_seq == ar.call_seq + 1
        assert_all_clean(ar2, oracle, bpp)
        rc, t = p.allreduce_twoshot_raw(a.ALLREDUCE_MAX_REPS + 1)
        assert rc == ERR_ARG and (t.abi, t.n, t.reps, t.call_seq, t.row_mask) == (2, n, 65, 0, 0)


def test_a_mapping_that_is_down_stops_every_rank_until_it_is_remapped(pkg, oracle):
    n = 4
    with open_same(pkg, n) as p:
        bpp = pkg.plan(n, 1 << 20, MODE_SLICED).bytes_per_pair
        assert_all_clean(p.AllReduceTwoShot(reps=2), oracle, bpp)  # builds the gather area with every mapping up
        p.UnmapPeer(2, 1)
        ar = p.AllReduceTwoShot(reps=2)
        assert ar.call_seq == 2 and ar.ms < 5000  # returned without waiting for a watchdog
        for r in range(n):
            assert not ar.measured[r] and ar.status[r] == ERR_STATE and ar.ns_median[r] is None
        p.RemapPeer(2, 1)
        ar = p.AllReduceTwoShot(reps=2)
        assert ar.call_seq == 3
        assert_all_clean(ar, oracle, bpp)


def test_simulated_mig_runs_no_rank(pkg):
    n = 2
    with open_same(pkg, n, flags=SIMULATE_MIG) as p:
        ar = p.AllReduceTwoShot(reps=2)
        assert ar.ms < 5000
        for r in range(n):
            assert not ar.measured[r] and ar.ns_median[r] is None and ar.status[r] == ERR_UNSUPPORTED


def test_callable_before_the_first_run_and_disturbs_nothing(pkg, oracle):
    n, nbytes = 2, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        one = p.AllReduce(reps=2)
        aa = p.AllToAll(reps=2)
        assert_all_clean(p.AllReduceTwoShot(reps=2), oracle, nbytes)
        r1 = p.Run()
        diags = [(op, i, j, p.Diagnose(op, i, j)) for i, j in ((0, 1), (1, 0)) for op in ("read", "write")]
        ts = p.AllReduceTwoShot(reps=2)
        assert ts.call_seq == 2
        assert_all_clean(ts, oracle, nbytes)
        for op, i, j, d in diags:
            d2 = p.Diagnose(op, i, j)
            assert (d2.bad_words, d2.run_seq, d2.region_offset) == (d.bad_words, d.run_seq, d.region_offset) == \
                (0, r1.run_seq, d.region_offset)
        one2 = p.AllReduce(reps=2)
        assert one2.call_seq == 2 and (one2.sum, one2.xr, one2.status, one2.bad_words) == \
            (one.sum, one.xr, one.status, one.bad_words)
        aa2 = p.AllToAll(reps=2)
        assert aa2.call_seq == 2 and aa2.area_bytes == aa.area_bytes
        assert aa2.cell_status == aa.cell_status and aa2.bad_words == aa.bad_words
        r2 = p.Run()
        assert r2.run_seq == r1.run_seq + 1 and r2.reach == r1.reach and not r2.aborted
        assert (r2.sum_read, r2.xor_read) == (r1.sum_read, r1.xor_read)
        words = r2.bytes_per_pair // 8
        for i, j in ((0, 1), (1, 0)):
            assert (r2.sum_write[i][j], r2.xor_write[i][j]) == oracle.write_checksum(SEED, i, j, r2.run_seq, words)


def test_the_rep_spans_the_slowest_rank(pkg):
    """A rep ends at the closing release, when every rank's pushes are in: with one rank on a single CTA the other
    ranks' reps take as long as its own, where in the one-shot they need not."""
    a = pkg.abi
    n = 3
    with open_same(pkg, n) as p:
        p.SetOption(a.OPT_CTAS_RANK, (1 << 16) | 1)
        ts = p.AllReduceTwoShot(reps=4)
        big = len(ts.sizes) - 1
        slow = ts.ns_median[0][big]
        for r in (1, 2):
            assert ts.ns_median[r][big] >= 0.5 * slow, (r, ts.ns_median[r][big], slow)


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world, n_local = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
    cfg = m.Config(ordinals=[0] * n_local, bytes=1 << 20, world_size=world, rank=rank, session=session,
                   flags=0x40 | (0x10 if n_local > 1 else 0), ctas=8, timeout_ms=30000)

    def dump(ar):
        return {"row_mask": ar.row_mask, "measured": ar.measured, "status": ar.status, "sum": ar.sum, "xr": ar.xr,
                "bad_words": ar.bad_words, "ns_min": ar.ns_min, "sizes": ar.sizes, "call_seq": ar.call_seq}

    with m.Open(cfg) as p:
        out = {"calls": [dump(p.AllReduceTwoShot(reps=2)), dump(p.AllReduceTwoShot(reps=3))]}
        rc, t = p.allreduce_twoshot_raw(2 + rank)  # the processes disagree
        out["mismatch"] = {"rc": rc, "call_seq": t.call_seq, "measured": sum(t.measured)}
        out["after"] = dump(p.AllReduceTwoShot(reps=2))
        out["one_shot"] = dump(p.AllReduce(reps=2))
        r = p.Run(gather=True)
        out["run"] = {"reach": r.reach, "aborted": r.aborted}
    print("RESULT " + json.dumps(out))
    """
) % ROOT


@pytest.mark.parametrize("n_local", [1, 2], ids=["2x1", "2x2"])
def test_two_processes_agree_and_fill_their_own_rows(pkg, n_local):
    """Both processes drive GPU 0, so their contexts are time-sliced and the times only need to be positive."""
    world = 2
    n = world * n_local
    outs = run_children(CHILD, world, n_local)
    sizes = allreduce_ref.ladder(pkg.plan(n, 1 << 20, MODE_SLICED).bytes_per_pair)
    expect = [list(sx) for sx in allreduce_ref.expected(SEED, n, tuple(sizes))]
    for rank, o in enumerate(outs):
        mine = set(range(rank * n_local, (rank + 1) * n_local))
        assert [c["call_seq"] for c in o["calls"]] + [o["after"]["call_seq"]] == [1, 2, 3]
        assert o["mismatch"] == {"rc": ERR_ARG, "call_seq": 0, "measured": 0}
        for c in o["calls"] + [o["after"], o["one_shot"]]:
            assert c["row_mask"] == sum(1 << r for r in mine) and c["sizes"] == sizes
            for r in range(n):
                assert c["measured"][r] == (r in mine), r
                if r in mine:
                    assert c["status"][r] == 0 and all(t > 0 for t in c["ns_min"][r])
                    assert [[s, x] for s, x in zip(c["sum"][r], c["xr"][r])] == expect, r
                    assert c["bad_words"][r] == [0] * len(sizes)
                else:
                    assert c["sum"][r] is None
        assert o["one_shot"]["call_seq"] == 1
        assert o["run"]["reach"] == [[1] * n for _ in range(n)] and not o["run"]["aborted"]
