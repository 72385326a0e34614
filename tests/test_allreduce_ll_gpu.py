"""cdprobe_allreduce_ll on the GPU: every row's output at every size of the LL ladder is the pattern's sum, word for
word and in (S, X), and equals the one-shot's and the two-shot's on the same handle; tiny ladders, ladders cut at
1 MiB, small and unequal grids (the agreed word partition); a word corrupted at rest fails exactly the sizes that
cover it in every row; a corrupted packet fails only its receiver's row and size; an output word a rank never stores
in a size fails exactly that row and size, whatever an earlier size, a one-shot call or a closed handle left there; a
delayed sender stretches every rank's rep and leaves every row exact; a mapping that is down stops every rank without waiting; two processes with
unequal grids agree; repeated calls stay exact and disturb nothing; the times are ordered and bounded.  Several ranks
share one device where a test needs N > 1, with CTA counts that let their grids be resident together (every rank
waits for every other's packets).  No test drives a kernel past its deadline."""
import functools
import textwrap

import numpy as np
import pytest

import allreduce_ll_ref as ref
import allreduce_ref
import word_ref
from conftest import ROOT
from harness import run_children

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
SIMULATE_MIG = 0x200
MODE_REACH, MODE_SLICED, MODE_FULL = 0, 1, 2
ERR_ARG, ERR_UNSUPPORTED, ERR_STATE, ERR_INTEGRITY = -2, -8, -9, -10
PATH_LL = 3
U64_MAX = word_ref.U64_MAX
EDGE_BPP = 57 * 8192 + 384  # a partial last line of a partial last granule: ladder 4096 ... 262144, 467328
PER_ROW = ("sum", "xr", "bad_words", "first_bad")


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


def check(ar, n, bpp, reps, corrupt=None, fault=None, unstored=None):
    """Every row at every size, from the words at rest: corrupt {(rank, word): mask} is xored into the sources, and
    fault (sender, receiver, k, word) xors the data of that packet, the sender's salted input, with 1 in timed rep 1
    only, which moves the receiver's output word by +1 or -1.  unstored (rank, k, word), the mode-2 fault: that rank
    makes no store to the word in any rep of size k, so the word check after the size reads 0 there (the output
    starts zeroed and every check clears it), while (S, X), folded from the sums, stays clean.  The word check and
    (S, X) are the last timed rep's; bad_sizes also counts every earlier rep's (S, X)."""
    corrupt = corrupt or {}
    sizes = ref.ladder(bpp)
    assert ar.sizes == sizes and ar.reps == reps and ar.n == n and ar.path == PATH_LL
    W = min(bpp, ref.MAX_BYTES) // 8
    clean = sum(src(j, W) for j in range(n))
    at_rest = clean.copy()
    for (j, w), m in corrupt.items():
        orig = int(src(j, W)[w])
        at_rest[w] = np.uint64((int(at_rest[w]) - orig + (orig ^ m)) % (1 << 64))
    for r in range(n):
        bits = 0
        for k, s in enumerate(sizes):
            last = at_rest[:s // 8]
            if fault is not None and (r, k) == fault[1:3]:
                bits |= 1 << k
                if reps == 1:
                    v = (int(src(fault[0], W)[fault[3]]) + ref.salt(SEED, fault[0], ref.flag(ar.call_seq, k, 1)))
                    last = last.copy()
                    last[fault[3]] = np.uint64((int(last[fault[3]]) + ((v ^ 1) - v)) % (1 << 64))
            seen = last
            if unstored is not None and (r, k) == unstored[:2]:
                seen = last.copy()
                seen[unstored[2]] = 0
            bad = np.flatnonzero(seen != clean[:s // 8])
            if len(bad):
                bits |= 1 << k
            ctx = (r, s, fault)
            assert (ar.sum[r][k], ar.xr[r][k]) == allreduce_ref.checksum(last), ctx
            assert ar.bad_words[r][k] == len(bad), (ctx, ar.bad_words[r][k])
            assert ar.first_bad[r][k] == (8 * int(bad[0]) if len(bad) else U64_MAX), (ctx, ar.first_bad[r][k])
            assert 0 < ar.ns_min[r][k] <= ar.ns_median[r][k] <= ar.ns_max[r][k], ctx
        assert ar.measured[r] and ar.bad_sizes[r] == bits, (r, ar.bad_sizes[r], bits)
        assert ar.status[r] == (ERR_INTEGRITY if bits else 0), r
        assert (ar.t0_ns[r], ar.peak_gbps[r], ar.half_bytes[r]) == allreduce_ref.summary(sizes, ar.ns_median[r])
    assert_fits_in_call(ar)
    return ar


def assert_fits_in_call(ar):
    """A rank's timed reps run one after another inside the call, so their times must fit its wall clock."""
    for r in range(ar.n):
        if ar.ns_min[r]:
            assert sum(ar.reps * t for t in ar.ns_min[r]) / 1e6 <= ar.ms, r
            assert sum(ar.reps * t for t in ar.ns_median[r]) / 1e6 <= ar.ms, r


def assert_rows_equal(ll, other):
    """LL's rows equal another all-reduce's at LL's sizes (a prefix of the bwcurve ladder)."""
    ns = len(ll.sizes)
    assert other.sizes[:ns] == ll.sizes
    for r in range(ll.n):
        assert ll.status[r] == other.status[r] and ll.measured[r] == other.measured[r], r
        assert ll.bad_sizes[r] == other.bad_sizes[r] & ((1 << ns) - 1), r
        for f in PER_ROW:
            assert getattr(ll, f)[r] == getattr(other, f)[r][:ns], (r, f)


@pytest.mark.parametrize("mode", [MODE_SLICED, MODE_FULL, MODE_REACH], ids=["sliced", "full", "reach"])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 8, 16])
def test_every_row_exact_and_equal_to_the_one_shot_and_the_two_shot(pkg, n, mode):
    with open_same(pkg, n, mode=mode) as p:
        bpp = p.Info().bytes_per_pair
        for path in (0, 2):  # LL ignores the data path; the one-shot and two-shot follow it
            p.SetOption(pkg.abi.OPT_PATH, path)
            ll = check(p.AllReduceLL(reps=2), n, bpp, 2)
            assert (ll.row_mask, ll.call_seq) == ((1 << n) - 1, path // 2 + 1)
            assert_rows_equal(ll, p.AllReduce(reps=2))
            assert_rows_equal(ll, p.AllReduceTwoShot(reps=2))


@pytest.mark.parametrize("bpp", [128, 4096, EDGE_BPP, (3 << 20) + 128])
@pytest.mark.parametrize("n", [1, 3])
def test_tiny_ladders_and_the_ladder_cut_at_1_mib(pkg, n, bpp):
    with open_bpp(pkg, n, bpp) as p:
        ll = check(p.AllReduceLL(reps=1), n, bpp, 1)
        assert ll.sizes[-1] == min(bpp, 1 << 20)
        check(p.AllReduceLL(reps=3), n, bpp, 3)
        assert_rows_equal(p.AllReduceLL(reps=2), p.AllReduce(reps=2))


GRIDS = [("ctas", 1), ("ctas", 2), ("ctas", 3), ("ctas", 7), ("rank", (1, 8, 3)), ("rank", (7, 2, 5))]


@pytest.mark.parametrize("grid", GRIDS, ids=[f"{g[0]}{'-'.join(map(str, g[1])) if g[0] == 'rank' else g[1]}"
                                             for g in GRIDS])
def test_grids_and_unequal_grids_split_the_words_alike(pkg, grid):
    """The words are split over the warps of the smallest grid on every rank; CTAs beyond it only join the barriers
    and the word check.  Clean calls, and a corrupted packet on the last word of the last, partial line."""
    a = pkg.abi
    n, bpp = 3, EDGE_BPP
    sizes = ref.ladder(bpp)
    with open_bpp(pkg, n, bpp) as p:
        if grid[0] == "ctas":
            p.SetOption(a.OPT_CTAS, grid[1])
        else:
            for li, c in enumerate(grid[1]):
                p.SetOption(a.OPT_CTAS_RANK, ((li + 1) << 16) | c)
        info = p.Info()
        assert [info.ctas[li] for li in range(n)] == (list(grid[1]) if grid[0] == "rank" else [grid[1]] * n)
        check(p.AllReduceLL(reps=1), n, bpp, 1)
        check(p.AllReduceLL(reps=4), n, bpp, 4)
        f = (2, 0, len(sizes) - 1, bpp // 8 - 1)
        p.SetOption(a.OPT_ALLREDUCE_LL_FAULT, a.allreduce_ll_fault(*f))
        check(p.AllReduceLL(reps=1), n, bpp, 1, fault=f)
        # an output word left unstored: word 0 of size 0, a word below the previous size at k >= 1 (which that size
        # stored and its check cleared), the last word of the largest LL size
        for u in ((0, 0, 0), (2, 3, sizes[2] // 8 - 1), (1, len(sizes) - 1, sizes[-1] // 8 - 1)):
            p.SetOption(a.OPT_ALLREDUCE_LL_FAULT, a.allreduce_ll_fault(u[0], u[0], u[1], u[2], mode=2))
            for reps in (1, 3):
                ar = check(p.AllReduceLL(reps=reps), n, bpp, reps, unstored=u)
                assert ar.bad_words[u[0]][u[1]] == 1 and ar.first_bad[u[0]][u[1]] == 8 * u[2], (u, reps)
        p.SetOption(a.OPT_ALLREDUCE_LL_FAULT, 0)
        check(p.AllReduceLL(reps=2), n, bpp, 2)


def test_a_corrupt_word_fails_exactly_the_sizes_that_cover_it_in_every_row(pkg):
    n, bpp = 3, EDGE_BPP
    W = bpp // 8
    with open_bpp(pkg, n, bpp) as p:
        for j, w in ((2, 5), (0, 40000), (1, W - 1)):
            p.Corrupt(j, 8 * w, 1 << 17)
            check(p.AllReduceLL(reps=2), n, bpp, 2, corrupt={(j, w): 1 << 17})
            p.Corrupt(j, 8 * w, 1 << 17)  # restore
        check(p.AllReduceLL(reps=1), n, bpp, 1)


def test_a_corrupted_packet_fails_only_its_receiver_and_size(pkg):
    """With reps == 1 the word check sees the word (first_bad is its offset); with more reps only rep 1's (S, X) does,
    and the last rep's output is clean again."""
    a = pkg.abi
    n, bpp = 4, 1 << 20
    sizes = ref.ladder(bpp)
    with open_bpp(pkg, n, bpp) as p:
        for f in ((0, 1, len(sizes) - 1, 3 * 1024 + 5), (3, 0, 2, 1000), (1, 2, 0, 0), (2, 3, 0, 511)):
            p.SetOption(a.OPT_ALLREDUCE_LL_FAULT, a.allreduce_ll_fault(*f))
            ar = check(p.AllReduceLL(reps=1), n, bpp, 1, fault=f)
            assert ar.bad_words[f[1]][f[2]] == 1 and ar.first_bad[f[1]][f[2]] == 8 * f[3]
            ar = check(p.AllReduceLL(reps=3), n, bpp, 3, fault=f)
            assert ar.bad_sizes[f[1]] == 1 << f[2] and ar.bad_words[f[1]][f[2]] == 0
        p.SetOption(a.OPT_ALLREDUCE_LL_FAULT, 0)
        check(p.AllReduceLL(reps=2), n, bpp, 2)


def test_an_unstored_word_is_seen_whatever_the_output_held_before(pkg):
    """Every rep, size and call stores the same sums into the same words, so a word the LL leaves unstored would still
    hold what a one-shot call on the same handle, or a closed handle's output in the same process, left there.  The
    output is zeroed at the start of every call, so the unstored word fails exactly its row and size each time."""
    a = pkg.abi
    n, bpp = 3, EDGE_BPP
    sizes = ref.ladder(bpp)
    u = (1, 4, sizes[3] // 8 - 2)  # below size 3, so size 3 also stored it in this call
    with open_bpp(pkg, n, bpp) as p:
        one = p.AllReduce(reps=2)
        assert all(one.status[r] == 0 for r in range(n)) and one.sizes[:len(sizes)] == sizes
        p.SetOption(a.OPT_ALLREDUCE_LL_FAULT, a.allreduce_ll_fault(u[0], u[0], u[1], u[2], mode=2))
        check(p.AllReduceLL(reps=2), n, bpp, 2, unstored=u)
    with open_bpp(pkg, n, bpp) as p:  # the same config and seed: its scratch may reuse the freed one
        p.SetOption(a.OPT_ALLREDUCE_LL_FAULT, a.allreduce_ll_fault(u[0], u[0], u[1], u[2], mode=2))
        ar = check(p.AllReduceLL(reps=1), n, bpp, 1, unstored=u)
        assert ar.call_seq == 1 and ar.bad_words[u[0]][u[1]] == 1


def test_a_delayed_sender_stretches_every_rank_and_every_row_stays_exact(pkg):
    """The sender waits 2 ms before its first push of timed rep 1 of size k.  Its own rep 1 spans the wait; every
    other rank's rep 1 ends only after the sender's packets arrive, and starts when its rep 0 ended, at most a few
    microseconds (the skew of the ranks' rep-0 ends) after the sender's rep 0 did.  Without the receiver's flag
    check the peers would add whatever rep 1's slots held before the sender's packets landed (an earlier rep's
    packets, with another salt), and their rows would fail."""
    a = pkg.abi
    n, bpp, delay_us = 4, 1 << 20, 2000
    sizes = ref.ladder(bpp)
    with open_bpp(pkg, n, bpp) as p:
        for sender, k in ((1, len(sizes) - 1), (3, 0)):
            p.SetOption(a.OPT_ALLREDUCE_LL_FAULT, a.allreduce_ll_fault(sender, 0, k, delay_us, mode=1))
            ar = check(p.AllReduceLL(reps=3), n, bpp, 3)
            assert ar.ns_max[sender][k] >= delay_us * 1e3, (sender, k, ar.ns_max[sender][k])
            for r in range(n):
                assert ar.ns_max[r][k] >= 0.99 * delay_us * 1e3, (r, k, ar.ns_max[r][k])
        p.SetOption(a.OPT_ALLREDUCE_LL_FAULT, 0)


NAMES_NOTHING = "the armed LL all-reduce fault names no packet, size or delay of this call"


def test_an_armed_fault_that_names_nothing_is_refused(pkg):
    a = pkg.abi
    n = 3
    with open_same(pkg, n) as p:
        bpp = p.Info().bytes_per_pair
        sizes = ref.ladder(bpp)
        ar = check(p.AllReduceLL(reps=2), n, bpp, 2)
        for bad in (a.allreduce_ll_fault(n, 0, 0, 0), a.allreduce_ll_fault(0, n, 0, 0),
                    a.allreduce_ll_fault(0, 1, len(sizes), 0), a.allreduce_ll_fault(0, 1, 0, sizes[0] // 8),
                    a.allreduce_ll_fault(1, 1, 0, 0), a.allreduce_ll_fault(0, 1, 0, 10_000_000, mode=1),
                    (2 << 48) | a.allreduce_ll_fault(0, 1, 0, 0), (3 << 48) | a.allreduce_ll_fault(0, 0, 0, 0),
                    (1 << 63) | a.allreduce_ll_fault(0, 1, 0, 0), a.allreduce_ll_fault(2, 0, len(sizes) - 1, 5, mode=2),
                    a.allreduce_ll_fault(1, 1, 0, sizes[0] // 8, mode=2), a.allreduce_ll_fault(n, n, 0, 0, mode=2),
                    a.allreduce_ll_fault(2, 2, len(sizes), 0, mode=2), (1 << 24) | 5):
            p.SetOption(a.OPT_ALLREDUCE_LL_FAULT, bad)
            rc, t = p.allreduce_ll_raw(2)
            assert rc == ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0, hex(bad)
            assert p._lib.cdprobe_last_error().decode() == NAMES_NOTHING, hex(bad)
        p.SetOption(a.OPT_ALLREDUCE_LL_FAULT, 0)
        ar2 = check(p.AllReduceLL(reps=2), n, bpp, 2)
        assert ar2.call_seq == ar.call_seq + 1
        rc, t = p.allreduce_ll_raw(a.ALLREDUCE_MAX_REPS + 1)
        assert rc == ERR_ARG and (t.abi, t.n, t.reps, t.call_seq, t.row_mask, t.path) == (2, n, 65, 0, 0, PATH_LL)


def test_a_mapping_that_is_down_stops_every_rank_until_it_is_remapped(pkg):
    n = 4
    with open_same(pkg, n) as p:
        bpp = p.Info().bytes_per_pair
        check(p.AllReduceLL(reps=2), n, bpp, 2)  # builds the LL area with every mapping up
        p.UnmapPeer(2, 1)
        ar = p.AllReduceLL(reps=2)
        assert ar.call_seq == 2 and ar.ms < 5000  # returned without waiting for a watchdog
        for r in range(n):
            assert not ar.measured[r] and ar.status[r] == ERR_STATE and ar.ns_median[r] is None
        p.RemapPeer(2, 1)
        assert check(p.AllReduceLL(reps=2), n, bpp, 2).call_seq == 3


def test_an_unmapped_peer_before_the_first_call_runs_no_rank(pkg):
    n = 3
    with open_same(pkg, n) as p:
        p.UnmapPeer(0, 2)
        ar = p.AllReduceLL(reps=2)
        assert ar.ms < 5000
        for r in range(n):
            assert not ar.measured[r] and ar.status[r] == ERR_STATE


def test_simulated_mig_runs_no_rank(pkg):
    n = 2
    with open_same(pkg, n, flags=SIMULATE_MIG) as p:
        ar = p.AllReduceLL(reps=2)
        assert ar.ms < 5000
        for r in range(n):
            assert not ar.measured[r] and ar.ns_median[r] is None and ar.status[r] == ERR_UNSUPPORTED


def test_repeated_calls_stay_exact_and_disturb_nothing(pkg, oracle):
    n, nbytes = 3, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        bpp = p.Info().bytes_per_pair
        one = p.AllReduce(reps=2)
        ts = p.AllReduceTwoShot(reps=2)
        aa = p.AllToAll(reps=2)
        r1 = p.Run()
        diags = [(i, j, p.Diagnose("write", i, j)) for i, j in ((0, 1), (2, 0))]
        for c in range(1, 7):
            ll = check(p.AllReduceLL(reps=1 + c % 3), n, bpp, 1 + c % 3)
            assert ll.call_seq == c
            if c == 3:
                assert_rows_equal(ll, p.AllReduceTwoShot(reps=2))
        for i, j, d in diags:
            d2 = p.Diagnose("write", i, j)
            assert (d2.bad_words, d2.run_seq, d2.region_offset) == (0, r1.run_seq, d.region_offset)
        one2 = p.AllReduce(reps=2)
        assert one2.call_seq == 2 and [getattr(one2, f) for f in PER_ROW + ("status",)] == \
            [getattr(one, f) for f in PER_ROW + ("status",)]
        ts2 = p.AllReduceTwoShot(reps=2)
        assert ts2.call_seq == 3 and [getattr(ts2, f) for f in PER_ROW] == [getattr(ts, f) for f in PER_ROW]
        aa2 = p.AllToAll(reps=2)
        assert aa2.call_seq == 2 and aa2.cell_status == aa.cell_status and aa2.bad_words == aa.bad_words
        r2 = p.Run()
        assert r2.run_seq == r1.run_seq + 1 and r2.reach == r1.reach and not r2.aborted
        assert (r2.sum_read, r2.xor_read) == (r1.sum_read, r1.xor_read)
        words = r2.bytes_per_pair // 8
        for i in range(n):
            for j in range(n):
                if i != j:
                    assert (r2.sum_write[i][j], r2.xor_write[i][j]) == oracle.write_checksum(SEED, i, j, r2.run_seq,
                                                                                              words)
        check(p.AllReduceLL(reps=2), n, bpp, 2)


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world, n_local = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
    cfg = m.Config(ordinals=[0] * n_local, bytes=1 << 20, world_size=world, rank=rank, session=session,
                   flags=0x40 | (0x10 if n_local > 1 else 0), ctas=8 if rank == 0 else 3, timeout_ms=30000)

    def dump(ar):
        return {"row_mask": ar.row_mask, "measured": ar.measured, "status": ar.status, "sum": ar.sum, "xr": ar.xr,
                "bad_words": ar.bad_words, "first_bad": ar.first_bad, "bad_sizes": ar.bad_sizes,
                "ns_min": ar.ns_min, "sizes": ar.sizes, "call_seq": ar.call_seq, "path": ar.path}

    with m.Open(cfg) as p:
        out = {"calls": [dump(p.AllReduceLL(reps=2)), dump(p.AllReduceLL(reps=3))]}
        rc, t = p.allreduce_ll_raw(2 + rank)  # the processes disagree
        out["mismatch"] = {"rc": rc, "call_seq": t.call_seq, "measured": sum(t.measured)}
        out["after"] = dump(p.AllReduceLL(reps=2))
        out["one_shot"] = dump(p.AllReduce(reps=2))
        r = p.Run(gather=True)
        out["run"] = {"reach": r.reach, "aborted": r.aborted}
    print("RESULT " + json.dumps(out))
    """
) % ROOT


@pytest.mark.parametrize("n_local", [1, 2], ids=["2x1", "2x2"])
def test_two_processes_with_unequal_grids_agree_and_fill_their_own_rows(pkg, n_local):
    """Both processes drive GPU 0 with 8 and 3 CTAs per rank, so the domain's smallest grid is 3 and the processes'
    rows must still be identical; their contexts are time-sliced, so the times only need to be positive."""
    world = 2
    n = world * n_local
    outs = run_children(CHILD, world, n_local)
    sizes = ref.ladder(pkg.plan(n, 1 << 20, MODE_SLICED).bytes_per_pair)
    expect = [list(sx) for sx in allreduce_ref.expected(SEED, n, tuple(sizes))]
    ns = len(sizes)
    for rank, o in enumerate(outs):
        mine = set(range(rank * n_local, (rank + 1) * n_local))
        assert [c["call_seq"] for c in o["calls"]] + [o["after"]["call_seq"]] == [1, 2, 3]
        assert o["mismatch"] == {"rc": ERR_ARG, "call_seq": 0, "measured": 0}
        for c in o["calls"] + [o["after"]]:
            assert c["row_mask"] == sum(1 << r for r in mine) and c["sizes"] == sizes and c["path"] == PATH_LL
            for r in range(n):
                assert c["measured"][r] == (r in mine), r
                if r in mine:
                    assert c["status"][r] == 0 and c["bad_sizes"][r] == 0 and all(t > 0 for t in c["ns_min"][r])
                    assert [[s, x] for s, x in zip(c["sum"][r], c["xr"][r])] == expect, r
                    assert c["bad_words"][r] == [0] * ns and c["first_bad"][r] == [U64_MAX] * ns
                    for f in ("sum", "xr", "bad_words", "first_bad"):
                        assert c[f][r] == o["one_shot"][f][r][:ns], (r, f)
                else:
                    assert c["sum"][r] is None
        assert o["run"]["reach"] == [[1] * n for _ in range(n)] and not o["run"]["aborted"]
    for r in range(n):  # identical rows in both processes' views of the domain
        owner = outs[r // n_local]["after"]
        assert [[s, x] for s, x in zip(owner["sum"][r], owner["xr"][r])] == expect
