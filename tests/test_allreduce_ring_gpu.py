"""cdprobe_allreduce_ring on the GPU: every row's output at every size is the pattern's sum, word for word and in
(S, X), and equals the one-shot's and the two-shot's on the same handle; tiny ladders where some ranks own no unit;
every grid, unequal grids and a single CTA finish (the deadlock-freedom of the steps); a word corrupted at rest fails
exactly the sizes that cover it in every row; a corrupted or dropped push fails exactly the rows the restatement
names; a delayed sender stretches every rank's rep and leaves every row exact; a mapping that is down stops every rank
without waiting; two processes agree; repeated calls stay exact and disturb nothing.  Several ranks share one device
where a test needs N > 1, with CTA counts that let their grids be resident together (every rank waits for its
predecessor's flags).  No test drives a kernel past its deadline."""
import functools
import textwrap

import numpy as np
import pytest

import allreduce_ref
import allreduce_ring_ref as ref
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
PATH_RING = 4
U64_MAX = word_ref.U64_MAX
GIB = 1 << 30
REF_MAX = 64 << 20  # sizes up to this get their (S, X) from the numpy reference; larger ones (N = 1) from the oracle
EDGE_BPP = 57 * 8192 + 384  # a partial last unit in a partial last granule: ladder 4096 ... 262144, 467328
PER_ROW = ("sum", "xr", "bad_words", "first_bad")
M64 = 1 << 64


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


def faulted(rest, n, r, size, fault):
    """What row r holds after the faulted rep: fault (sender, k, word, phase, mode) of mode 0 or 1."""
    sender, _, word, phase, mode = fault
    if r not in ref.failing_rows(n, sender, phase, size, word):
        return rest
    out = rest.copy()
    u0 = word // ref.UNIT_WORDS * ref.UNIT_WORDS
    u1 = min(u0 + ref.UNIT_WORDS, size // 8)
    c = ref.chunk_of(size, n, word)
    if phase == 1 and mode == 0:  # the full chunk: the word leaves xored with 1
        out[word] ^= np.uint64(1)
        return out
    # the partial of chunk c the sender pushed in the reduce-scatter: the inputs of ranks sender - s ... sender
    part = sum(src(j, size // 8) for j in ref.partial_ranks(n, sender, c)) if sender != c else None
    if phase == 1:  # the full chunk never arrives: its place still holds what the receiver got in the reduce-scatter,
        out[u0:u1] = 0 if part is None else part[u0:u1]  # the sender's partial, or the clear's 0s if it got none
        return out
    if mode == 0:
        p = int(part[word])
        out[word] = np.uint64((int(out[word]) + (p ^ 1) - p) % M64)
    else:
        out[u0:u1] -= part[u0:u1]
    return out


def check(ar, n, bpp, reps, corrupt=None, fault=None):
    """Every row at every size, from the words at rest: corrupt {(rank, word): mask} is xored into the sources, and
    fault (sender, k, word, phase, mode) acts in timed rep 1 only.  bad_words count every rep, warm-up included;
    (S, X) is the last timed rep's."""
    corrupt = corrupt or {}
    sizes = allreduce_ref.ladder(bpp)
    assert ar.sizes == sizes and ar.reps == reps and ar.n == n and ar.path == PATH_RING
    W = bpp // 8
    clean = sum(src(j, W) for j in range(n))
    at_rest = clean.copy()
    for (j, w), m in corrupt.items():
        orig = int(src(j, W)[w])
        at_rest[w] = np.uint64((int(at_rest[w]) - orig + (orig ^ m)) % M64)
    for r in range(n):
        bits = 0
        for k, s in enumerate(sizes):
            rep_words = at_rest[:s // 8]
            bad = np.flatnonzero(rep_words != clean[:s // 8])
            n_bad, first = (reps + 1) * len(bad), [int(bad[0])] if len(bad) else []
            last = rep_words
            if fault is not None and fault[1] == k and fault[4] < 2:
                hit = faulted(rep_words, n, r, s, fault)
                hbad = np.flatnonzero(hit != clean[:s // 8])
                n_bad += len(hbad) - len(bad)
                first += [int(hbad[0])] if len(hbad) else []
                if len(hbad) != len(bad) or (hit != rep_words).any():
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


def assert_fits_in_call(ar):
    """A rank's timed reps run one after another inside the call, so their least times must fit its wall clock."""
    for r in range(ar.n):
        if ar.ns_min[r]:
            assert sum(ar.reps * t for t in ar.ns_min[r]) / 1e6 <= ar.ms, r
            assert max(ar.ns_median[r]) / 1e6 <= ar.ms


def assert_rows_equal(ring, other):
    for r in range(ring.n):
        assert ring.status[r] == other.status[r] and ring.measured[r] == other.measured[r], r
        assert ring.bad_sizes[r] == other.bad_sizes[r], r
        for f in PER_ROW:
            assert getattr(ring, f)[r] == getattr(other, f)[r], (r, f)


def want(oracle, n, sizes):
    small = tuple(s for s in sizes if s <= REF_MAX)
    got = dict(zip(small, allreduce_ref.expected(SEED, n, small))) if small else {}
    for s in sizes:
        if s not in got:
            assert n == 1, "only the single-rank output is checked against the oracle beyond REF_MAX"
            got[s] = oracle.src_checksum(SEED, 0, 0, s // 8)
    return [got[s] for s in sizes]


@pytest.mark.parametrize("nbytes", [4 << 20, GIB], ids=["4MiB", "1GiB"])
def test_single_rank_every_size_clean(pkg, oracle, nbytes):
    """At N = 1 there are no steps: the rank stores its own prefix into its output, and the check runs as usual.  So
    a 1 GiB rep reads 1 GiB and stores 1 GiB through HBM (ring_rep at n == 1: one step, s = 0, that neither receives
    nor pushes), and takes no less than 2 GiB need at the data sheet's bandwidth."""
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, timeout_ms=60000)) as p:
        ar = p.AllReduceRing(reps=2)
        assert ar.sizes == allreduce_ref.ladder(nbytes) and ar.path == PATH_RING and ar.call_seq == 1
        expect = want(oracle, 1, ar.sizes)
        assert ar.measured[0] and ar.status[0] == 0 and ar.bad_sizes[0] == 0
        assert [(s, x) for s, x in zip(ar.sum[0], ar.xr[0])] == expect
        assert ar.bad_words[0] == [0] * len(ar.sizes) and ar.first_bad[0] == [U64_MAX] * len(ar.sizes)
        assert_fits_in_call(ar)
        if nbytes == GIB:
            assert_hbm_floor(ar, 2 * GIB)


@pytest.mark.parametrize("mode", [MODE_SLICED, MODE_FULL, MODE_REACH], ids=["sliced", "full", "reach"])
@pytest.mark.parametrize("n", [2, 3, 4, 5, 8, 16])
def test_every_row_exact_and_equal_to_the_one_shot_and_the_two_shot(pkg, n, mode):
    with open_same(pkg, n, mode=mode) as p:
        bpp = p.Info().bytes_per_pair
        ring = check(p.AllReduceRing(reps=2), n, bpp, 2)
        assert (ring.row_mask, ring.call_seq) == ((1 << n) - 1, 1)
        assert_rows_equal(ring, p.AllReduceTwoShot(reps=2))
        one = p.AllReduce(reps=2)
        for r in range(n):
            assert (ring.sum[r], ring.xr[r], ring.bad_words[r]) == (one.sum[r], one.xr[r], one.bad_words[r]), r


@pytest.mark.parametrize("bpp", [128, 4224, 16512, 24704])
@pytest.mark.parametrize("n", [3, 5])
def test_tiny_ladders_where_ranks_own_no_unit(pkg, n, bpp):
    with open_bpp(pkg, n, bpp) as p:
        check(p.AllReduceRing(reps=1), n, bpp, 1)
        check(p.AllReduceRing(reps=3), n, bpp, 3)


GRIDS = [("ctas", 1), ("ctas", 2), ("ctas", 3), ("ctas", 7), ("ctas", 40), ("rank", (1, 8, 3)),
         ("rank", (7, 2, 5)), ("rank", (40, 1, 1))]


@pytest.mark.parametrize("grid", GRIDS, ids=[f"{g[0]}{'-'.join(map(str, g[1])) if g[0] == 'rank' else g[1]}"
                                             for g in GRIDS])
def test_every_grid_finishes_exact(pkg, grid):
    """Each warp carries its grains through every step in order and waits only on its predecessor rank's flags, so
    any grid on any rank finishes, down to one CTA and unequal grids; 3 x 40 CTAs fill most of the device's SMs, one CTA
    each, the largest grid whose three ranks stay resident together."""
    a = pkg.abi
    n, bpp = 3, EDGE_BPP
    with open_bpp(pkg, n, bpp) as p:
        if grid[0] == "ctas":
            p.SetOption(a.OPT_CTAS, grid[1])
        else:
            for li, c in enumerate(grid[1]):
                p.SetOption(a.OPT_CTAS_RANK, ((li + 1) << 16) | c)
        info = p.Info()
        assert [info.ctas[li] for li in range(n)] == (list(grid[1]) if grid[0] == "rank" else [grid[1]] * n)
        check(p.AllReduceRing(reps=1), n, bpp, 1)
        check(p.AllReduceRing(reps=4), n, bpp, 4)


def test_a_corrupt_word_fails_exactly_the_sizes_that_cover_it_in_every_row(pkg):
    n, bpp = 3, EDGE_BPP
    W = bpp // 8
    with open_bpp(pkg, n, bpp) as p:
        for j, w in ((2, 5), (0, 40000), (1, W - 1)):
            p.Corrupt(j, 8 * w, 1 << 17)
            check(p.AllReduceRing(reps=2), n, bpp, 2, corrupt={(j, w): 1 << 17})
            p.Corrupt(j, 8 * w, 1 << 17)  # restore
        check(p.AllReduceRing(reps=1), n, bpp, 1)


def pushed_word(n, size, sender, phase, at):
    """A word at fraction `at` of a chunk `sender` pushes in `phase`."""
    U = ref.units(size)
    c = next(c for c in sorted(ref.pushes(n, sender, phase)) if U * (c + 1) // n > U * c // n)
    lo, hi = U * c // n, U * (c + 1) // n
    return min(lo * ref.UNIT_WORDS + int((hi - lo) * ref.UNIT_WORDS * at), size // 8 - 1)


@pytest.mark.parametrize("mode", [0, 1], ids=["corrupt", "drop"])
def test_a_faulted_push_fails_exactly_the_rows_the_restatement_names(pkg, mode):
    """In the reduce-scatter the error enters the full sum and every row fails the size; in the all-gather only the
    rows from the hop to the rank before the chunk's owner do, with first_bad at the word (mode 0) or the unit
    (mode 1).  A dropped unit reads as the clear's 0s where nothing else landed in its place this rep: in the
    reduce-scatter, and in the all-gather when the sender owns the chunk.  With reps == 1 the word check sees it; with
    3 reps only rep 1's (S, X) and the summed bad words do."""
    a = pkg.abi
    n, bpp = 4, 1 << 20
    sizes = allreduce_ref.ladder(bpp)
    with open_bpp(pkg, n, bpp) as p:
        for sender, k, phase, at in ((0, len(sizes) - 1, 0, 0.3), (2, len(sizes) - 1, 1, 0.7), (3, 2, 1, 0.0),
                                     (1, 0, 0, 0.99), (1, len(sizes) - 2, 1, 0.5)):
            word = pushed_word(n, sizes[k], sender, phase, at)
            f = (sender, k, word, phase, mode)
            p.SetOption(a.OPT_ALLREDUCE_RING_FAULT, a.allreduce_ring_fault(sender, k, word, phase, mode))
            ar = check(p.AllReduceRing(reps=1), n, bpp, 1, fault=f)
            rows = ref.failing_rows(n, sender, phase, sizes[k], word)
            assert [r for r in range(n) if ar.bad_sizes[r]] == sorted(rows), f
            for r in rows:
                assert ar.first_bad[r][k] == (8 * word if mode == 0 else 8 * (word // ref.UNIT_WORDS * ref.UNIT_WORDS))
                if mode == 1 and phase == 1 and sender == ref.chunk_of(sizes[k], n, word):
                    assert ar.sum[r][k] == allreduce_ref.checksum(faulted(np.zeros(sizes[k] // 8, np.uint64), n, r,
                                                                          sizes[k], f))[0]  # the unit reads as 0s
                if mode == 0:
                    assert ar.bad_words[r][k] == 1
            check(p.AllReduceRing(reps=3), n, bpp, 3, fault=f)
        p.SetOption(a.OPT_ALLREDUCE_RING_FAULT, 0)
        check(p.AllReduceRing(reps=2), n, bpp, 2)


def test_a_delayed_sender_stretches_every_rank_and_every_row_stays_exact(pkg):
    """Every output chunk passes through every rank, so a sender that waits 2 ms before its first push of timed rep 1
    stretches every rank's rep 1 by at least the wait."""
    a = pkg.abi
    n, bpp, delay_us = 4, 1 << 20, 2000
    sizes = allreduce_ref.ladder(bpp)
    with open_bpp(pkg, n, bpp) as p:
        for sender, k in ((1, len(sizes) - 1), (3, 0)):
            p.SetOption(a.OPT_ALLREDUCE_RING_FAULT, a.allreduce_ring_fault(sender, k, delay_us, mode=2))
            ar = check(p.AllReduceRing(reps=3), n, bpp, 3)
            assert ar.ns_max[sender][k] >= delay_us * 1e3, (sender, k, ar.ns_max[sender][k])
            for r in range(n):  # the others' reps open within microseconds of the sender's
                assert ar.ns_max[r][k] >= 0.99 * delay_us * 1e3, (r, k, ar.ns_max[r][k])
        p.SetOption(a.OPT_ALLREDUCE_RING_FAULT, 0)


def test_an_armed_fault_that_names_nothing_is_refused(pkg):
    a = pkg.abi
    n = 3
    with open_same(pkg, n) as p:
        bpp = p.Info().bytes_per_pair
        sizes = allreduce_ref.ladder(bpp)
        ar = check(p.AllReduceRing(reps=2), n, bpp, 2)
        own0 = pushed_word(n, sizes[0], 1, 0, 0.0)  # a word of a chunk rank 1 pushes in the reduce-scatter
        unpushed = [(s, ph, w) for s in range(n) for ph in (0, 1) for w in (0, sizes[-1] // 8 - 1)
                    if ref.chunk_of(sizes[-1], n, w) not in ref.pushes(n, s, ph)]
        assert unpushed
        bad = [a.allreduce_ring_fault(n, 0, own0), a.allreduce_ring_fault(1, len(sizes), 0),
               a.allreduce_ring_fault(1, 0, sizes[0] // 8), a.allreduce_ring_fault(0, 0, 10_000_000, mode=2),
               (3 << 48) | a.allreduce_ring_fault(1, 0, own0), (2 << 40) | a.allreduce_ring_fault(1, 0, own0),
               (1 << 63) | a.allreduce_ring_fault(1, 0, own0), (1 << 24) | 5]
        bad += [a.allreduce_ring_fault(s, len(sizes) - 1, w, ph, m) for s, ph, w in unpushed for m in (0, 1)]
        for v in bad:
            p.SetOption(a.OPT_ALLREDUCE_RING_FAULT, v)
            rc, t = p.allreduce_ring_raw(2)
            assert rc == ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0, hex(v)
        p.SetOption(a.OPT_ALLREDUCE_RING_FAULT, 0)
        ar2 = check(p.AllReduceRing(reps=2), n, bpp, 2)
        assert ar2.call_seq == ar.call_seq + 1
        rc, t = p.allreduce_ring_raw(a.ALLREDUCE_MAX_REPS + 1)
        assert rc == ERR_ARG and (t.abi, t.n, t.reps, t.call_seq, t.row_mask, t.path) == (2, n, 65, 0, 0, PATH_RING)
    with pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 20, timeout_ms=20000)) as p:  # n = 1 pushes nothing
        p.SetOption(a.OPT_ALLREDUCE_RING_FAULT, a.allreduce_ring_fault(0, 0, 0))
        rc, t = p.allreduce_ring_raw(2)
        assert rc == ERR_ARG and t.call_seq == 0


def test_a_mapping_that_is_down_stops_every_rank_until_it_is_remapped(pkg):
    n = 4
    with open_same(pkg, n) as p:
        bpp = p.Info().bytes_per_pair
        check(p.AllReduceRing(reps=2), n, bpp, 2)  # builds the ring area with every mapping up
        p.UnmapPeer(2, 1)
        ar = p.AllReduceRing(reps=2)
        assert ar.call_seq == 2 and ar.ms < 5000  # returned without waiting for a watchdog
        for r in range(n):
            assert not ar.measured[r] and ar.status[r] == ERR_STATE and ar.ns_median[r] is None
        p.RemapPeer(2, 1)
        assert check(p.AllReduceRing(reps=2), n, bpp, 2).call_seq == 3


def test_an_unmapped_peer_before_the_first_call_keeps_the_ring_off_until_reopened(pkg):
    n = 3
    with open_same(pkg, n) as p:
        p.UnmapPeer(0, 2)
        for remap in (False, True):
            if remap:
                p.RemapPeer(0, 2)  # the probe mapping is back, but the ring area was built without it
            ar = p.AllReduceRing(reps=2)
            assert ar.ms < 5000
            for r in range(n):
                assert not ar.measured[r] and ar.status[r] != 0, (remap, r)
    with open_same(pkg, n) as p:
        check(p.AllReduceRing(reps=2), n, p.Info().bytes_per_pair, 2)


def test_simulated_mig_runs_no_rank(pkg):
    n = 2
    with open_same(pkg, n, flags=SIMULATE_MIG) as p:
        ar = p.AllReduceRing(reps=2)
        assert ar.ms < 5000
        for r in range(n):
            assert not ar.measured[r] and ar.ns_median[r] is None and ar.status[r] == ERR_UNSUPPORTED


def test_repeated_calls_stay_exact_and_disturb_nothing(pkg, oracle):
    n, nbytes = 3, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        bpp = p.Info().bytes_per_pair
        one = p.AllReduce(reps=2)
        ts = p.AllReduceTwoShot(reps=2)
        ll = p.AllReduceLL(reps=2)
        aa = p.AllToAll(reps=2)
        r1 = p.Run()
        diags = [(i, j, p.Diagnose("write", i, j)) for i, j in ((0, 1), (2, 0))]
        for c in range(1, 7):
            ring = check(p.AllReduceRing(reps=1 + c % 3), n, bpp, 1 + c % 3)
            assert ring.call_seq == c
        for i, j, d in diags:
            d2 = p.Diagnose("write", i, j)
            assert (d2.bad_words, d2.run_seq, d2.region_offset) == (0, r1.run_seq, d.region_offset)
        one2 = p.AllReduce(reps=2)
        assert one2.call_seq == 2 and [getattr(one2, f) for f in PER_ROW + ("status",)] == \
            [getattr(one, f) for f in PER_ROW + ("status",)]
        ts2 = p.AllReduceTwoShot(reps=2)
        assert ts2.call_seq == 2 and [getattr(ts2, f) for f in PER_ROW] == [getattr(ts, f) for f in PER_ROW]
        ll2 = p.AllReduceLL(reps=2)
        assert ll2.call_seq == 2 and [getattr(ll2, f) for f in PER_ROW] == [getattr(ll, f) for f in PER_ROW]
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
        check(p.AllReduceRing(reps=2), n, bpp, 2)


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
        out = {"calls": [dump(p.AllReduceRing(reps=2)), dump(p.AllReduceRing(reps=3))]}
        rc, t = p.allreduce_ring_raw(2 + rank)  # the processes disagree
        out["mismatch"] = {"rc": rc, "call_seq": t.call_seq, "measured": sum(t.measured)}
        out["after"] = dump(p.AllReduceRing(reps=2))
        out["one_shot"] = dump(p.AllReduce(reps=2))
        r = p.Run(gather=True)
        out["run"] = {"reach": r.reach, "aborted": r.aborted}
    print("RESULT " + json.dumps(out))
    """
) % ROOT


@pytest.mark.parametrize("n_local", [1, 2], ids=["2x1", "2x2"])
def test_two_processes_agree_and_fill_their_own_rows(pkg, n_local):
    """Both processes drive GPU 0 with 8 and 3 CTAs per rank; their contexts are time-sliced, so the times only need to
    be positive."""
    world = 2
    n = world * n_local
    outs = run_children(CHILD, world, n_local)
    sizes = allreduce_ref.ladder(pkg.plan(n, 1 << 20, MODE_SLICED).bytes_per_pair)
    expect = [list(sx) for sx in allreduce_ref.expected(SEED, n, tuple(sizes))]
    ns = len(sizes)
    for rank, o in enumerate(outs):
        mine = set(range(rank * n_local, (rank + 1) * n_local))
        assert [c["call_seq"] for c in o["calls"]] + [o["after"]["call_seq"]] == [1, 2, 3]
        assert o["mismatch"] == {"rc": ERR_ARG, "call_seq": 0, "measured": 0}
        for c in o["calls"] + [o["after"]]:
            assert c["row_mask"] == sum(1 << r for r in mine) and c["sizes"] == sizes and c["path"] == PATH_RING
            for r in range(n):
                assert c["measured"][r] == (r in mine), r
                if r in mine:
                    assert c["status"][r] == 0 and c["bad_sizes"][r] == 0 and all(t > 0 for t in c["ns_min"][r])
                    assert [[s, x] for s, x in zip(c["sum"][r], c["xr"][r])] == expect, r
                    assert c["bad_words"][r] == [0] * ns and c["first_bad"][r] == [U64_MAX] * ns
                    for f in PER_ROW:
                        assert c[f][r] == o["one_shot"][f][r], (r, f)
                else:
                    assert c["sum"][r] is None
        assert o["run"]["reach"] == [[1] * n for _ in range(n)] and not o["run"]["aborted"]
