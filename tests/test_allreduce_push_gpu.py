"""cdprobe_allreduce_push on the GPU: every row's output at every size is the pattern's sum, word for word and in
(S, X), on all three data paths, and equals the one-shot's and the two-shot's on the same handle; 2 to 16 ranks that
share one device add into the same units at once (the contended-reduction case); tiny ladders where some ranks own no
unit, a partial last unit, small and unequal grids; a word corrupted at rest fails exactly the sizes that cover it in
every row; an altered, skipped or doubled reduction and a corrupted all-gather push fail exactly the rows and words the
restatement names (allreduce_push_ref); armed faults that name nothing are refused with their exact text; a mapping that
is down stops every rank without waiting; two processes agree; repeated calls stay exact and disturb nothing.  Several
ranks share one device where a test needs N > 1.  No test drives a kernel past its deadline.

Not covered here: the refusal of a domain whose devices lack native peer atomics (cudaDevP2PAttrNativeAtomicSupported)
needs two GPUs, and every rank of these tests shares one device, which is atomic with itself."""
import functools
import textwrap

import numpy as np
import pytest

import allreduce_push_ref as ref
import allreduce_ref
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
PATHS = [0, 1, 2]
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


def check(ar, n, bpp, reps, path, corrupt=None, fault=None):
    """Every row at every size, from the words at rest: corrupt {(rank, word): mask} is xored into the sources, and
    fault (mode, rank, k, word) acts in timed rep 1 only.  bad_words count every rep, warm-up included; (S, X) is the
    last timed rep's."""
    corrupt = corrupt or {}
    sizes = allreduce_ref.ladder(bpp)
    assert ar.sizes == sizes and ar.reps == reps and ar.n == n and ar.path == path
    W = bpp // 8
    srcs = [src(j, W).copy() for j in range(n)]
    for (j, w), m in corrupt.items():
        srcs[j][w] ^= np.uint64(m)
    clean = sum(src(j, W) for j in range(n))
    at_rest = sum(srcs[1:], srcs[0].copy())
    hits = {}
    if fault is not None:
        mode, rank, k, word = fault
        hits = dict(enumerate(ref.rep([s[:sizes[k] // 8] for s in srcs], sizes[k], (mode, rank, word))))
    for r in range(n):
        bits = 0
        for k, s in enumerate(sizes):
            rep_words = at_rest[:s // 8]
            bad = np.flatnonzero(rep_words != clean[:s // 8])
            n_bad, first = (reps + 1) * len(bad), [int(bad[0])] if len(bad) else []
            last = rep_words
            if fault is not None and fault[2] == k:
                hit = hits[r]
                hbad = np.flatnonzero(hit != clean[:s // 8])
                n_bad += len(hbad) - len(bad)
                first += [int(hbad[0])] if len(hbad) else []
                if len(hbad) or (hit != rep_words).any():
                    bits |= 1 << k
                if reps == 1:
                    last = hit
            if len(bad):
                bits |= 1 << k
            ctx = (r, s, path, fault)
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


def assert_rows_equal(push, other):
    for r in range(push.n):
        assert push.status[r] == other.status[r] and push.measured[r] == other.measured[r], r
        assert push.bad_sizes[r] == other.bad_sizes[r], r
        for f in PER_ROW:
            assert getattr(push, f)[r] == getattr(other, f)[r], (r, f)


def want(oracle, n, sizes):
    small = tuple(s for s in sizes if s <= REF_MAX)
    got = dict(zip(small, allreduce_ref.expected(SEED, n, small))) if small else {}
    for s in sizes:
        if s not in got:
            assert n == 1, "only the single-rank output is checked against the oracle beyond REF_MAX"
            got[s] = oracle.src_checksum(SEED, 0, 0, s // 8)
    return [got[s] for s in sizes]


def set_path(pkg, p, path):
    p.SetOption(pkg.abi.OPT_PATH, path)


@pytest.mark.parametrize("path", PATHS)
def test_single_rank_every_size_of_a_1_gib_ladder_clean(pkg, oracle, path):
    """At N = 1 the rank reduces its input into its own zeroed area, and the all-gather has no targets.  A 1 GiB rep
    reads its 1 GiB input, and each bulk reduction (or red.global) makes the memory system read and write the area's
    1 GiB: 3 GiB through HBM (allreduce_push_kernel at n == 1: reduce_tma / reduce_ldst, then no ar_units pass)."""
    with pkg.Open(pkg.Config(ordinals=[0], bytes=GIB, timeout_ms=60000)) as p:
        set_path(pkg, p, path)
        ar = p.AllReducePush(reps=2)
        assert ar.sizes == allreduce_ref.ladder(GIB) and ar.path == path and ar.call_seq == 1
        assert ar.measured[0] and ar.status[0] == 0 and ar.bad_sizes[0] == 0
        assert [(s, x) for s, x in zip(ar.sum[0], ar.xr[0])] == want(oracle, 1, ar.sizes)
        assert ar.bad_words[0] == [0] * len(ar.sizes) and ar.first_bad[0] == [U64_MAX] * len(ar.sizes)
        assert_fits_in_call(ar)
        assert_hbm_floor(ar, 3 * GIB)


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 8, 16])
def test_every_row_exact_and_equal_to_the_one_shot_and_the_two_shot(pkg, n, path):
    """Every sender adds into every owner's units at once: up to 16 ranks reduce into the same 8 KiB unit together."""
    with open_same(pkg, n) as p:
        set_path(pkg, p, path)
        bpp = p.Info().bytes_per_pair
        push = check(p.AllReducePush(reps=2), n, bpp, 2, path)
        assert (push.row_mask, push.call_seq) == ((1 << n) - 1, 1)
        assert_rows_equal(push, p.AllReduceTwoShot(reps=2))
        one = p.AllReduce(reps=2)
        for r in range(n):
            assert (push.sum[r], push.xr[r], push.bad_words[r], push.first_bad[r]) == \
                (one.sum[r], one.xr[r], one.bad_words[r], one.first_bad[r]), r


@pytest.mark.parametrize("bpp", [128, 4224, 16512, 24704, EDGE_BPP])
@pytest.mark.parametrize("n", [3, 5])
def test_tiny_ladders_where_ranks_own_no_unit_and_a_partial_last_unit(pkg, n, bpp):
    with open_bpp(pkg, n, bpp) as p:
        for path in PATHS:
            set_path(pkg, p, path)
            check(p.AllReducePush(reps=1), n, bpp, 1, path)
            check(p.AllReducePush(reps=3), n, bpp, 3, path)


GRIDS = [("ctas", 1), ("ctas", 2), ("ctas", 3), ("ctas", 7), ("ctas", 40), ("rank", (1, 8, 3)),
         ("rank", (7, 2, 5)), ("rank", (40, 1, 1))]


@pytest.mark.parametrize("grid", GRIDS, ids=[f"{g[0]}{'-'.join(map(str, g[1])) if g[0] == 'rank' else g[1]}"
                                             for g in GRIDS])
def test_every_grid_finishes_exact(pkg, grid):
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
        for path in PATHS:
            set_path(pkg, p, path)
            check(p.AllReducePush(reps=1), n, bpp, 1, path)
            check(p.AllReducePush(reps=4), n, bpp, 4, path)


def test_a_corrupt_word_fails_exactly_the_sizes_that_cover_it_in_every_row(pkg):
    n, bpp = 3, EDGE_BPP
    W = bpp // 8
    with open_bpp(pkg, n, bpp) as p:
        for path in PATHS:
            set_path(pkg, p, path)
            for j, w in ((2, 5), (0, 40000), (1, W - 1)):
                p.Corrupt(j, 8 * w, 1 << 17)
                check(p.AllReducePush(reps=2), n, bpp, 2, path, corrupt={(j, w): 1 << 17})
                p.Corrupt(j, 8 * w, 1 << 17)  # restore
            check(p.AllReducePush(reps=1), n, bpp, 1, path)


def fault_cases(n, sizes):
    """(mode, rank, k, word) for every mode the domain allows, at a few sizes and places."""
    out = []
    last = len(sizes) - 1
    for mode in (0, 1, 2, 3):
        if mode == 3 and n == 1:
            continue
        for rank, k, at in ((n - 1, last, 0.3), (0, 0, 0.99), (n // 2, max(last - 2, 0), 0.0)):
            W = sizes[k] // 8
            word = min(int(W * at), W - 1)
            if mode == 3 and ref.word_owner(sizes[k], n, word) == rank:
                rank = (ref.word_owner(sizes[k], n, word) + 1) % n
            out.append((mode, rank, k, word))
    return out


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("n", [1, 2, 3, 8])
def test_each_fault_fails_exactly_the_rows_and_words_the_restatement_names(pkg, n, path):
    """Modes 0-2 change a sender's contribution, so every row fails at the word (mode 0) or at the unit's words whose
    source word is not 0 (modes 1 and 2); mode 3 changes one all-gather push, so only its receiver's row fails.  With
    reps == 1 the word check and the last (S, X) see it; with 3 reps the summed bad words and rep 1's (S, X) do.  The
    area is cleared after every rep, so only size[k] fails, and the next call is clean."""
    a = pkg.abi
    with open_same(pkg, n) as p:
        set_path(pkg, p, path)
        bpp = p.Info().bytes_per_pair
        sizes = allreduce_ref.ladder(bpp)
        W = bpp // 8
        for f in fault_cases(n, sizes):
            mode, rank, k, word = f
            p.SetOption(a.OPT_ALLREDUCE_PUSH_FAULT, a.allreduce_push_fault(rank, k, word, mode))
            ar = check(p.AllReducePush(reps=1), n, bpp, 1, path, fault=f)
            rows = ref.failing([src(j, W)[:sizes[k] // 8] for j in range(n)], sizes[k], (mode, rank, word))
            assert [r for r in range(n) if ar.bad_sizes[r]] == sorted(rows), f
            for r, words in rows.items():
                assert ar.bad_sizes[r] == 1 << k and ar.bad_words[r][k] == len(words), (f, r)
                assert ar.first_bad[r][k] == 8 * words[0], (f, r)
            check(p.AllReducePush(reps=3), n, bpp, 3, path, fault=f)
        p.SetOption(a.OPT_ALLREDUCE_PUSH_FAULT, 0)
        check(p.AllReducePush(reps=2), n, bpp, 2, path)


NO_MODE = "the armed push all-reduce fault has a mode above 3"
NO_RANK = "the armed push all-reduce fault names no rank of this domain"
NO_SIZE = "the armed push all-reduce fault names no size of this call"
NO_WORD = "the armed push all-reduce fault names no output word of its size"
NO_PEER = "the armed push all-reduce fault's mode 3 has no peer to push to at n == 1"
OWNER = "the armed push all-reduce fault's mode-3 receiver owns the word and is pushed no copy of it"


def test_an_armed_fault_that_names_nothing_is_refused_with_its_text(pkg):
    a = pkg.abi
    n = 3
    with open_same(pkg, n) as p:
        bpp = p.Info().bytes_per_pair
        sizes = allreduce_ref.ladder(bpp)
        ar = check(p.AllReducePush(reps=2), n, bpp, 2, 0)
        last = sizes[-1]
        owned = ref.word_owner(last, n, 0)
        bad = [((4 << 48) | a.allreduce_push_fault(0, 0, 0), NO_MODE),
               ((1 << 63) | a.allreduce_push_fault(0, 0, 0), NO_MODE),
               (a.allreduce_push_fault(n, 0, 0), NO_RANK),
               ((1 << 24) | 5, NO_RANK),
               (a.allreduce_push_fault(0, len(sizes), 0), NO_SIZE),
               (a.allreduce_push_fault(1, 0, sizes[0] // 8), NO_WORD),
               (a.allreduce_push_fault(owned, len(sizes) - 1, 0, mode=3), OWNER)]
        for v, message in bad:
            p.SetOption(a.OPT_ALLREDUCE_PUSH_FAULT, v)
            rc, t = p.allreduce_push_raw(2)
            assert rc == ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0, hex(v)
            assert p._lib.cdprobe_last_error().decode() == message, hex(v)
        p.SetOption(a.OPT_ALLREDUCE_PUSH_FAULT, 0)
        ar2 = check(p.AllReducePush(reps=2), n, bpp, 2, 0)
        assert ar2.call_seq == ar.call_seq + 1
        rc, t = p.allreduce_push_raw(a.ALLREDUCE_MAX_REPS + 1)
        assert rc == ERR_ARG and (t.abi, t.n, t.reps, t.call_seq, t.row_mask, t.path) == (2, n, 65, 0, 0, 0)
    with pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 20, timeout_ms=20000)) as p:  # n = 1 pushes nothing
        p.SetOption(a.OPT_ALLREDUCE_PUSH_FAULT, a.allreduce_push_fault(0, 0, 0, mode=3))
        rc, t = p.allreduce_push_raw(2)
        assert rc == ERR_ARG and t.call_seq == 0 and p._lib.cdprobe_last_error().decode() == NO_PEER


def test_a_mapping_that_is_down_stops_every_rank_until_it_is_remapped(pkg):
    n = 4
    with open_same(pkg, n) as p:
        bpp = p.Info().bytes_per_pair
        check(p.AllReducePush(reps=2), n, bpp, 2, 0)  # builds the push area with every mapping up
        p.UnmapPeer(2, 1)
        ar = p.AllReducePush(reps=2)
        assert ar.call_seq == 2 and ar.ms < 5000  # returned without waiting for a watchdog
        for r in range(n):
            assert not ar.measured[r] and ar.status[r] == ERR_STATE and ar.ns_median[r] is None
        p.RemapPeer(2, 1)
        assert check(p.AllReducePush(reps=2), n, bpp, 2, 0).call_seq == 3


def test_an_unmapped_peer_before_the_first_call_keeps_the_push_all_reduce_off_until_reopened(pkg):
    n = 3
    with open_same(pkg, n) as p:
        p.UnmapPeer(0, 2)
        for remap in (False, True):
            if remap:
                p.RemapPeer(0, 2)  # the probe mapping is back, but the push area was built without it
            ar = p.AllReducePush(reps=2)
            assert ar.ms < 5000
            for r in range(n):
                assert not ar.measured[r] and ar.status[r] != 0, (remap, r)
    with open_same(pkg, n) as p:
        check(p.AllReducePush(reps=2), n, p.Info().bytes_per_pair, 2, 0)


def test_simulated_mig_runs_no_rank(pkg):
    n = 2
    with open_same(pkg, n, flags=SIMULATE_MIG) as p:
        ar = p.AllReducePush(reps=2)
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
        ring = p.AllReduceRing(reps=2)
        aa = p.AllToAll(reps=2)
        r1 = p.Run()
        diags = [(i, j, p.Diagnose("write", i, j)) for i, j in ((0, 1), (2, 0))]
        for c in range(1, 7):
            set_path(pkg, p, c % 3)
            push = check(p.AllReducePush(reps=1 + c % 3), n, bpp, 1 + c % 3, c % 3)
            assert push.call_seq == c
        set_path(pkg, p, 0)
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
        ring2 = p.AllReduceRing(reps=2)
        assert ring2.call_seq == 2 and [getattr(ring2, f) for f in PER_ROW] == [getattr(ring, f) for f in PER_ROW]
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
        assert check(p.AllReducePush(reps=2), n, bpp, 2, 0).call_seq == 7


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
        out = {"calls": [dump(p.AllReducePush(reps=2))]}
        p.SetOption(m.abi.OPT_PATH, 1)
        out["calls"].append(dump(p.AllReducePush(reps=3)))
        rc, t = p.allreduce_push_raw(2 + rank)  # the processes disagree
        out["mismatch"] = {"rc": rc, "call_seq": t.call_seq, "measured": sum(t.measured)}
        out["after"] = dump(p.AllReducePush(reps=2))
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
        assert [c["path"] for c in o["calls"]] + [o["after"]["path"]] == [0, 1, 1]
        assert o["mismatch"] == {"rc": ERR_ARG, "call_seq": 0, "measured": 0}
        for c in o["calls"] + [o["after"]]:
            assert c["row_mask"] == sum(1 << r for r in mine) and c["sizes"] == sizes
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
