"""allreduce_nvls_kernel run as N ranks on one H100, with its two multicast instructions emulated by unicast loads and
stores (tests/nvls_emulate.py, tests/c/nvls_emulate.cuh), checked word for word against numpy.

A multicast object needs a team of devices, so on one GPU cdprobe_allreduce_nvls itself never runs its data path.  Most
of the kernel does not depend on multicast: the chunk walk over twoshot_chunk, the per-lane vector layout, partial
units, the fault's placement, the two fenced domain barriers per rep and the word check and clear through the unicast
output.  Those run here, unchanged, with every rep of every size compared.  What stays unexercised: the two real
instructions and the in-switch sum, fence.proxy.alias (it runs, but every access goes through one mapping), the
creation, binding and mapping of the multicast object, and the export and import of its handle.

The harness runs in a child process with 32 hardware queues, so every rank's stream has one; every CTA of every rank
is resident at once (the harness refuses more CTAs than multiprocessors).  Emulated times are checked only for order.
NVLS_EMULATE_MUTATION, when set, builds the copy with one of nvls_emulate.MUTATIONS applied."""
import contextlib
import functools
import os

import numpy as np
import pytest

import allreduce_nvls_ref as ref
import allreduce_ref
import large_ref
import nvls_emulate as emu
import word_ref
from test_large_regions_gpu import MODE_SLICED, SPARE, VMM, alloc_bytes, round_up

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
U64_MAX = word_ref.U64_MAX
UNIT_WORDS = ref.UNIT_WORDS
GIB = 1 << 30
EDGE_BPP = 57 * 8192 + 384  # a partial last unit in a partial last granule
BPPS = [128, 4224, 16512, 24704, EDGE_BPP, (4 << 20) + 384]
NS = [1, 2, 3, 5, 8, 16]
BIG_BPP = (4 << 30) + 8192 + 128  # the last unit 128 B, the last size past 2^32
HEADROOM = 4 * GIB


@pytest.fixture(scope="module")
def remote(tmp_path_factory):
    lib, _ = emu.build(tmp_path_factory.mktemp("nvls_emulate"), os.environ.get("NVLS_EMULATE_MUTATION") or None)
    with emu.Remote(lib) as r:
        yield r


@pytest.fixture(scope="module")
def sms(remote):
    return remote.device()["sms"]


@contextlib.contextmanager
def opened(remote, n, grids, bpp):
    h = remote.open(n, list(grids), bpp, SEED)
    try:
        yield h
    finally:
        remote.close(h)


def grid_sets(n, sms):
    """Per-rank grids: 1, 2, 3 and 7 CTAs each, the largest equal grid that fits, and unequal grids 1, 8, 3, ..."""
    out = [[g] * n for g in (1, 2, 3, 7, sms // n) if g * n <= sms]
    out.append([(1, 8, 3)[i % 3] for i in range(n)])
    return [g for i, g in enumerate(out) if g not in out[:i]]


@functools.lru_cache(maxsize=None)
def clean(n, n_words):
    w = allreduce_ref.output_words(SEED, n, n_words)
    w.setflags(write=False)
    return w


@functools.lru_cache(maxsize=None)
def src(rank, n_words):
    w = word_ref.src_words(SEED, rank, 0, n_words)
    w.setflags(write=False)
    return w


def check(rows, n, sizes, reps, held, bad_words, first_bad):
    """held(k, r): the words every row's output holds after rep r (0: the warm-up) of size k; bad_words[k] and
    first_bad[k] (a word index or None) the word check over every rep of size k.  No row aborts, and in every rep the
    opening release precedes the closing one, which precedes the next rep's opening."""
    assert len(rows) == n
    want = [[allreduce_ref.checksum(held(k, r)) for r in range(reps + 1)] for k in range(len(sizes))]
    for i, row in enumerate(rows):
        assert row["abort"] == 0, i
        for k, s in enumerate(sizes):
            got = list(zip(row["sum"][k], row["xr"][k]))
            assert got == want[k], (i, s, [r for r in range(reps + 1) if got[r] != want[k][r]])
            assert row["bad_words"][k] == bad_words[k], (i, s, row["bad_words"][k], bad_words[k])
            assert row["first_bad"][k] == (U64_MAX if first_bad[k] is None else 8 * first_bad[k]), (i, s)
            t_rel, t_end = row["t_rel"][k], row["t_end"][k]
            assert all(t_rel[r] < t_end[r] for r in range(reps + 1)), (i, s, t_rel, t_end)
            assert all(t_end[r] <= t_rel[r + 1] for r in range(reps)), (i, s, t_rel, t_end)


def check_clean(rows, n, sizes, reps):
    W = sizes[-1] // 8
    check(rows, n, sizes, reps, lambda k, r: clean(n, W)[:sizes[k] // 8], [0] * len(sizes), [None] * len(sizes))


def check_fault(rows, n, sizes, reps, fault):
    """fault (mode, k, word) acted in timed rep 1 of size k only: that rep's output is the restatement's, and the
    word check counts its failing words once."""
    mode, fk, word = fault
    W = sizes[-1] // 8
    s = sizes[fk]
    hit = ref.rep([src(j, W)[:s // 8] for j in range(n)], s, (mode, word))[0]
    failing = ref.failing([src(j, W)[:s // 8] for j in range(n)], s, (mode, word))
    words = failing.get(0, [])
    assert sorted(failing) == (list(range(n)) if words else [])
    bad = [len(words) if k == fk else 0 for k in range(len(sizes))]
    first = [words[0] if k == fk and words else None for k in range(len(sizes))]
    check(rows, n, sizes, reps, lambda k, r: hit if (k, r) == (fk, 1) else clean(n, W)[:sizes[k] // 8], bad, first)
    return words


# ---- clean ladders --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bpp", BPPS)
@pytest.mark.parametrize("n", NS)
def test_clean_ladders_on_every_grid(remote, sms, n, bpp):
    """Every rep of every size equals the checksum of the clean sum, on small, odd, full and unequal grids.  bpp 128 at
    N = 16 leaves 15 chunks empty; N = 5 over 4224 B splits its one unit unevenly."""
    sizes = allreduce_ref.ladder(bpp)
    for grids in grid_sets(n, sms):
        with opened(remote, n, grids, bpp) as h:
            for seq, reps in ((1, 1), (2, 3)):
                check_clean(remote.call(h, sizes, reps, call_seq=seq), n, sizes, reps)


# ---- the same rows as the one-shot --------------------------------------------------------------------------------
@pytest.mark.parametrize("bpp", [1 << 20, GIB], ids=["1MiB", "1GiB"])
@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_the_same_rows_as_the_one_shot_on_a_real_handle(pkg, remote, sms, n, bpp):
    """cdprobe_allreduce of a handle of N ranks on one device, with the same seed and bytes per pair, reports the same
    sum, xr, bad_words and first_bad in every row as the emulated kernel's last timed rep."""
    # the handle is closed before the emulated ranks open, so the larger of the two needs applies: the handle's
    # allocations from its plan plus the one-shot's output in each rank's scratch, or the emulated NVLS areas
    handle = n * (alloc_bytes(pkg, n, bpp * max(n - 1, 1), MODE_SLICED, SAME) + round_up(bpp, VMM) + SPARE)
    need = max(handle, n * (2 * bpp + (1 << 20)))
    free = remote.device()["free"]
    if free < need + HEADROOM:
        pytest.skip(f"needs {need} bytes plus {HEADROOM} spare on the device; {free} free")
    reps = 2
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=bpp * max(n - 1, 1), flags=SAME, ctas=8,
                             timeout_ms=60000)) as p:
        assert p.Info().bytes_per_pair == bpp
        one = p.AllReduce(reps=reps)
    sizes = allreduce_ref.ladder(bpp)
    assert one.sizes == sizes and one.status == [0] * n
    with opened(remote, n, [min(16, sms // n)] * n, bpp) as h:
        rows = remote.call(h, sizes, reps)
    for r, row in enumerate(rows):
        assert row["abort"] == 0
        assert [row["sum"][k][reps] for k in range(len(sizes))] == one.sum[r], r
        assert [row["xr"][k][reps] for k in range(len(sizes))] == one.xr[r], r
        assert row["bad_words"] == one.bad_words[r] == [0] * len(sizes), r
        assert row["first_bad"] == one.first_bad[r] == [U64_MAX] * len(sizes), r


# ---- faults -------------------------------------------------------------------------------------------------------
def fault_places(sizes, n, grid):
    """(k, word): word 0; an even and an odd word of one 16-byte vector (lane 5's second vector of unit 1, or of unit 0
    when there is one unit); the first and last word of every rank's chunk, the last of the last rank's being the last
    word of a partial unit; a word of the unit the last warp of the word-0 owner's grid takes first; and the last word
    of a size below the largest."""
    K = len(sizes) - 1
    W, U = sizes[K] // 8, ref.units(sizes[K])
    u = min(1, U - 1)
    vec = u * UNIT_WORDS + (16 * 5 + 512) // 8
    out = [(K, 0), (K, vec), (K, vec + 1)]
    for r in range(n):
        lo, hi = U * r // n, U * (r + 1) // n
        if hi > lo:
            out += [(K, lo * UNIT_WORDS), (K, min(hi * UNIT_WORDS, W) - 1)]
    o = ref.owner(U, n, 0)
    last_warp = U * o // n + 8 * grid - 1
    if last_warp < U * (o + 1) // n:
        out.append((K, last_warp * UNIT_WORDS + 7))
    if K >= 2:
        out.append((K - 2, sizes[K - 2] // 8 - 1))
    return [p for i, p in enumerate(out) if p not in out[:i]]


@pytest.mark.parametrize("n, bpp, grid", [(1, EDGE_BPP, 2), (2, (4 << 20) + 384, 8), (3, EDGE_BPP, 2),
                                          (5, (4 << 20) + 384, 3), (16, EDGE_BPP, 1)])
def test_each_fault_fails_exactly_the_words_the_restatement_names(remote, n, bpp, grid):
    """Mode 0 stores one word xored with 1, mode 1 skips the store of one unit, in timed rep 1 only, in the word's
    owner.  At reps = 1 the failing words, first_bad and the last (S, X) are the restatement's; at reps = 3 only rep 1's
    (S, X) differs, so a mode-1 unit reads as 0 only in that rep: the clear after every rep works.  The next call is
    clean."""
    sizes = allreduce_ref.ladder(bpp)
    seq = 0
    with opened(remote, n, [grid] * n, bpp) as h:
        for mode in (0, 1):
            for k, word in fault_places(sizes, n, grid):
                for reps in (1, 3):
                    seq += 1
                    rows = remote.call(h, sizes, reps, fault=(mode, k, word), call_seq=seq)
                    words = check_fault(rows, n, sizes, reps, (mode, k, word))
                    assert words and (mode == 1 or words == [word]), (mode, k, word)
                seq += 1
                check_clean(remote.call(h, sizes, 2, call_seq=seq), n, sizes, 2)


@pytest.mark.parametrize("n", [2, 5])
def test_a_fault_handed_to_a_rank_that_does_not_own_the_word_changes_nothing(remote, n):
    """Only the word's owner reduces and stores its unit, so the host must hand the fault to twoshot_owner's rank, as
    cdprobe_allreduce_nvls does: any other rank never meets the word."""
    bpp = EDGE_BPP
    sizes = allreduce_ref.ladder(bpp)
    K, U = len(sizes) - 1, ref.units(bpp)
    seq = 0
    with opened(remote, n, [2] * n, bpp) as h:
        for mode in (0, 1):
            for word in (0, bpp // 16, bpp // 8 - 1):
                o = ref.owner(U, n, word // UNIT_WORDS)
                for other in sorted({(o + 1) % n, (o + n - 1) % n}):
                    seq += 1
                    rows = remote.call(h, sizes, 1, fault=(mode, K, word), fault_rank=other, call_seq=seq)
                    check_clean(rows, n, sizes, 1)
                seq += 1
                check_fault(remote.call(h, sizes, 1, fault=(mode, K, word), call_seq=seq), n, sizes, 1, (mode, K, word))


# ---- corruption at rest ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [2, 5])
def test_a_word_corrupted_at_rest_fails_every_rep_of_every_size_that_covers_it(remote, n):
    """One rank's input word flipped in the partial last unit, or at the edge between two ranks' chunks: every row
    fails that word in every rep, the warm-up included, at every size that holds it, and (S, X) is the sum at rest.
    After the restore the call is clean."""
    bpp, reps = EDGE_BPP, 2
    sizes = allreduce_ref.ladder(bpp)
    W, U = bpp // 8, ref.units(bpp)
    edge = (U * 1 // n) * UNIT_WORDS  # the first word of rank 1's chunk at the largest size
    seq = 0
    with opened(remote, n, [3] * n, bpp) as h:
        for j, w, mask in ((n - 1, W - 3, 1 << 17), (0, edge, 1 << 63), (n // 2, edge - 1, 1)):
            remote.corrupt(h, j, w, mask)
            seq += 1
            rows = remote.call(h, sizes, reps, call_seq=seq)
            at_rest = clean(n, W).copy()
            o = int(src(j, W)[w])
            at_rest[w] = np.uint64((int(at_rest[w]) - o + (o ^ mask)) % (1 << 64))
            covers = [w < s // 8 for s in sizes]
            check(rows, n, sizes, reps, lambda k, r: at_rest[:sizes[k] // 8],
                  [(reps + 1) if c else 0 for c in covers], [w if c else None for c in covers])
            remote.corrupt(h, j, w, mask)  # restore
            seq += 1
            check_clean(remote.call(h, sizes, reps, call_seq=seq), n, sizes, reps)


# ---- several contexts ---------------------------------------------------------------------------------------------
def test_contexts_called_in_turn_each_use_their_own_members(remote):
    """The member tables are one per module: each call loads its own context's, so a context called after another was
    opened, called and closed still sums and stores through its own areas."""
    bpp_a, bpp_b = EDGE_BPP, (4 << 20) + 384
    sizes_a, sizes_b = allreduce_ref.ladder(bpp_a), allreduce_ref.ladder(bpp_b)
    with opened(remote, 2, [3, 3], bpp_a) as a:
        check_clean(remote.call(a, sizes_a, 1, call_seq=1), 2, sizes_a, 1)
        with opened(remote, 3, [2, 2, 2], bpp_b) as b:
            check_clean(remote.call(a, sizes_a, 2, call_seq=2), 2, sizes_a, 2)
            check_clean(remote.call(b, sizes_b, 1, call_seq=1), 3, sizes_b, 1)
            check_clean(remote.call(a, sizes_a, 1, call_seq=3), 2, sizes_a, 1)
        check_clean(remote.call(a, sizes_a, 3, call_seq=4), 2, sizes_a, 3)


# ---- repeated calls -------------------------------------------------------------------------------------------------
def test_repeated_calls_on_one_context_stay_exact(remote):
    """Calls with rising call_seq and varying reps on the same barrier lines: the lines only ever rise, so every call
    must pass each barrier on its own values, never on an earlier call's."""
    n, bpp = 5, EDGE_BPP
    sizes = allreduce_ref.ladder(bpp)
    with opened(remote, n, [1, 8, 3, 2, 7], bpp) as h:
        for seq in range(1, 9):
            reps = 1 + seq % 4
            check_clean(remote.call(h, sizes, reps, call_seq=seq), n, sizes, reps)


# ---- past 2^32 ------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def big_sums(n):
    return tuple(large_ref.allreduce_sums(SEED, n, allreduce_ref.ladder(BIG_BPP)))


@pytest.mark.parametrize("n", [1, 2])
def test_every_size_past_2_32_and_a_corrupted_word_there(remote, sms, n):
    """At 4 GiB + 8 KiB + 128 per rank every size is clean against the streamed reference; a word past byte 2^32
    corrupted at rest fails only the last size, with its byte offset as first_bad.  The fault option's word has 24
    bits, so a fault cannot name a word past 2^32 and none is placed there."""
    need = n * (2 * BIG_BPP + (1 << 20))
    free = remote.device()["free"]
    if free < need + HEADROOM:
        pytest.skip(f"needs {need} bytes plus {HEADROOM} spare on the device; {free} free")
    sizes = allreduce_ref.ladder(BIG_BPP)
    assert sizes[-2] == 1 << 32
    want = big_sums(n)
    reps = 1
    word, mask, j = (1 << 29) + 3, 1 << 21, n - 1
    with opened(remote, n, [sms // n] * n, BIG_BPP) as h:
        rows = remote.call(h, sizes, reps, call_seq=1)
        for i, row in enumerate(rows):
            assert row["abort"] == 0
            for k in range(len(sizes)):
                assert [(row["sum"][k][r], row["xr"][k][r]) for r in range(reps + 1)] == \
                    [(want[k].sum, want[k].xr)] * (reps + 1), (i, sizes[k])
            assert row["bad_words"] == [0] * len(sizes) and row["first_bad"] == [U64_MAX] * len(sizes), i
        remote.corrupt(h, j, word, mask)
        rows = remote.call(h, sizes, reps, call_seq=2)
        remote.corrupt(h, j, word, mask)  # restore
    # the corrupted output word changes the last size's (S, X) by its difference, in its granule
    total = sum(int(word_ref.src_words(SEED, q, word, 1)[0]) for q in range(n)) % (1 << 64)
    o = int(word_ref.src_words(SEED, j, word, 1)[0])
    new = (total - o + (o ^ mask)) % (1 << 64)
    rot = word_ref.fold6(word // word_ref.GRANULE_WORDS)
    d = total ^ new
    last = ((want[-1].sum - total + new) % (1 << 64),
            want[-1].xr ^ (((d << rot) | (d >> (64 - rot))) & U64_MAX if rot else d))
    for i, row in enumerate(rows):
        assert row["abort"] == 0
        for k in range(len(sizes) - 1):
            assert (row["sum"][k][reps], row["xr"][k][reps]) == (want[k].sum, want[k].xr), (i, sizes[k])
        assert [(row["sum"][-1][r], row["xr"][-1][r]) for r in range(reps + 1)] == [last] * (reps + 1), i
        assert row["bad_words"] == [0] * (len(sizes) - 1) + [reps + 1], i
        assert row["first_bad"] == [U64_MAX] * (len(sizes) - 1) + [8 * word], i
