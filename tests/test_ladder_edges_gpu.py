"""The ladder measurements (cdprobe_bwcurve, cdprobe_allreduce, cdprobe_alltoall, cdprobe_memcpy) where their kernels
go wrong, checked word for word against the numpy references (bwcurve_ref, allreduce_ref, alltoall_ref, memcpy_ref,
word_ref) on every data path:

- tiny ladders: bytes_per_pair below one 8 KiB unit, below the ladder's 4096-byte minimum, exactly one ladder step, one
  128-byte vector past a unit, one 16 KiB granule and one vector past it, and a partial unit in the second granule.
  These run the partial-unit branches (a 128-byte TMA bulk copy, 32-byte ld/st with 4 of 32 lanes active) and the
  expected sums with no whole granule;
- grids of 1, 2, 3 and 7 CTAs per rank, the full grid at N = 1, and unequal per-rank grids (OPT_CTAS_RANK), which
  change which warp walks which unit;
- faults placed at the edges: the all-reduce's at word 0 of size 0 and at the last word of the last, partial unit,
  each as a word off by one and as a unit not stored;
  the all-to-all's at the last word of a partial unit, at a word of the last warp of the grid and on the diagonal
  block; memcpy's at word 0 of size 0, at the last word of the last, partial unit and on the diagonal cell, each
  flipped and dropped; and a corrupted source word in a partial unit, which fails exactly the bwcurve cell and sizes
  that read it, every all-reduce row at those sizes, exactly the memcpy cells and sizes that copy it (pulled and
  pushed), and no all-to-all cell.

Memcpy's checks run diag_launch and bwcurve_kernel on the issuer's grid over a destination in the exchange area, so
its tiny ladders and small grids reach the same partial-unit branches.  The copy-engine all-to-all's owners check its
blocks, memcpy's blocks, the same way on their own grid and path: it runs the tiny ladders and EDGE_BPP at N = 1, 2
(with and without LOCAL_DIAG) and 3, on every path and the grids of 1, 2, 3 and 7 CTAs, with flips at word 0 of size 0
and at the last word of the last, partial unit and a drop at the last size, on the loop-back cell too, and a corrupted
source word in a partial unit failing exactly the cells and sizes it fails for memcpy.

Every call uses one timed rep, so the faulted rep is the one folded into (S, X); the all-reduce's word check runs
after the warm-up and after the timed rep, and its bad words are summed over both.  Several ranks share GPU 0 with at
most 8 CTAs each, so every rank's grid stays resident."""
import functools
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import allreduce_ref
import alltoall_ref
import bwcurve_ref
import memcpy_ref
import word_ref
from conftest import ROOT
from test_bwcurve_gpu import slice_first_word

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
LOCAL_DIAG = 0x04
ERR_INTEGRITY = -10
U64_MAX = word_ref.U64_MAX
UNIT_WORDS = 1024   # 8 KiB
WARPS_PER_CTA = 8
PATHS = (0, 1, 2)   # TMA, 16-byte ld/st, 32-byte ld/st
OPS = (memcpy_ref.OP_READ, memcpy_ref.OP_WRITE)
# below one unit, below the 4096-byte minimum, exactly one ladder step, one vector past a unit, one granule, one vector
# past a granule, a partial unit in the second granule
TINY = (128, 3968, 4096, 4224, 8320, 16384, 16512, 24704)
# a partial last unit (384 bytes) in a partial last granule (8576 bytes), and enough units (58) that the last warp of
# a 7-CTA grid gets one: ladder 4096 ... 262144, 467328
EDGE_BPP = 57 * 8192 + 384


@functools.lru_cache(maxsize=None)
def src_words(rank, n_words):
    """Words [0, n_words) of rank's source buffer, from the pattern definition (cached)."""
    w = word_ref.src_words(SEED, rank, 0, n_words)
    w.setflags(write=False)
    return w


@pytest.fixture(scope="module")
def src():
    return src_words


def open_probe(pkg, n, bpp, flags=0):
    """A handle whose bytes_per_pair is bpp (sliced mode: bytes / peers)."""
    cfg = pkg.Config(ordinals=[0] * n, bytes=bpp * max(n - 1, 1), flags=(SAME if n > 1 else 0) | flags, ctas=8,
                     timeout_ms=20000)
    p = pkg.Open(cfg)
    assert p.Info().bytes_per_pair == bpp
    return p


def source(src, rank, n_words, corrupt):
    """Rank's source words [0, n_words) as they are at rest, with corrupt {(rank, word): mask} xored in."""
    w = src(rank, n_words).copy()
    for (r, k), m in corrupt.items():
        if r == rank and k < n_words:
            w[k] ^= np.uint64(m)
    return w


def check_bwcurve(bw, src, n, bpp, diag, corrupt=None):
    """Every cell at every size has the (S, X) of its slice's prefix as it is at rest; a cell fails exactly the sizes
    whose prefix holds a corrupted word."""
    corrupt = corrupt or {}
    sizes = bwcurve_ref.ladder(bpp)
    assert bw.sizes == sizes and bw.reps == 1
    W = bpp // 8
    for i in range(n):
        for j in range(n):
            if i == j and not diag:
                assert not bw.measured[i][j] and bw.status[i][j] == 0, (i, j)
                continue
            first = slice_first_word(n, i, j, bpp, False)
            words = source(src, j, first + W, corrupt)[first:]
            clean = src(j, first + W)[first:]
            bits = 0
            for k, s in enumerate(sizes):
                assert (bw.sum[i][j][k], bw.xr[i][j][k]) == allreduce_ref.checksum(words[:s // 8]), (i, j, s)
                if (words[:s // 8] != clean[:s // 8]).any():
                    bits |= 1 << k
            assert bw.measured[i][j] and bw.bad_sizes[i][j] == bits, (i, j, bw.bad_sizes[i][j], bits)
            assert bw.status[i][j] == (ERR_INTEGRITY if bits else 0), (i, j)
            assert (bw.t0_ns[i][j], bw.peak_gbps[i][j], bw.half_bytes[i][j]) == \
                bwcurve_ref.summary(sizes, bw.ns_median[i][j])
    return bw


def check_allreduce(ar, src, n, bpp, corrupt=None, fault=None):
    """Every row at every size holds the sum of the words at rest; a word is bad when that differs from the clean
    sum.  fault (rank, k, word, drop): timed rep 1 of size k on that rank adds 1 to the word, or (drop) stores
    nothing of its 8 KiB unit, which then reads as 0s.  The warm-up and the timed rep are both checked."""
    corrupt = corrupt or {}
    sizes = bwcurve_ref.ladder(bpp)
    assert ar.sizes == sizes and ar.reps == 1
    W = bpp // 8
    clean = sum(src(j, W) for j in range(n))
    at_rest = sum(source(src, j, W, corrupt) for j in range(n))
    for r in range(n):
        bits = 0
        for k, s in enumerate(sizes):
            warm = at_rest[:s // 8]
            words = warm.copy()  # timed rep 1's output
            if fault is not None and (r, k) == fault[:2]:
                if len(fault) > 3 and fault[3]:
                    unit = allreduce_ref.unit_words(fault[2], s)
                    words[unit[0]:unit[-1] + 1] = 0
                else:
                    words[fault[2]] += np.uint64(1)
            bad = [np.flatnonzero(w != clean[:s // 8]) for w in (warm, words)]
            ctx = (r, s, fault)
            assert (ar.sum[r][k], ar.xr[r][k]) == allreduce_ref.checksum(words), ctx
            assert ar.bad_words[r][k] == sum(len(b) for b in bad), (ctx, ar.bad_words[r][k])
            first = min((int(b[0]) for b in bad if len(b)), default=None)
            assert ar.first_bad[r][k] == (U64_MAX if first is None else 8 * first), (ctx, ar.first_bad[r][k])
            if first is not None:
                bits |= 1 << k
        assert ar.measured[r] and ar.bad_sizes[r] == bits, (r, ar.bad_sizes[r], bits)
        assert ar.status[r] == (ERR_INTEGRITY if bits else 0), r
        assert (ar.t0_ns[r], ar.peak_gbps[r], ar.half_bytes[r]) == allreduce_ref.summary(sizes, ar.ns_median[r])
    return ar


def check_memcpy(mc, src, n, bpp, diag, op, corrupt=None, fault=None):
    """Every cell at every size lands its source slice (memcpy_ref.cell) as it is at rest, in the warm-up and the timed
    rep, and is checked after each: a corrupted source word is one FLIP per rep at its offset in every cell and size
    that copies it.  fault (issuer, target, k, word, mode): timed rep 1 of that cell and size holds the word's pattern
    value xored with 1 (mode 0), or nothing, as the clear's 0s (mode 1)."""
    sizes = memcpy_ref.ladder(bpp)
    assert mc.sizes == sizes and mc.reps == 1 and mc.op == op
    for g in range(n):
        for j in range(n):
            if g == j and not diag:
                assert not mc.measured[g][j] and mc.status[g][j] == 0, (g, j)
                continue
            bits = check_block(mc, src, n, bpp, op, g, j, corrupt, fault)
            assert mc.measured[g][j] and mc.bad_sizes[g][j] == bits, (g, j, mc.bad_sizes[g][j], bits)
            assert mc.status[g][j] == (ERR_INTEGRITY if bits else 0), (g, j)
            assert (mc.t0_ns[g][j], mc.peak_gbps[g][j], mc.half_bytes[g][j]) == \
                memcpy_ref.summary(sizes, mc.ns_median[g][j])
    return mc


def check_block(out, src, n, bpp, op, g, j, corrupt=None, fault=None):
    """The checks of cell (g, j)'s block in `out` (a Memcpy or a CeAllToAll: the same blocks, checked the same way)
    against whole arrays: per size the (S, X) of timed rep 1, the bad words of the warm-up and rep 1 and the lowest
    bad offset.  Returns the sizes that must fail, as bits."""
    corrupt = corrupt or {}
    W = bpp // 8
    c = memcpy_ref.cell(n, bpp, 1, op, g, j)
    first = c["first_word"]
    words = source(src, c["src_rank"], first + W, corrupt)[first:]
    pattern = src(c["src_rank"], first + W)[first:]
    bits = 0
    for k, s in enumerate(memcpy_ref.ladder(bpp)):
        nw = s // 8
        warm, rep1 = words[:nw], words[:nw].copy()
        if fault is not None and (g, j, k) == fault[:3]:
            if fault[4]:
                rep1[:] = 0
            else:
                rep1[fault[3]] = pattern[fault[3]] ^ np.uint64(1)
        bad = [np.flatnonzero(w != pattern[:nw]) for w in (warm, rep1)]
        first_bad = min((int(b[0]) for b in bad if len(b)), default=None)
        ctx = (g, j, s, op, fault)
        assert (out.sum[g][j][k], out.xr[g][j][k]) == allreduce_ref.checksum(rep1), ctx
        assert out.bad_words[g][j][k] == sum(len(b) for b in bad), (ctx, out.bad_words[g][j][k])
        assert out.first_bad[g][j][k] == (U64_MAX if first_bad is None else 8 * first_bad), \
            (ctx, out.first_bad[g][j][k])
        if first_bad is not None:
            bits |= 1 << k
    return bits


def check_ce_alltoall(ca, src, n, bpp, diag, op, corrupt=None, fault=None):
    """Every rank issued every cell, and every block its owner checked holds, in the warm-up and the timed rep, what
    memcpy's cell (issuer, target) lands (check_block); fault (issuer, target, k, word, mode) as memcpy's."""
    sizes = memcpy_ref.ladder(bpp)
    assert ca.sizes == sizes and ca.reps == 1 and ca.op == op
    for r in range(n):
        assert ca.measured[r] and ca.status[r] == 0 and ca.blocks[r] == n - 1 + diag, r
    for g in range(n):
        for j in range(n):
            if g == j and not diag:
                assert not ca.cell_measured[g][j] and ca.cell_status[g][j] == 0, (g, j)
                continue
            bits = check_block(ca, src, n, bpp, op, g, j, corrupt, fault)
            assert ca.cell_measured[g][j] and ca.bad_sizes[g][j] == bits, (g, j, ca.bad_sizes[g][j], bits)
            assert ca.cell_status[g][j] == (ERR_INTEGRITY if bits else 0), (g, j)
    return ca


def check_alltoall(aa, n, bpp, diag, fault=None):
    """Every block at every size holds its sender's pattern of this call; fault (sender, receiver, k, word): timed rep
    1 of size k delivers that word xored with 1, and only there."""
    sizes = bwcurve_ref.ladder(bpp)
    assert aa.sizes == sizes and aa.reps == 1
    blocks = n - 1 + (1 if diag else 0)
    for s in range(n):
        assert aa.measured[s] and aa.status[s] == 0 and aa.blocks[s] == blocks, s
        assert (aa.t0_ns[s], aa.peak_gbps[s], aa.half_bytes[s]) == \
            alltoall_ref.summary(sizes, aa.ns_median[s], blocks)
        for d in range(n):
            if s == d and not diag:
                assert not aa.cell_measured[s][d], (s, d)
                continue
            bits = 0
            for k, size in enumerate(sizes):
                words = alltoall_ref.block_words(SEED, s, d, aa.call_seq, k, 1, size // 8)
                hit = fault is not None and (s, d, k) == fault[:3]
                if hit:
                    words[fault[3]] ^= np.uint64(1)
                    bits |= 1 << k
                ctx = (s, d, size, fault)
                assert (aa.sum[s][d][k], aa.xr[s][d][k]) == allreduce_ref.checksum(words), ctx
                assert aa.bad_words[s][d][k] == (1 if hit else 0), (ctx, aa.bad_words[s][d][k])
                assert aa.first_bad[s][d][k] == (8 * fault[3] if hit else U64_MAX), (ctx, aa.first_bad[s][d][k])
            assert aa.cell_measured[s][d] and aa.bad_sizes[s][d] == bits, (s, d, aa.bad_sizes[s][d], bits)
            assert aa.cell_status[s][d] == (ERR_INTEGRITY if bits else 0), (s, d)
    return aa


def block_index(n, s, d):
    """Position of block (s -> d) in sender s's walk: receivers s + 1, s + 2, ... (mod n), then the diagonal."""
    return n - 1 if s == d else (d - s - 1) % n


def last_warp_fault(n, bpp, diag, nwarps):
    """(sender, receiver, k, word) of a word whose walk unit falls to warp nwarps - 1 (walk unit t = unit x blocks +
    block goes to warp t % nwarps), at the largest size that has one; None when the grid has more warps than units."""
    sizes = bwcurve_ref.ladder(bpp)
    blocks = n - 1 + (1 if diag else 0)
    for k in reversed(range(len(sizes))):
        words = sizes[k] // 8
        for s in range(n):
            for d in range(n):
                if s == d and not diag:
                    continue
                for u in range((words + UNIT_WORDS - 1) // UNIT_WORDS):
                    if (u * blocks + block_index(n, s, d)) % nwarps == nwarps - 1:
                        return s, d, k, min((u + 1) * UNIT_WORDS, words) - 1
    return None


# ---- tiny ladders ------------------------------------------------------------------------------------------------
TINY_CASES = [(n, bpp) for n in (1, 2) for bpp in TINY]


@pytest.mark.parametrize("n,bpp", TINY_CASES, ids=[f"n{n}-{bpp}B" for n, bpp in TINY_CASES])
def test_tiny_ladders_every_path_clean(pkg, src, n, bpp):
    with open_probe(pkg, n, bpp) as p:
        for path in PATHS:
            p.SetOption(pkg.abi.OPT_PATH, path)
            check_bwcurve(p.BwCurve(reps=1), src, n, bpp, n == 1)
            check_allreduce(p.AllReduce(reps=1), src, n, bpp)
            check_alltoall(p.AllToAll(reps=1), n, bpp, n == 1)
            for op in OPS:
                check_memcpy(p.Memcpy(op, reps=1), src, n, bpp, n == 1, op)


@pytest.mark.parametrize("bpp", TINY)
def test_tiny_ladders_with_the_diagonal_block(pkg, src, bpp):
    n = 3
    with open_probe(pkg, n, bpp, LOCAL_DIAG) as p:
        for path in PATHS:
            p.SetOption(pkg.abi.OPT_PATH, path)
            check_bwcurve(p.BwCurve(reps=1), src, n, bpp, True)
            check_alltoall(p.AllToAll(reps=1), n, bpp, True)
            for op in OPS:
                check_memcpy(p.Memcpy(op, reps=1), src, n, bpp, True, op)


# ---- grids and edge-placed faults ----------------------------------------------------------------------------------
GRIDS = [(1, ("ctas", 0)), (1, ("ctas", 1)), (1, ("ctas", 2)), (1, ("ctas", 3)), (1, ("ctas", 7)),
         (3, ("ctas", 1)), (3, ("ctas", 2)), (3, ("ctas", 3)), (3, ("ctas", 7)), (3, ("rank", (1, 8, 3)))]


@pytest.mark.parametrize("n,grid", GRIDS, ids=[f"n{n}-{g[0]}{'-'.join(map(str, g[1])) if g[0] == 'rank' else g[1]}"
                                                for n, g in GRIDS])
def test_grids_and_faults_at_the_edges(pkg, src, n, grid):
    a = pkg.abi
    bpp, diag = EDGE_BPP, True  # N = 3 opens with the diagonal block, so the all-to-all has one to fault
    sizes = bwcurve_ref.ladder(bpp)
    last, W = len(sizes) - 1, bpp // 8
    assert bpp % 8192 and bpp % 16384
    with open_probe(pkg, n, bpp, LOCAL_DIAG if n > 1 else 0) as p:
        if grid[0] == "ctas":
            p.SetOption(a.OPT_CTAS, grid[1])
        else:
            for li, c in enumerate(grid[1]):
                p.SetOption(a.OPT_CTAS_RANK, ((li + 1) << 16) | c)
        info = p.Info()
        ctas = [info.ctas[li] for li in range(n)]
        assert ctas == ([info.sm_count[0]] if grid[1] == 0 else list(grid[1]) if grid[0] == "rank" else [grid[1]] * n)
        for path in PATHS:
            p.SetOption(a.OPT_PATH, path)
            check_bwcurve(p.BwCurve(reps=1), src, n, bpp, diag)
            # the all-reduce: word 0 of size 0, and the last word of the last, partial unit of the last size, each off
            # by one and as its unit not stored (size 0's half unit, the last size's 384-byte unit)
            for fault in ((n - 1, 0, 0, False), (0, last, W - 1, False), (n - 1, 0, 0, True), (0, last, W - 1, True)):
                p.SetOption(a.OPT_ALLREDUCE_FAULT, a.allreduce_fault(*fault))
                check_allreduce(p.AllReduce(reps=1), src, n, bpp, fault=fault)
            p.SetOption(a.OPT_ALLREDUCE_FAULT, 0)
            check_allreduce(p.AllReduce(reps=1), src, n, bpp)
            # the all-to-all: the last word of a partial unit, a word of the grid's last warp, the diagonal block
            faults = [(0, 1 % n, last, W - 1), (n - 1, n - 1, 0, sizes[0] // 8 - 1)]
            lw = last_warp_fault(n, bpp, diag, WARPS_PER_CTA * ctas[0]) if len(set(ctas)) == 1 else None
            if lw is not None:
                faults.append(lw)
            for fault in faults:
                p.SetOption(a.OPT_ALLTOALL_FAULT, a.alltoall_fault(*fault))
                check_alltoall(p.AllToAll(reps=1), n, bpp, diag, fault)
            p.SetOption(a.OPT_ALLTOALL_FAULT, 0)
            check_alltoall(p.AllToAll(reps=1), n, bpp, diag)
            # memcpy: word 0 of size 0, the last word of the last, partial unit, the diagonal cell; flipped, dropped
            for op in OPS:
                check_memcpy(p.Memcpy(op, reps=1), src, n, bpp, diag, op)
            for q, (g, j, k, word) in enumerate(((0, 1 % n, 0, 0), (n - 1, 0, last, W - 1), (n - 1, n - 1, 1, 7))):
                for mode in (0, 1):
                    op = OPS[(q + mode) % 2]
                    p.SetOption(a.OPT_MEMCPY_FAULT, a.memcpy_fault(g, j, k, word, mode))
                    check_memcpy(p.Memcpy(op, reps=1), src, n, bpp, diag, op, fault=(g, j, k, word, mode))
            p.SetOption(a.OPT_MEMCPY_FAULT, 0)
            if path != 2:
                continue
            # a source word in a partial unit, on the 32-byte ld/st path: the last word of slice 0 of rank n - 1 (only
            # the last size reads it), then the last word of size 0's half unit (every size reads it)
            j = n - 1
            i = 0 if n == 1 else (1 if j == 0 else 0)  # the cell that reads slice 0 of j's buffer
            assert slice_first_word(n, i, j, bpp, False) == 0
            for word in (W - 1, sizes[0] // 8 - 1):
                corrupt = {(j, word): 1 << 33}
                p.Corrupt(j, 8 * word, 1 << 33)
                check_bwcurve(p.BwCurve(reps=1), src, n, bpp, diag, corrupt)
                check_allreduce(p.AllReduce(reps=1), src, n, bpp, corrupt)
                check_alltoall(p.AllToAll(reps=1), n, bpp, diag)
                for op in OPS:
                    mc = check_memcpy(p.Memcpy(op, reps=1), src, n, bpp, diag, op, corrupt)
                    assert any(mc.bad_sizes[g][d] for g in range(n) for d in range(n) if mc.measured[g][d])
                p.Corrupt(j, 8 * word, 1 << 33)  # restore: the next calls are clean
                check_bwcurve(p.BwCurve(reps=1), src, n, bpp, diag)
                check_allreduce(p.AllReduce(reps=1), src, n, bpp)


def test_the_last_warp_placement_exists_on_small_grids():
    """The grid test's placement of an all-to-all fault on the grid's last warp is not vacuous on any grid but the full
    one."""
    for n, ctas in ((1, 1), (1, 2), (1, 3), (1, 7), (3, 1), (3, 2), (3, 3), (3, 7)):
        s, d, k, word = last_warp_fault(n, EDGE_BPP, True, WARPS_PER_CTA * ctas)
        blocks = n
        t = word // UNIT_WORDS * blocks + block_index(n, s, d)
        assert t % (WARPS_PER_CTA * ctas) == WARPS_PER_CTA * ctas - 1 and word < bwcurve_ref.ladder(EDGE_BPP)[k] // 8


# ---- the copy-engine all-to-all ---------------------------------------------------------------------------------------
# Its owners check every block with memcpy's diag_launch and bwcurve_kernel, on the owner's grid and path.  N ranks on
# one device need N x N streams (N x (N + 1) with the loop-back), so every case runs in a child process with 32 hardware
# queues per device; the CUDA runtime reads the variable once, at its start.
CE_CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path[:0] = [%r, %r]
    sys.modules["torch"] = None
    import cdprobe_pkg
    import test_ladder_edges_gpu as t
    getattr(t, sys.argv[1])(cdprobe_pkg.load(), *json.loads(sys.argv[2]))
    print("CHILD OK")
    """
) % (ROOT, os.path.join(ROOT, "tests"))


def ce_in_child(case, *args):
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    pr = subprocess.run([sys.executable, "-c", CE_CHILD, case, json.dumps(args)], env=env, capture_output=True,
                        text=True, timeout=1200)
    assert pr.returncode == 0 and "CHILD OK" in pr.stdout, pr.stderr[-8000:]


def case_ce_alltoall_tiny(pkg, n, flags):
    """Both ops on every tiny ladder and on EDGE_BPP, on every path: every block clean."""
    diag = n == 1 or bool(flags & LOCAL_DIAG)
    for bpp in TINY + (EDGE_BPP,):
        with open_probe(pkg, n, bpp, flags) as p:
            for path in PATHS:
                p.SetOption(pkg.abi.OPT_PATH, path)
                for op in OPS:
                    check_ce_alltoall(p.CeAllToAll(op, reps=1), src_words, n, bpp, diag, op)


def case_ce_alltoall_grids_and_edges(pkg, n, flags):
    """EDGE_BPP on grids of 1, 2, 3 and 7 CTAs per rank and every path: clean; a flip at word 0 of size 0, a flip at
    the last word of the last, partial unit and a drop at the last size, on the loop-back cell too when there is one,
    each failing exactly its cell and size; and a corrupted source word in a partial unit failing exactly the cells and
    sizes memcpy fails for it on the same handle."""
    a = pkg.abi
    bpp = EDGE_BPP
    diag = n == 1 or bool(flags & LOCAL_DIAG)
    sizes = memcpy_ref.ladder(bpp)
    last, W = len(sizes) - 1, bpp // 8
    faults = [(0, 1 % n, 0, 0, 0), (n - 1, 0, last, W - 1, 0), (n - 1, 0, last, W // UNIT_WORDS * UNIT_WORDS + 5, 1)]
    if diag:
        faults += [(n - 1, n - 1, 0, 0, 0), (n - 1, n - 1, last, W - 1, 0), (0, 0, last, 0, 1)]
    faults = [f for f in faults if f[0] != f[1] or diag]
    with open_probe(pkg, n, bpp, flags) as p:
        for q, ctas in enumerate((1, 2, 3, 7)):
            p.SetOption(a.OPT_CTAS, ctas)
            assert [p.Info().ctas[li] for li in range(n)] == [ctas] * n
            for path in PATHS:
                p.SetOption(a.OPT_PATH, path)
                for op in OPS:
                    check_ce_alltoall(p.CeAllToAll(op, reps=1), src_words, n, bpp, diag, op)
            p.SetOption(a.OPT_PATH, q % 3)
            for f, fault in enumerate(faults):
                op = OPS[(q + f) % 2]
                p.SetOption(a.OPT_CE_ALLTOALL_FAULT, a.ce_alltoall_fault(*fault))
                ca = check_ce_alltoall(p.CeAllToAll(op, reps=1), src_words, n, bpp, diag, op, fault=fault)
                assert ca.bad_sizes[fault[0]][fault[1]] == 1 << fault[2], fault
            p.SetOption(a.OPT_CE_ALLTOALL_FAULT, 0)
        # a source word in a partial unit, on the 32-byte ld/st path: the last word of slice 0 of rank n - 1, then the
        # last word of size 0's half unit
        p.SetOption(a.OPT_PATH, 2)
        j = n - 1
        for word in (W - 1, sizes[0] // 8 - 1):
            corrupt = {(j, word): 1 << 33}
            p.Corrupt(j, 8 * word, 1 << 33)
            for op in OPS:
                ca = check_ce_alltoall(p.CeAllToAll(op, reps=1), src_words, n, bpp, diag, op, corrupt)
                mc = check_memcpy(p.Memcpy(op, reps=1), src_words, n, bpp, diag, op, corrupt)
                cells = [(g, d) for g in range(n) for d in range(n) if g != d or diag]
                assert [ca.bad_sizes[g][d] for g, d in cells] == [mc.bad_sizes[g][d] for g, d in cells], (word, op)
                assert any(ca.bad_sizes[g][d] for g, d in cells), (word, op)
            p.Corrupt(j, 8 * word, 1 << 33)  # restore: the next calls are clean
            for op in OPS:
                check_ce_alltoall(p.CeAllToAll(op, reps=1), src_words, n, bpp, diag, op)


CE_SHAPES = [(1, 0), (2, 0), (2, LOCAL_DIAG), (3, 0)]
CE_IDS = ["n1", "n2", "n2-local-diag", "n3"]


@pytest.mark.parametrize("n,flags", CE_SHAPES, ids=CE_IDS)
def test_ce_alltoall_tiny_ladders_every_path_clean(n, flags):
    ce_in_child("case_ce_alltoall_tiny", n, flags)


@pytest.mark.parametrize("n,flags", CE_SHAPES, ids=CE_IDS)
def test_ce_alltoall_grids_and_faults_at_the_edges(n, flags):
    ce_in_child("case_ce_alltoall_grids_and_edges", n, flags)
