"""tests/ladder_traffic.py against the index sets the references define, at small n and sizes: what each rank of a rep
reads and writes, as (memory, byte) ranges taken from alltoall_ref's block order, the two-shot's chunks, the push
all-reduce's owners, the ring's pushed chunks and memcpy_ref's and ce_alltoall_ref's cells; the union of those ranges
must be exactly unique_bytes.  The same sets give each rank's bytes to and from its peers, which must be DESIGN's
algorithmic-byte statements.  And the floor itself: its arithmetic, and the measurements it leaves out."""
import pytest

import allreduce_push_ref as push_ref
import allreduce_ring_ref as ring_ref
import allreduce_twoshot_ref as ts
import alltoall_ref
import ce_alltoall_ref
import ladder_traffic as lt
import memcpy_ref

UNIT = ts.UNIT_BYTES
SIZES = (4096, 8192, 3 * 8192, 40 * 8192 + 128, 1 << 20)
NS = (1, 2, 3, 4, 5)


def union(ranges):
    """Bytes covered by ranges (memory, lo, hi); memory is any hashable name."""
    by = {}
    for mem, lo, hi in ranges:
        by.setdefault(mem, []).append((lo, hi))
    total = 0
    for spans in by.values():
        end = -1
        for lo, hi in sorted(spans):
            total += max(0, hi - max(lo, end))
            end = max(end, hi)
    return total


def unit_range(size, u):
    return u * UNIT, min((u + 1) * UNIT, size)


def rep_ranges(name, n, size, op=lt.OP_READ, diag=False, bpp=None):
    """(reads, writes) of one rep over the whole domain, each [(memory, lo, hi)] with memory (kind, rank[, block])."""
    U = ts.units(size)
    reads, writes = [], []
    if name == "bwcurve":
        reads = [(("src", 0), 0, size)]
    elif name == "allreduce":
        for r in range(n):
            reads += [(("src", (r + t) % n), 0, size) for t in range(n)]
            writes += [(("out", r), 0, size)]
    elif name == "twoshot":
        for r in range(n):
            for u in range(*ts.chunk(U, n, r)):
                reads += [(("src", j), *unit_range(size, u)) for j in range(n)]
                writes += [(("gather", d), *unit_range(size, u)) for d in range(n)]
    elif name == "push":
        for r in range(n):
            for u in range(U):
                reads += [(("src", r), *unit_range(size, u))]
                writes += [(("push", push_ref.owner(U, n, u)), *unit_range(size, u))]  # the reduction into the owner
            for u in range(*ts.chunk(U, n, r)):
                assert push_ref.owner(U, n, u) == r
                writes += [(("push", d), *unit_range(size, u)) for d in range(n) if d != r]  # the all-gather
    elif name == "ring":
        for g in range(n):
            reads += [(("src", g), 0, size)]
            for phase in (0, 1):
                for c in ring_ref.pushes(n, g, phase):
                    for u in range(*ts.chunk(U, n, c)):
                        writes += [(("ring", (g + 1) % n), *unit_range(size, u))]
            if n == 1:
                writes += [(("ring", g), 0, size)]
            else:  # the chunk each rank finishes in the last reduce-scatter step stays in its own area
                for u in range(*ts.chunk(U, n, (g + 1) % n)):
                    writes += [(("ring", g), *unit_range(size, u))]
    elif name == "alltoall":
        runs = lambda s, d: s != d or diag or n == 1  # noqa: E731
        for s in range(n):
            writes += [(("area", d, s), 0, size) for d in alltoall_ref.block_order(s, n, runs)]
    elif name in ("memcpy", "ce_alltoall"):
        cells = [(0, 0)] if name == "memcpy" else ce_alltoall_ref.cells(n, diag)
        nn = 1 if name == "memcpy" else n
        for g, j in cells:
            c = memcpy_ref.cell(nn, bpp, 1, op, g, j)
            reads += [(("src", c["src_rank"]), c["src_off"], c["src_off"] + size)]
            writes += [(("area", c["dst_rank"]), c["dst_off"], c["dst_off"] + size)]
    return reads, writes


@pytest.mark.parametrize("name", lt.MEASUREMENTS)
def test_unique_bytes_are_the_union_of_the_index_sets(name):
    for n in NS if name not in ("bwcurve", "memcpy") else (1,):
        for size in SIZES:
            for diag in (False, True):
                for op in (lt.OP_READ, lt.OP_WRITE):
                    reads, writes = rep_ranges(name, n, size, op, diag, bpp=size + 4096)
                    got = union(reads) + union(writes)
                    assert got == lt.unique_bytes(name, n, size, op, diag), (name, n, size, op, diag, got)


def link_bytes(name, n, size, g):
    """(bytes rank g reads from peers, bytes it writes into peers) in one rep, from the index sets."""
    reads, writes = [], []
    if name == "allreduce":
        reads = [r for r in rep_ranges(name, n, size)[0] if r[0][1] != g][:n - 1]  # rank g's own n - 1 remote reads
    U = ts.units(size)
    if name == "twoshot":
        for u in range(*ts.chunk(U, n, g)):
            reads += [(j, *unit_range(size, u)) for j in range(n) if j != g]
            writes += [(d, *unit_range(size, u)) for d in range(n) if d != g]
    if name == "ring":
        for phase in (0, 1):
            for c in ring_ref.pushes(n, g, phase):
                writes += [((g + 1) % n, phase, *unit_range(size, u)) for u in range(*ts.chunk(U, n, c))]
    if name == "push":
        for u in range(U):
            o = push_ref.owner(U, n, u)
            writes += [(o, *unit_range(size, u))] if o != g else [(d, *unit_range(size, u)) for d in range(n) if d != g]
    return sum(r[-1] - r[-2] for r in reads), sum(w[-1] - w[-2] for w in writes)


@pytest.mark.parametrize("n", (2, 3, 4, 8))
def test_peer_bytes_are_designs(n):
    """§5g: the one-shot moves (n - 1) x size into each rank.  §5i, §5k, §5l: the two-shot, the ring and the push move
    2 (n - 1) / n x size per rank, when the units split evenly."""
    size = n * 4 * UNIT
    for g in range(n):
        assert link_bytes("allreduce", n, size, g) == ((n - 1) * size, 0)
        assert sum(link_bytes("twoshot", n, size, g)) == 2 * (n - 1) * size // n
        assert sum(link_bytes("ring", n, size, g)) == 2 * (n - 1) * size // n
        assert sum(link_bytes("push", n, size, g)) == 2 * (n - 1) * size // n


def test_alltoall_blocks_are_the_reported_blocks():
    """§5h: a rank pushes one block to every cell it has; the domain's blocks are what every rank's `blocks` sums to."""
    for n in NS:
        for diag in (False, True):
            runs = lambda s, d: s != d or diag or n == 1  # noqa: E731
            assert sum(len(alltoall_ref.block_order(s, n, runs)) for s in range(n)) == lt.blocks(n, diag)
            assert len(ce_alltoall_ref.cells(n, diag)) == lt.blocks(n, diag)


def test_floor_arithmetic():
    GIB = 1 << 30
    assert lt.floor_ns(0) == 0.0 and lt.floor_ns(2 * lt.L2_BYTES) == 0.0
    assert lt.floor_ns(GIB) == (GIB - 100_000_000) / 3350.0
    # N = 1 at 1 GiB: one input and one output through HBM
    assert lt.unique_bytes("allreduce", 1, GIB) == lt.unique_bytes("memcpy", 1, GIB) == 2 * GIB
    assert lt.unique_bytes("bwcurve", 1, GIB) == lt.unique_bytes("alltoall", 1, GIB) == GIB
    assert round(lt.floor_ns(2 * GIB)) == 611_189


@pytest.mark.parametrize("name", ["ll", "nvls", "allreduce_ll"])
def test_l2_resident_and_multicast_ladders_have_no_floor(name):
    with pytest.raises(ValueError):
        lt.unique_bytes(name, 1, 1 << 20)
