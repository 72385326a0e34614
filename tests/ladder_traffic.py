"""The least HBM traffic one timed rep of a ladder measurement must cause when all N ranks share one device, and the
time floor that follows from it.  For the timing tests (test_ladder_timing_gpu.py); pinned by test_ladder_traffic_cpu.py.

unique_bytes counts the distinct bytes a rep must read and write: every input read once and every output written once.
L2 reuse between ranks that read the same input cannot undercut that count; it only removes repeats.  The counts are
read off the kernels and DESIGN §5f-§5p:

  bwcurve       one cell reads its source prefix; nothing is written.  The cells of one round run at once, each on its
                own grid, but their reps are not aligned (no domain barrier per rep), so the count is one cell's.
  allreduce     one-shot: every rank reads all n inputs (shared: n x size) and writes its own output (n x size).
  twoshot       each rank reads its chunk of all n inputs (n x size in all) and stores the summed chunk into every
                rank's gather area (n x size).
  ring          each rank reads its own input (n x size) and every rank's ring area ends holding the whole output
                (n x size); the partials passed hop by hop land in those same bytes, and the flags add 4 bytes per unit,
                which the count leaves out.
  push          each rank reads its own input (n x size); the reductions and the all-gather write the push areas
                (n x size).
  alltoall      no source is read (the words come from the write pattern); every block that runs is written once:
                n (n - 1) off-diagonal blocks, plus n with a loop-back slice (n = 1 or LOCAL_DIAG).
  memcpy        one cell copies its source slice into an exchange-area block, pull or push: size read, size written.
                Like bwcurve, the count is one cell's.
  ce_alltoall   every cell copies at once in every rep, each its own source slice (sliced mode, which the timing tests
                open) into its own block: 2 x size per cell, with cells as for the all-to-all, pull or push alike.

floor_ns = (unique - 2 x 50 MB) / 3350 GB/s: the H100 SXM data-sheet HBM rate, less one resident read set and one dirty
tail of the 50 MB L2 that the warm-up rep or the rep's own writes may leave there.  At N = 1 this is tight: the rep
moves nearly exactly these bytes.  At N > 1 it is sound but loose: ranks re-read shared inputs and pass partials, all
of which the count leaves out, and only the union of the ranks' windows has to hold the traffic.

The LL all-reduce is excluded: its ladder stops at 1 MiB, which stays in L2.  So is the multicast all-reduce, which
needs one device per rank."""
HBM_GBPS = 3350.0      # NVIDIA H100 SXM data sheet, HBM3
L2_BYTES = 50_000_000  # H100 SXM L2
MEASUREMENTS = ("bwcurve", "allreduce", "twoshot", "ring", "push", "alltoall", "memcpy", "ce_alltoall")
COLLECTIVES = ("allreduce", "twoshot", "ring", "push", "alltoall", "ce_alltoall")
OP_READ, OP_WRITE = 1, 2


def blocks(n: int, diag: bool) -> int:
    """Blocks the all-to-all and the CE all-to-all move per rep over the whole domain."""
    return n * (n - 1) + (n if diag or n == 1 else 0)


def unique_bytes(name: str, n: int, size: int, op: int = OP_READ, diag: bool = False) -> int:
    """Distinct bytes one timed rep of `name` at `size` moves through the one device's memory, for n ranks on it."""
    assert op in (OP_READ, OP_WRITE), op
    if name in ("bwcurve",):
        return size
    if name in ("allreduce", "twoshot", "ring", "push"):
        return 2 * n * size
    if name == "alltoall":
        return blocks(n, diag) * size
    if name == "memcpy":
        return 2 * size
    if name == "ce_alltoall":
        return 2 * blocks(n, diag) * size
    raise ValueError(f"no HBM floor for {name}")


def floor_ns(unique: int) -> float:
    """The least time that many unique bytes take through HBM, beyond what L2 can hold; 0 when L2 holds them all."""
    return max(0.0, unique - 2 * L2_BYTES) / HBM_GBPS
