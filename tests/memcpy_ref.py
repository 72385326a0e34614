"""Plain restatement of what cdprobe_memcpy copies and where it lands, for the tests: which cells run in which round,
the source slice and destination block of a cell for each op, the words every ladder prefix must land and their (S, X).
It follows the doc comments of cdprobe_memcpy and cdprobe_memcpy_t in include/cdprobe.h and DESIGN §5n; the partner
table comes from the oracle's plan, which is written apart from the library's."""
import numpy as np

import word_ref
from allreduce_ref import checksum  # noqa: F401  (the (S, X) definition)
from bwcurve_ref import ladder, summary  # noqa: F401

OP_READ, OP_WRITE = 1, 2
MODE_FULL = 2
REF_MAX_BYTES = 64 << 20  # prefixes up to this get their (S, X) from numpy; longer ones from the oracle


def cell(n: int, bpp: int, mode: int, op: int, g: int, j: int) -> dict:
    """The copy of cell (issuer g, target j): a pull (OP_READ) moves the slice g reads from j into block j of g's
    exchange area; a push (OP_WRITE) moves the slice j reads from g into block g of j's.  A slice is the reader's slot
    in the owner's source buffer (n - 1 for the loop-back), or slice 0 in full mode."""
    reader, owner = (j, g) if op == OP_WRITE else (g, j)
    slot = n - 1 if reader == owner else (reader if reader < owner else reader - 1)
    sl = 0 if mode == MODE_FULL else slot
    return dict(src_rank=owner, src_off=sl * bpp, first_word=sl * bpp // 8, dst_rank=reader, dst_off=owner * bpp)


def schedule(oracle, n: int, nbytes: int, mode: int, diag: bool, op: int):
    """(bytes_per_pair, [(round, issuer, target, cell)]) in the order cdprobe_memcpy runs the cells: the tournament's
    rounds of the oracle's plan, then the loop-back round when there is a loop-back slice (n == 1 or LOCAL_DIAG)."""
    diag = diag or n == 1
    pl = oracle.plan(n, nbytes, mode, diag)
    bpp = pl.bytes_per_pair
    out = []
    for r in range(pl.rounds):
        for g in range(n):
            q = pl.partner[r][g]
            if q >= 0:
                out.append((r, g, q, cell(n, bpp, mode, op, g, q)))
    if diag:
        out += [(pl.rounds, g, g, cell(n, bpp, mode, op, g, g)) for g in range(n)]
    return bpp, out


def words(seed: int, c: dict, nbytes: int) -> np.ndarray:
    """The words the first nbytes of the cell's destination must hold: its source slice's pattern words."""
    return word_ref.src_words(seed, c["src_rank"], c["first_word"], nbytes // 8)


def expected(oracle, seed: int, c: dict, sizes) -> list:
    """(S, X) of every ladder prefix of the cell's destination: numpy up to REF_MAX_BYTES, the oracle above."""
    return [checksum(words(seed, c, s)) if s <= REF_MAX_BYTES else
            oracle.src_checksum(seed, c["src_rank"], c["first_word"], s // 8) for s in sizes]
