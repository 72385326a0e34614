"""Plain CPU restatement of cdprobe_latency's dependent-load chase, for the tests.

Restated from the spec (DESIGN §5c, include/cdprobe.h), not from the CUDA, in Python integers; numpy only builds the
word table of a small region for a cross-check.  A chase ranges over the L = bytes / 128 lines of the source slice
issuer i reads from target j, whose word 0 is word `first` of j's source pattern:

    fastrange(x, L)  = (x * L) >> 64
    start of rep r   = fastrange(splitmix64(seed ^ "LATENCY" ^ i << 56 ^ j << 48 ^ r), L)      r = 0: the warm-up
    hop h loads      v = word 16 * line of the region = src_word(seed, j, first + 16 * line)
    next line        = fastrange(v ^ (h + 1) * golden, L)
    digest           = xor of every loaded v over reps 0 .. reps
"""
from __future__ import annotations

from typing import Dict, Iterator, Optional, Tuple

import numpy as np

M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15
TAG = int.from_bytes(b"LATENCY", "big")  # 0x4C4154454E4359
LINE_WORDS = 16
LINE_BYTES = 128


def splitmix64(x: int) -> int:
    z = (x + GOLDEN) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def src_word(seed: int, rank: int, k: int) -> int:
    return splitmix64(seed ^ ((rank << 56) & M64) ^ k)


def fastrange(x: int, n: int) -> int:
    return (x * n) >> 64


def start_line(seed: int, i: int, j: int, rep: int, lines: int) -> int:
    return fastrange(splitmix64(seed ^ TAG ^ ((i << 56) & M64) ^ ((j << 48) & M64) ^ rep), lines)


def next_line(v: int, hop: int, lines: int) -> int:
    return fastrange(v ^ (((hop + 1) * GOLDEN) & M64), lines)


def chase(seed: int, i: int, j: int, first: int, lines: int, rep: int, hops: int,
          words: Optional[Dict[int, int]] = None) -> Iterator[Tuple[int, int]]:
    """(line, v) of every hop of one rep.  `words` overrides source words by index in j's buffer (a corrupted
    pattern); every other word is the spec's."""
    line = start_line(seed, i, j, rep, lines)
    for h in range(hops):
        k = first + LINE_WORDS * line
        v = words[k] if words is not None and k in words else src_word(seed, j, k)
        yield line, v
        line = next_line(v, h, lines)


def digest(seed: int, i: int, j: int, first: int, lines: int, hops: int, reps: int,
           words: Optional[Dict[int, int]] = None) -> int:
    """What cdprobe_latency reports for the cell: the xor of every loaded word over the warm-up and `reps` reps."""
    d = 0
    for r in range(reps + 1):
        for _, v in chase(seed, i, j, first, lines, r, hops, words):
            d ^= v
    return d


def loaded_word(seed: int, i: int, j: int, first: int, lines: int, rep: int, hop: int) -> int:
    """Index in j's source buffer of the word that hop `hop` of rep `rep` loads (intact pattern)."""
    for h, (line, _) in enumerate(chase(seed, i, j, first, lines, rep, hop + 1)):
        if h == hop:
            return first + LINE_WORDS * line
    raise ValueError(hop)


def region_words(seed: int, j: int, first: int, lines: int) -> np.ndarray:
    """Every word of a (small) region, vectorised: the table a chase indexes."""
    k = np.arange(lines * LINE_WORDS, dtype=np.uint64) + np.uint64(first)
    z = (np.uint64(seed) ^ np.uint64((j << 56) & M64) ^ k) + np.uint64(GOLDEN)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def first_word(cell_slice: int, bytes_per_pair: int) -> int:
    """Index of the region's word 0 in the target's source buffer (slice `cell_slice`, 0 in full mode)."""
    return cell_slice * (bytes_per_pair // 8)
