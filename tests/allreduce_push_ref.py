"""Plain restatement of one rep of cdprobe_allreduce_push and of what each armed fault does to it, for the tests
(include/cdprobe.h, DESIGN §5l).

    chunks            the two-shot's: rank r owns units [floor(r U / n), floor((r + 1) U / n)), U = ceil(size / 8 KiB)
    owner(U, n, u)    the rank whose chunk holds unit u: floor(((u + 1) n - 1) / U)
    reduce-scatter    every sender adds every unit of its input into the zeroed area of the unit's owner, at its place
    all-gather        every owner copies its finished chunk into every peer's area
    bus bandwidth     algorithm bandwidth x 2 (n - 1) / n

Fault (mode, rank, word), in the rep it is armed for:

    mode 0   sender `rank` contributes its source word + 1             every row, one bad word at 8 word
    mode 1   sender `rank` skips the reduction of the word's unit        every row, the unit's words where the sender's
    mode 2   sender `rank` reduces the word's unit twice                   source word is not 0
    mode 3   the word's owner pushes it xored with 1 to receiver `rank`  row `rank`, one bad word at 8 word

Every rank ends a clean rep holding the whole all-reduce output, so what it must hold is allreduce_ref's."""
import numpy as np

import allreduce_twoshot_ref as ts

UNIT_BYTES = ts.UNIT_BYTES
UNIT_WORDS = ts.UNIT_WORDS


def units(size: int) -> int:
    return ts.units(size)


def owner(n_units: int, n: int, u: int) -> int:
    """The rank whose chunk holds unit u < n_units."""
    return ((u + 1) * n - 1) // n_units


def word_owner(size: int, n: int, word: int) -> int:
    return owner(units(size), n, word // UNIT_WORDS)


def unit_span(size: int, u: int) -> tuple:
    """(first word, end word) of unit u of a size-byte prefix."""
    return u * UNIT_WORDS, min((u + 1) * UNIT_WORDS, size // 8)


def rep(srcs, size: int, fault=None) -> list:
    """Every rank's output after one rep: srcs[j] is rank j's source words (at least size / 8 of them), fault
    (mode, rank, word) or None.  Wrapping 64-bit adds, in any order."""
    n, W, U = len(srcs), size // 8, units(size)
    area = [np.zeros(W, np.uint64) for _ in range(n)]
    for j in range(n):
        contrib = np.array(srcs[j][:W], dtype=np.uint64)
        times = [1] * U
        if fault is not None and fault[0] < 3 and fault[1] == j:
            mode, _, word = fault
            if mode == 0:
                contrib[word] += np.uint64(1)
            else:
                times[word // UNIT_WORDS] = 0 if mode == 1 else 2
        for u in range(U):
            lo, hi = unit_span(size, u)
            for _ in range(times[u]):
                area[owner(U, n, u)][lo:hi] += contrib[lo:hi]
    out = [a.copy() for a in area]
    for u in range(U):
        lo, hi = unit_span(size, u)
        o = owner(U, n, u)
        for t in range(1, n):
            out[(o + t) % n][lo:hi] = area[o][lo:hi]
    if fault is not None and fault[0] == 3:
        _, recv, word = fault
        out[recv][word] ^= np.uint64(1)
    return out


def failing(srcs, size: int, fault) -> dict:
    """{row: sorted word indices} that differ from the clean sum after the faulted rep, as the table above states."""
    mode, rank, word = fault
    n = len(srcs)
    if mode == 0:
        return {r: [word] for r in range(n)}
    if mode == 3:
        return {rank: [word]}
    lo, hi = unit_span(size, word // UNIT_WORDS)
    s = np.asarray(srcs[rank][lo:hi], dtype=np.uint64)
    words = [lo + int(i) for i in np.flatnonzero(s != 0)]
    return {r: words for r in range(n)} if words else {}


def busbw(algbw: float, n: int) -> float:
    return algbw * 2 * (n - 1) / n
