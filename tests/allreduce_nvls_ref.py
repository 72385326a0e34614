"""Plain restatement of one rep of cdprobe_allreduce_nvls and of what each armed fault does to it, for the tests
(include/cdprobe.h, DESIGN §5m).

    NVLS area         per rank: input [0, s_max), output [s_max, 2 s_max), s_max the ladder's largest size
    chunks            the two-shot's: rank r owns units [floor(r U / n), floor((r + 1) U / n)), U = ceil(size / 8 KiB)
    reduce            the owner of each unit reads each of its words with multimem.ld_reduce .add.u64: the wrapping
                      sum of that word over every member's input
    store             the owner stores each summed 16 bytes with one multimem.st: into every member's output at once
    bus bandwidth     algorithm bandwidth x 2 (n - 1) / n

Fault (mode, word), in the rep it is armed for, acted on by the word's owner:

    mode 0   the owner stores the word xored with 1           every row, one bad word at 8 word
    mode 1   the owner skips the store of the word's unit      every row, the unit's words whose sum is not 0

Every rank ends a clean rep holding the whole all-reduce output, so what it must hold is allreduce_ref's."""
import numpy as np

import allreduce_push_ref as push

UNIT_BYTES = push.UNIT_BYTES
UNIT_WORDS = push.UNIT_WORDS
units = push.units
owner = push.owner
word_owner = push.word_owner
unit_span = push.unit_span


def rep(srcs, size: int, fault=None) -> list:
    """Every rank's output after one rep: srcs[j] is rank j's source words (at least size / 8 of them), fault
    (mode, word) or None.  Wrapping 64-bit adds."""
    n, W = len(srcs), size // 8
    total = np.zeros(W, np.uint64)
    for j in range(n):
        total += np.asarray(srcs[j][:W], dtype=np.uint64)
    stored = total.copy()
    if fault is not None:
        mode, word = fault
        if mode == 0:
            stored[word] ^= np.uint64(1)
        else:
            lo, hi = unit_span(size, word // UNIT_WORDS)
            stored[lo:hi] = 0
    return [stored.copy() for _ in range(n)]


def failing(srcs, size: int, fault) -> dict:
    """{row: sorted word indices} that differ from the clean sum after the faulted rep, as the table above states."""
    mode, word = fault
    n = len(srcs)
    if mode == 0:
        return {r: [word] for r in range(n)}
    lo, hi = unit_span(size, word // UNIT_WORDS)
    total = np.zeros(hi - lo, np.uint64)
    for s in srcs:
        total += np.asarray(s[lo:hi], dtype=np.uint64)
    words = [lo + int(i) for i in np.flatnonzero(total != 0)]
    return {r: words for r in range(n)} if words else {}


def busbw(algbw: float, n: int) -> float:
    return algbw * 2 * (n - 1) / n
