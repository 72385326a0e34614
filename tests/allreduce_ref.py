"""Plain restatement of what cdprobe_allreduce must leave in every rank's output, and of its (S, X), for the tests.

Numpy only, from include/cdprobe.h and the checksum definition (DESIGN §5), not from the CUDA:

    output word w    sum over ranks j < n of src word w of rank j, mod 2^64 (the same on every rank)
    S                sum of the words mod 2^64
    X                xor over 16 KiB granules g of rotl64(xor of the words of granule g, fold6(g))

The size ladder and the per-row summary are cdprobe_bwcurve's (bwcurve_ref)."""
import functools

import numpy as np

import word_ref
from bwcurve_ref import ladder, summary  # noqa: F401  (the all-reduce uses bwcurve's ladder and summary)

GRANULE_WORDS = word_ref.GRANULE_WORDS
U64_MAX = word_ref.U64_MAX
_u = np.uint64


def output_words(seed: int, n: int, n_words: int) -> np.ndarray:
    """Words 0 .. n_words - 1 of the output of an n-rank all-reduce."""
    out = np.zeros(n_words, dtype=np.uint64)
    for j in range(n):
        out += word_ref.src_words(seed, j, 0, n_words)
    return out


def checksum(words) -> tuple:
    """(S, X) of a word array."""
    w = np.asarray(words, dtype=np.uint64)
    s = int(w.sum(dtype=np.uint64))
    ng = (len(w) + GRANULE_WORDS - 1) // GRANULE_WORDS
    if ng == 0:
        return s, 0
    padded = np.zeros(ng * GRANULE_WORDS, dtype=np.uint64)
    padded[:len(w)] = w
    gx = np.bitwise_xor.reduce(padded.reshape(ng, GRANULE_WORDS), axis=1)
    r = np.array([word_ref.fold6(g) for g in range(ng)], dtype=np.uint64)
    rot = np.where(r == 0, gx, (gx << r) | (gx >> ((_u(64) - r) % _u(64))))
    return s, int(np.bitwise_xor.reduce(rot))


@functools.lru_cache(maxsize=None)
def expected(seed: int, n: int, sizes: tuple) -> tuple:
    """((S, X) of the output prefix of every size in `sizes`), computing the output words once."""
    words = output_words(seed, n, max(sizes) // 8)
    return tuple(checksum(words[:s // 8]) for s in sizes)


def expected_corrupted(seed: int, n: int, sizes, rank: int, word: int, mask: int) -> list:
    """(S, X) of every prefix when word `word` of rank's source buffer is xored with `mask` at rest."""
    words = output_words(seed, n, max(sizes) // 8)
    if word < len(words):
        orig = int(word_ref.src_words(seed, rank, word, 1)[0])
        words[word] = _u((int(words[word]) - orig + (orig ^ mask)) % (1 << 64))
    return [checksum(words[:s // 8]) for s in sizes]
