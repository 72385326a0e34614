"""Plain CPU references that stream, for regions too large to hold in host memory: the (S, X) of every ladder prefix
of a pattern, of the all-reduce's output, and the whole cdprobe_diagnose report of a region that is the pattern except
at a few listed words.

Restated from the pattern and checksum definitions (DESIGN §5, oracle/pattern.c's header) in numpy, in chunks of at
most CHUNK_WORDS words, so a 16 GiB region costs 64 MiB of host memory at a time:

    S    sum of the words mod 2^64
    X    xor over 16 KiB granules g of rotl64(xor of the granule's words, fold6(g)); a prefix that ends inside a
         granule closes that partial granule with the words it holds

The diagnosis report is word_ref.expected_report's, computed from the listed words alone: a word not listed holds the
pattern, so it can be neither bad nor sampled."""
from __future__ import annotations

import collections
from typing import Callable, Iterable, List, Optional, Tuple

import numpy as np

import word_ref

CHUNK_WORDS = 8 << 20          # 64 MiB of uint64 words
G = word_ref.GRANULE_WORDS     # 2048 words, 16 KiB
U64_MAX = word_ref.U64_MAX
_u = np.uint64

WordFn = Callable[[int, int], np.ndarray]


def src_fn(seed: int, rank: int, first: int = 0) -> WordFn:
    """word_fn of rank's source pattern from its word `first` on."""
    return lambda k, n: word_ref.src_words(seed, rank, first + k, n)


def write_fn(seed: int, src: int, dst: int, run_seq: int) -> WordFn:
    """word_fn of the write pattern src lands in dst's slot in run run_seq."""
    salt = word_ref.write_salt(seed, src, dst, run_seq)
    return lambda k, n: word_ref.write_words(salt, k, n)


def _fold6(g: np.ndarray) -> np.ndarray:
    f = np.zeros_like(g)
    g = g.copy()
    while g.any():
        f ^= g & _u(63)
        g >>= _u(6)
    return f


def _rotl(x: np.ndarray, r: np.ndarray) -> np.ndarray:
    """rotl64 elementwise; r == 0 gives x | x."""
    return (x << r) | (x >> ((_u(64) - r) & _u(63)))


def prefix_sums(word_fn: WordFn, n_words: int, sizes: Iterable[int]) -> List[Tuple[int, int]]:
    """(S, X) of the first s bytes of the region whose words word_fn(first, n) gives, for every s in `sizes` (multiples
    of 8, at most 8 n_words), in one pass over the largest."""
    sizes = list(sizes)
    assert all(s % 8 == 0 and 0 < s <= 8 * n_words for s in sizes), sizes
    cuts = sorted({s // 8 for s in sizes})
    at = {}
    s_acc = 0
    x_acc = _u(0)          # the complete granules
    gx = _u(0)             # xor of the words of the open granule (k % G words of it)
    k = 0
    for c in cuts:
        while k < c:
            n = min(CHUNK_WORDS - k % CHUNK_WORDS, c - k)  # chunks stay granule-aligned away from the cuts
            w = word_fn(k, n)
            assert len(w) == n and w.dtype == np.uint64
            s_acc = (s_acc + int(w.sum(dtype=np.uint64))) & word_ref.M64
            head, end = k % G, k + n
            rows = -(-(head + n) // G)
            if head == 0 and n % G == 0:
                gxs = np.bitwise_xor.reduce(w.reshape(rows, G), axis=1)
            else:
                buf = np.zeros(rows * G, dtype=np.uint64)
                buf[head:head + n] = w
                gxs = np.bitwise_xor.reduce(buf.reshape(rows, G), axis=1)
            gxs[0] ^= gx
            g0 = k // G
            if end % G:
                gx = gxs[-1]
                gxs = gxs[:-1]
            else:
                gx = _u(0)
            if len(gxs):
                idx = np.arange(g0, g0 + len(gxs), dtype=np.uint64)
                x_acc ^= np.bitwise_xor.reduce(_rotl(gxs, _fold6(idx)))
            k = end
        x = x_acc
        if k % G:
            x = x ^ _rotl(np.array([gx]), _fold6(np.array([k // G], dtype=np.uint64)))[0]
        at[c] = (s_acc, int(x))
    return [at[s // 8] for s in sizes]


AllReduceSums = collections.namedtuple("AllReduceSums", "sum xr bad_words first_bad")


def allreduce_sums(seed: int, n: int, sizes: Iterable[int],
                   corrupt: Optional[Tuple[int, int, int]] = None) -> List[AllReduceSums]:
    """For every size: (S, X) of the output prefix of an n-rank all-reduce, word w = sum over ranks j < n of src word
    w of rank j mod 2^64, and the word check of that prefix against the clean sum (bad_words per checked rep, and
    first_bad, the byte offset of the lowest bad word or U64_MAX).  corrupt = (rank, word, mask): that source word is
    xored with mask at rest."""
    sizes = list(sizes)

    def words(k, m):
        out = np.zeros(m, dtype=np.uint64)
        for j in range(n):
            w = word_ref.src_words(seed, j, k, m)
            if corrupt is not None and corrupt[0] == j and k <= corrupt[1] < k + m:
                w[corrupt[1] - k] ^= _u(corrupt[2])
            out += w
        return out

    sums = prefix_sums(words, max(sizes) // 8, sizes)
    out = []
    for s, (sm, xr) in zip(sizes, sums):
        hit = corrupt is not None and corrupt[2] != 0 and corrupt[1] < s // 8
        out.append(AllReduceSums(sm, xr, 1 if hit else 0, 8 * corrupt[1] if hit else U64_MAX))
    return out


def _expected_at(spec: word_ref.Spec, idx: np.ndarray) -> np.ndarray:
    """The pattern's words at region word indices idx (any order), without building the region."""
    if spec.is_write:
        z = (idx + _u(word_ref.write_salt(spec.seed, spec.issuer, spec.target, spec.run_seq))) * _u(word_ref.GOLDEN)
        return z ^ (z >> _u(32))
    return word_ref.splitmix64(_u(spec.seed) ^ (_u(spec.target) << _u(56)) ^ (idx + _u(spec.first_word)))


def sparse_report(spec: word_ref.Spec, faults: Iterable[Tuple[int, int]]) -> dict:
    """word_ref.expected_report of a region that holds spec's pattern except word k holds `observed`, for each
    (k, observed) of `faults` (a later pair for the same k wins)."""
    obs_at = {int(k): int(v) for k, v in faults}
    assert all(0 <= k < spec.n_words for k in obs_at), "a fault outside the region"
    idx = np.array(sorted(obs_at), dtype=np.uint64)
    obs = np.array([obs_at[int(k)] for k in idx], dtype=np.uint64)
    exp = _expected_at(spec, idx)
    bad_i = np.flatnonzero(obs != exp)
    bad, obs_b, exp_b = idx[bad_i], obs[bad_i], exp[bad_i]
    kind, rank, word, seq = word_ref.classify(spec, obs_b)
    d = exp_b[kind == word_ref.FLIP] ^ obs_b[kind == word_ref.FLIP]
    flips = [int(np.count_nonzero((d >> _u(b)) & _u(1))) for b in range(64)]
    samples = [{"offset": int(bad[i]) * 8, "expected": int(exp_b[i]), "observed": int(obs_b[i]), "kind": int(kind[i]),
                "rank": int(rank[i]), "word": int(word[i]), "run_seq": int(seq[i])}
               for i in range(min(word_ref.SAMPLES, len(bad)))]
    return {
        "bad_words": len(bad),
        "bad_granules": len(np.unique(bad // _u(G))),
        "first_bad": int(bad[0]) * 8 if len(bad) else U64_MAX,
        "last_bad": int(bad[-1]) * 8 if len(bad) else 0,
        "zero_words": int(np.count_nonzero(kind == word_ref.ZERO)),
        "kind_count": [int(np.count_nonzero(kind == c)) for c in range(5)],
        "bit_flips": flips,
        "n_samples": min(word_ref.SAMPLES, len(bad)),
        "sample": samples,
    }
