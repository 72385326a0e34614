"""Plain CPU reference of the probe's word patterns and of what cdprobe_diagnose must report about one region.

Test helper, numpy only.  Restated from the pattern spec (DESIGN §5 and §5b, include/cdprobe.h, oracle/pattern.c's
header), not from the CUDA: every function works on whole uint64 arrays with wrap-around arithmetic, and the
inverses are derived here (modular inverses from Python's pow, xor-shifts undone by repeated shifting).

    src word k of rank r   splitmix64(seed ^ r << 56 ^ k)
    write salt             splitmix64(seed ^ 0x5752495445 ^ src << 56 ^ dst << 48 ^ run_seq)
    write word k           z ^ z >> 32,  z = (salt + k) * golden

A diagnosis compares a region word for word with the pattern of one cell and classifies each word that differs:
ZERO, then a pattern word from another place (DISPLACED / STALE / FOREIGN), else FLIP.
"""
from __future__ import annotations

import dataclasses
from typing import List

import numpy as np

M64 = (1 << 64) - 1
U64_MAX = M64
GOLDEN = 0x9E3779B97F4A7C15
MIX1 = 0xBF58476D1CE4E5B9
MIX2 = 0x94D049BB133111EB
WRITE_TAG = 0x5752495445  # "WRITE"
GRANULE_WORDS = 2048      # 16 KiB
STALE_RUNS = 8            # earlier runs of the same writer a STALE word is traced back to
SAMPLES = 16
FLIP, ZERO, DISPLACED, STALE, FOREIGN = 0, 1, 2, 3, 4

_u = np.uint64


def _arr(x) -> np.ndarray:
    return np.atleast_1d(np.asarray(x, dtype=np.uint64))


def splitmix64(x) -> np.ndarray:
    z = _arr(x) + _u(GOLDEN)
    z = (z ^ (z >> _u(30))) * _u(MIX1)
    z = (z ^ (z >> _u(27))) * _u(MIX2)
    return z ^ (z >> _u(31))


def _unxorshift(y: np.ndarray, s: int) -> np.ndarray:
    """Inverse of x -> x ^ (x >> s): x = y ^ y >> s ^ y >> 2s ^ ..."""
    x = y.copy()
    t = y
    for _ in range(64 // s):
        t = t >> _u(s)
        x ^= t
    return x


def unsplitmix64(z) -> np.ndarray:
    z = _unxorshift(_arr(z), 31)
    z = _unxorshift(z * _u(pow(MIX2, -1, 1 << 64)), 27)
    z = _unxorshift(z * _u(pow(MIX1, -1, 1 << 64)), 30)
    return z - _u(GOLDEN)


def src_words(seed: int, rank: int, first: int, n: int) -> np.ndarray:
    """Words first .. first + n - 1 of rank's source pattern."""
    k = np.arange(n, dtype=np.uint64) + _u(first)
    return splitmix64(_u(seed) ^ (_u(rank) << _u(56)) ^ k)


def write_salt(seed: int, src: int, dst: int, run_seq: int) -> int:
    x = seed ^ WRITE_TAG ^ ((src << 56) & M64) ^ ((dst << 48) & M64) ^ run_seq
    return int(splitmix64(x)[0])


def write_words(salt: int, first: int, n: int) -> np.ndarray:
    z = (np.arange(n, dtype=np.uint64) + _u(first) + _u(salt)) * _u(GOLDEN)
    return z ^ (z >> _u(32))


def unwrite_word(y) -> np.ndarray:
    """salt + k of a write-pattern word (the high half of z survives the xor-shift)."""
    y = _arr(y)
    return (y ^ (y >> _u(32))) * _u(pow(GOLDEN, -1, 1 << 64))


def fold6(g: int) -> int:
    f = 0
    while g:
        f ^= g & 63
        g >>= 6
    return f


# ---- what one cell's region must hold -------------------------------------------------------------------------
@dataclasses.dataclass
class Spec:
    seed: int
    n_ranks: int
    target: int
    n_words: int
    is_write: bool = False
    first_word: int = 0    # read: index of the region's word 0 in the target's source pattern
    src_words: int = 0     # read: words in one rank's source buffer
    issuer: int = 0        # write
    run_seq: int = 0       # write: the run whose pattern is expected

    def expected(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = self.n_words - first if n is None else n
        if self.is_write:
            return write_words(write_salt(self.seed, self.issuer, self.target, self.run_seq), first, n)
        return src_words(self.seed, self.target, self.first_word + first, n)

    def candidates(self):
        """Write cells: (salt, kind, rank, run_seq) in the order a word is matched against them."""
        c = [(self.issuer, self.run_seq, DISPLACED)]
        c += [(self.issuer, self.run_seq - d, STALE) for d in range(1, STALE_RUNS + 1) if d < self.run_seq]
        c += [(r, self.run_seq, FOREIGN) for r in range(self.n_ranks) if r != self.issuer]
        return [(write_salt(self.seed, w, self.target, seq), kind, w, seq) for w, seq, kind in c]


def read_spec(seed, n_ranks, target, first_word, n_words, src_words_) -> Spec:
    return Spec(seed=seed, n_ranks=n_ranks, target=target, n_words=n_words, first_word=first_word,
                src_words=src_words_)


def write_spec(seed, n_ranks, issuer, target, run_seq, n_words) -> Spec:
    return Spec(seed=seed, n_ranks=n_ranks, target=target, n_words=n_words, is_write=True, issuer=issuer,
                run_seq=run_seq)


def classify(spec: Spec, observed):
    """Class of each observed word that differs from the expected one: arrays (kind, rank, word, run_seq)."""
    obs = _arr(observed)
    n = len(obs)
    kind = np.full(n, FLIP, dtype=np.int64)
    rank = np.full(n, -1, dtype=np.int64)
    word = np.zeros(n, dtype=np.uint64)
    seq = np.zeros(n, dtype=np.uint64)
    zero = obs == 0
    kind[zero] = ZERO
    if not spec.is_write:
        x = unsplitmix64(obs) ^ _u(spec.seed)
        r = x >> _u(56)
        k = x & _u((1 << 56) - 1)
        hit = ~zero & (r < _u(spec.n_ranks)) & (k < _u(spec.src_words))
        kind[hit] = np.where(r[hit] == _u(spec.target), DISPLACED, FOREIGN)
        rank[hit] = r[hit].astype(np.int64)
        word[hit] = k[hit]
        return kind, rank, word, seq
    z = unwrite_word(obs)
    open_ = ~zero
    for salt, c_kind, c_rank, c_seq in spec.candidates():
        k = z - _u(salt)
        hit = open_ & (k < _u(spec.n_words))
        kind[hit] = c_kind
        rank[hit] = c_rank
        word[hit] = k[hit]
        if c_kind == STALE:
            seq[hit] = c_seq
        open_ &= ~hit
    return kind, rank, word, seq


def expected_report(spec: Spec, observed_words) -> dict:
    """The fields cdprobe_diagnose fills from the bytes of a region that holds `observed_words`."""
    obs = _arr(observed_words)
    assert len(obs) == spec.n_words
    exp = spec.expected()
    bad = np.nonzero(obs != exp)[0]
    kind, rank, word, seq = classify(spec, obs[bad])
    flips = [0] * 64
    d = exp[bad][kind == FLIP] ^ obs[bad][kind == FLIP]
    for b in range(64):
        flips[b] = int(np.count_nonzero((d >> _u(b)) & _u(1)))
    samples: List[dict] = [
        {"offset": int(k) * 8, "expected": int(exp[k]), "observed": int(obs[k]), "kind": int(kind[i]),
         "rank": int(rank[i]), "word": int(word[i]), "run_seq": int(seq[i])}
        for i, k in enumerate(bad[:SAMPLES])]
    return {
        "bad_words": len(bad),
        "bad_granules": len(np.unique(bad // GRANULE_WORDS)),
        "first_bad": int(bad[0]) * 8 if len(bad) else U64_MAX,
        "last_bad": int(bad[-1]) * 8 if len(bad) else 0,
        "zero_words": int(np.count_nonzero(kind == ZERO)),
        "kind_count": [int(np.count_nonzero(kind == c)) for c in range(5)],
        "bit_flips": flips,
        "n_samples": min(SAMPLES, len(bad)),
        "sample": samples,
    }
