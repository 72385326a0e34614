"""Plain restatement of what cdprobe_alltoall must deliver into every receiver's exchange area, and of its (S, X), for
the tests.

From include/cdprobe.h and the pattern definition (DESIGN §5), not from the CUDA:

    sequence value   alltoall_seq(call_seq, k, r) = 2^63 | (call_seq mod 2^51) << 12 | k << 7 | r
    block word w     write_word(write_salt(seed, sender, receiver, alltoall_seq(call_seq, k, r)), w)
    blocks of rank   its cells that run: rank + 1, rank + 2, ... (mod n), then the diagonal with a loop-back slice

The size ladder and the checksum are bwcurve's and the all-reduce's; the per-rank summary is bwcurve's with the rates
scaled by the blocks a rank pushes (egress)."""
import numpy as np

import word_ref
from allreduce_ref import checksum  # noqa: F401  (the (S, X) definition)
from bwcurve_ref import ladder, summary as _summary  # noqa: F401

U64_MAX = word_ref.U64_MAX


def alltoall_seq(call_seq: int, k: int, r: int) -> int:
    return (1 << 63) | ((call_seq % (1 << 51)) << 12) | ((k & 31) << 7) | (r & 127)


def block_words(seed: int, sender: int, receiver: int, call_seq: int, k: int, r: int, n_words: int) -> np.ndarray:
    """The first n_words words of block (sender -> receiver) in rep r of size k of call call_seq."""
    salt = word_ref.write_salt(seed, sender, receiver, alltoall_seq(call_seq, k, r))
    return word_ref.write_words(salt, 0, n_words)


def expected(seed: int, sender: int, receiver: int, call_seq: int, reps: int, sizes) -> list:
    """(S, X) the receiver folds for every size: the block of the last timed rep (r = reps)."""
    return [checksum(block_words(seed, sender, receiver, call_seq, k, reps, s // 8)) for k, s in enumerate(sizes)]


def block_order(rank: int, n: int, runs) -> list:
    """The receivers of rank's blocks, in the order its walk interleaves them; runs(s, d) says whether a cell runs."""
    order = [(rank + d) % n for d in range(1, n)] + [rank]
    return [j for j in order if runs(rank, j)]


def summary(sizes, medians, blocks):
    """(t0_ns, peak_gbps, half_bytes) of a rank: bwcurve's summary with egress rates blocks x size / median."""
    t0, peak, half = _summary([blocks * s for s in sizes], medians)
    return t0, peak, sizes[[blocks * s for s in sizes].index(half)]
