"""Plain CPU restatement of cdprobe_atomics' values and digests, for the tests.

Restated from the spec (DESIGN §5e, include/cdprobe.h), not from the CUDA, in Python integers.  Rep `rep` of a call
opens by storing its start value into the cell's word

    start = (call_seq mod 2^32) << 31 | kind << 29 | rep << 22

then `lanes * ops` increments follow, so the values they return are start, start + 1, ..., start + lanes * ops - 1, in
some order for CONTENDED and in op order for the chains.  The digest of a cell is the xor of every returned value over
reps 0 (the warm-up) .. reps.

With the fault armed on a cell, the first op of timed rep 1 steps the word by 2 instead of 1: a FETCH_ADD chain then
returns start, start + 2, ..., start + ops; a CAS chain returns start once and then, its compare (the last return + 1)
never matching again, start + 2 for every later op.
"""
from __future__ import annotations

FETCH_ADD, CAS, CONTENDED = 0, 1, 2
M64 = (1 << 64) - 1


def lanes(kind: int) -> int:
    return 32 if kind == CONTENDED else 1


def start(call_seq: int, kind: int, rep: int) -> int:
    assert 0 <= kind <= 2 and 0 <= rep <= 64 and call_seq >= 0
    return ((call_seq & 0xFFFFFFFF) << 31) | (kind << 29) | (rep << 22)


def range_xor(first: int, count: int) -> int:
    d = 0
    for v in range(first, first + count):
        d ^= v
    return d


def range_sum(first: int, count: int) -> int:
    return sum(range(first, first + count)) & M64


def chain_returns(s: int, kind: int, ops: int, fault: bool = False):
    """What one lane's chain returns in one rep that opened with `s`, simulating the word."""
    word, out = s, []
    for k in range(ops):
        step = 2 if fault and k == 0 else 1
        if kind == FETCH_ADD:
            out.append(word)
            word += step
        else:
            cmp = s if k == 0 else out[-1] + 1
            out.append(word)
            if word == cmp:
                word = cmp + step
    return out, word


def rep_digest(call_seq: int, kind: int, rep: int, ops: int, fault: bool = False) -> int:
    s = start(call_seq, kind, rep)
    if kind == CONTENDED:
        assert not fault, "a faulted contended rep has no fixed digest"
        return range_xor(s, 32 * ops)
    d = 0
    for v in chain_returns(s, kind, ops, fault)[0]:
        d ^= v
    return d


def cell_digest(call_seq: int, kind: int, ops: int, reps: int, fault: bool = False) -> int:
    """What cdprobe_atomics reports as a cell's digest: reps 0 .. reps, the fault (if armed) in timed rep 1."""
    d = 0
    for rep in range(reps + 1):
        d ^= rep_digest(call_seq, kind, rep, ops, fault and rep == 1)
    return d


def fault_value(issuer: int, target: int) -> int:
    """CDPROBE_OPT_ATOMICS_FAULT's encoding."""
    return ((issuer + 1) << 16) | (target + 1)
