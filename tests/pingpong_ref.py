"""Plain CPU restatement of cdprobe_pingpong's words and digests, for the tests.

Restated from the spec (DESIGN §5d, include/cdprobe.h), not from the CUDA, in Python integers.  In round r of the
tournament a rank and its partner run two legs, the lower rank initiating in leg 0.  A leg is rep 0 (the warm-up)
and reps timed reps of `trips` round trips; trip t of a rep sends

    ping = word(call_seq, r, leg, rep, t, 0)        echo = word(call_seq, r, leg, rep, t, 1)

    word = call_seq << 29 | round << 25 | leg << 24 | rep << 17 | (2 * trip + echo)

The digest of cell (initiator, target) is the xor of every echo word the initiator received over reps 0 .. reps.  With
the skip-ahead fault armed at trip f, the responder answers trip f of rep 1 with the echo of trip f + 1; the
initiator then receives that word at trip f and, its next wait being already satisfied, the same word at trip f + 1.
"""
from __future__ import annotations

from typing import Optional, Sequence

M64 = (1 << 64) - 1


def word(call_seq: int, rnd: int, leg: int, rep: int, trip: int, echo: int) -> int:
    assert 0 <= 2 * trip + echo < 1 << 17 and 0 <= rep < 1 << 7 and leg in (0, 1) and 0 <= rnd < 16
    assert 0 < call_seq < 1 << 35
    return (call_seq << 29) | (rnd << 25) | (leg << 24) | (rep << 17) | (2 * trip + echo)


def received(call_seq: int, rnd: int, leg: int, trips: int, reps: int, fault_trip: Optional[int] = None):
    """Every echo word the initiator receives in one leg, in order."""
    for rep in range(reps + 1):
        for t in range(trips):
            skip = fault_trip is not None and rep == 1 and t == fault_trip
            yield word(call_seq, rnd, leg, rep, t + 1 if skip else t, 1)


def leg_digest(call_seq: int, rnd: int, leg: int, trips: int, reps: int, fault_trip: Optional[int] = None) -> int:
    d = 0
    for w in received(call_seq, rnd, leg, trips, reps, fault_trip):
        d ^= w
    return d


def cell_round(partner: Sequence[Sequence[int]], rounds: int, i: int, j: int) -> int:
    """The round in which i and j are partners (partner[round][rank] of cdprobe_plan)."""
    rs = [r for r in range(rounds) if partner[r][i] == j]
    assert len(rs) == 1 and partner[rs[0]][j] == i, (i, j, rs)
    return rs[0]


def cell_digest(call_seq: int, partner, rounds: int, i: int, j: int, trips: int, reps: int,
                fault_trip: Optional[int] = None) -> int:
    """What cdprobe_pingpong reports as the digest of cell (initiator i, target j)."""
    return leg_digest(call_seq, cell_round(partner, rounds, i, j), 0 if i < j else 1, trips, reps, fault_trip)


def fault_value(initiator: int, target: int, trip: int) -> int:
    """CDPROBE_OPT_PINGPONG_FAULT's encoding."""
    return ((initiator + 1) << 32) | ((target + 1) << 16) | trip
