"""Plain restatement of cdprobe_allreduce_ring's steps, faults, flags and ring-area layout, for the tests
(include/cdprobe.h, DESIGN §5k).

    chunks                   the two-shot's: rank r's chunk is units [floor(r U / n), floor((r + 1) U / n))
    reduce-scatter step s    rank g pushes chunk (g - 1 - s) mod n to g + 1: every chunk but g
    all-gather step s        rank g pushes chunk (g - s) mod n to g + 1: every chunk but g + 1
    flag(call, k, r, phase)  (call mod 2^16) << 16 | k << 8 | phase << 7 | (r + 1)       r = 0: the warm-up
    ring area                s_max output bytes, up to the next 128, then one 32-bit flag per 8 KiB unit of s_max
    bus bandwidth            algorithm bandwidth x 2 (n - 1) / n

Every rank ends a rep holding the whole all-reduce output, so what it must hold is allreduce_ref's."""
import allreduce_ll_ref
import allreduce_twoshot_ref as ts

UNIT_BYTES = ts.UNIT_BYTES
UNIT_WORDS = ts.UNIT_WORDS


def pushed_chunk(n: int, g: int, s: int, phase: int) -> int:
    """The chunk rank g pushes to g + 1 at step s of the reduce-scatter (phase 0) or the all-gather (phase 1)."""
    return (g - 1 - s) % n if phase == 0 else (g - s) % n


def pushes(n: int, g: int, phase: int) -> set:
    """Every chunk rank g pushes in a phase."""
    return {pushed_chunk(n, g, s, phase) for s in range(n - 1)}


def chunk_of(size: int, n: int, word: int) -> int:
    """The chunk (its owner rank) that holds output word `word` of a size-byte prefix."""
    return ts.owner(size, n, word)


def partial_ranks(n: int, g: int, c: int) -> list:
    """The ranks whose inputs the partial of chunk c that rank g pushes in the reduce-scatter sums: g - s ... g."""
    s = (g - 1 - c) % n
    return [(g - s + i) % n for i in range(s + 1)]


def failing_rows(n: int, sender: int, phase: int, size: int, word: int) -> list:
    """The rows a corrupted (mode 0) or dropped (mode 1) push of `word` by `sender` fails: every row in the
    reduce-scatter, whose error enters the full sum; in the all-gather the rows downstream of the hop, sender + 1 up to
    the rank just before the chunk's owner."""
    if phase == 0:
        return list(range(n))
    c = chunk_of(size, n, word)
    return [(sender + 1 + i) % n for i in range((c - sender - 2) % n + 1)]


def flag(call_seq: int, k: int, r: int, phase: int) -> int:
    return allreduce_ll_ref.flag(call_seq, k, r) | (phase << 7)


def units(size: int) -> int:
    return ts.units(size)


def flags_off(s_max: int) -> int:
    return (s_max + 127) // 128 * 128


def flag_off(s_max: int, u: int) -> int:
    return flags_off(s_max) + 4 * u


def area_bytes(s_max: int) -> int:
    return flag_off(s_max, units(s_max))


def busbw(algbw: float, n: int) -> float:
    return algbw * 2 * (n - 1) / n
