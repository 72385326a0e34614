"""Plain restatement of how cdprobe_allreduce_twoshot splits the work, for the tests (include/cdprobe.h, DESIGN §5i).

    units of a size      U = ceil(size / 8 KiB)
    rank r's chunk       units [floor(r U / n), floor((r + 1) U / n))
    bus bandwidth        algorithm bandwidth x 2 (n - 1) / n, the nccl-tests figure

Every rank ends a rep holding the whole all-reduce output, so what it must hold is allreduce_ref's."""
UNIT_BYTES = 8192
UNIT_WORDS = UNIT_BYTES // 8


def units(size: int) -> int:
    return (size + UNIT_BYTES - 1) // UNIT_BYTES


def chunk(n_units: int, n: int, r: int) -> tuple:
    """(lo, hi): the units rank r of n reduces."""
    return n_units * r // n, n_units * (r + 1) // n


def owner(size: int, n: int, word: int) -> int:
    """The rank whose chunk of a size-byte prefix holds output word `word`."""
    u = word // UNIT_WORDS
    return next(r for r in range(n) if chunk(units(size), n, r)[0] <= u < chunk(units(size), n, r)[1])


def unit_words(size: int, word: int) -> int:
    """Words of the size-byte prefix in the 8 KiB unit that holds `word`."""
    u = word // UNIT_WORDS
    return min(UNIT_WORDS, size // 8 - u * UNIT_WORDS)


def busbw(algbw: float, n: int) -> float:
    return algbw * 2 * (n - 1) / n
