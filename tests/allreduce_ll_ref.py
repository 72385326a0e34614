"""Plain restatement of cdprobe_allreduce_ll's ladder, packet flags, salts and LL-area layout, for the tests
(include/cdprobe.h, DESIGN §5j).

    ladder               the bwcurve ladder's sizes of at most 1 MiB
    flag(call, k, r)     (call mod 2^16) << 16 | k << 8 | (r + 1)       r = 0: the warm-up
    salt(seed, j, flag)  splitmix64(seed ^ "LLSALT" ^ j << 56 ^ flag << 8)
    slot(p, n, s, w)     ((p n + s) S_max / 8 + w) x 16 bytes            in an area of 2 n 2 S_max bytes

Every rank ends a rep holding the whole all-reduce output, so what it must hold is allreduce_ref's."""
import bwcurve_ref
import word_ref

MAX_BYTES = 1 << 20
SALT_TAG = 0x4C4C53414C54  # "LLSALT"
M64 = (1 << 64) - 1


def ladder(bpp: int) -> list:
    return [s for s in bwcurve_ref.ladder(bpp) if s <= MAX_BYTES]


def flag(call_seq: int, k: int, r: int) -> int:
    return ((call_seq & 0xFFFF) << 16) | ((k & 0xFF) << 8) | ((r + 1) & 0xFF)


def salt(seed: int, j: int, fl: int) -> int:
    return int(word_ref.splitmix64((seed ^ SALT_TAG ^ (j << 56) ^ (fl << 8)) & M64)[0])


def slot(p: int, n: int, s: int, s_max: int, w: int) -> int:
    return ((p * n + s) * (s_max // 8) + w) * 16


def area_bytes(n: int, s_max: int) -> int:
    return 2 * n * 2 * s_max


def packet(word: int, fl: int) -> tuple:
    """The two 8-byte elements one input word travels as."""
    return (word & 0xFFFFFFFF) | (fl << 32), (word >> 32) | (fl << 32)
