"""Plain restatement of cdprobe_ce_alltoall for the tests: which cells copy in every rep, who owns and checks each
block, the words and (S, X) every ladder prefix must land, the flag values, the hardware queues a process needs, and
what each armed fault does to the word checks.  The blocks are cdprobe_memcpy's, so it builds on memcpy_ref; it
follows the doc comments of cdprobe_ce_alltoall and cdprobe_ce_alltoall_t in include/cdprobe.h and DESIGN §5p."""
import memcpy_ref
from memcpy_ref import OP_READ, OP_WRITE, ladder  # noqa: F401

U64_MAX = (1 << 64) - 1
DEFAULT_QUEUES = 8


def cells(n: int, diag: bool):
    """Every cell (issuer, target) of the domain, all copied in every rep: each rank to every peer, and to itself with a
    loop-back slice (n == 1 or LOCAL_DIAG)."""
    diag = diag or n == 1
    return [(g, j) for g in range(n) for j in range(n) if g != j or diag]


def owner(op: int, g: int, j: int) -> int:
    """The rank whose exchange area receives cell (g, j) and which checks it: the issuer on a pull, the target on a
    push."""
    return j if op == OP_WRITE else g


def expected(oracle, seed: int, n: int, bpp: int, mode: int, op: int, g: int, j: int, sizes) -> list:
    """(S, X) of every ladder prefix of cell (g, j)'s block: the words of its source slice, as in cdprobe_memcpy."""
    return memcpy_ref.expected(oracle, seed, memcpy_ref.cell(n, bpp, mode, op, g, j), sizes)


def value(call_seq: int, k: int, rep: int, reps: int) -> int:
    """The value rep `rep` (0: the warm-up) of size k of call call_seq opens and lands with."""
    return (call_seq << 16) | (k * (reps + 1) + rep + 1)


def queues(n: int, diag: bool, ordinals) -> tuple:
    """(need, ordinal): the streams one process holds on its most loaded device, each local rank's own plus one copy
    stream per cell it issues (n - 1 peers, and itself with a loop-back slice), and that device (the lowest ordinal on
    a tie)."""
    per_rank = 1 + (n - 1) + (1 if diag else 0)
    load = {o: per_rank * list(ordinals).count(o) for o in ordinals}
    need = max(load.values())
    return need, min(o for o in load if load[o] == need)


def queue_message(need: int, ordinal: int, limit: int) -> str:
    return f"needs {need} queues on ordinal {ordinal}, CUDA_DEVICE_MAX_CONNECTIONS allows {limit}"


def fault_words(mode: int, size: int, arg: int):
    """(bad_words, first_bad) of the faulted cell's size: mode 0 flips one word in rep 1; mode 1 lands nothing in rep 1,
    so every word of the cleared block reads 0; mode 2 only delays the copy."""
    if mode == 0:
        return 1, 8 * arg
    if mode == 1:
        return size // 8, 0
    return 0, U64_MAX
