"""The Python binding without a GPU: every measurement's from_c against one table of when each field is None, over
seeded random results, and every fault encoder's fields at the edges of their widths."""
import dataclasses
import random

import numpy as np
import pytest

M = 16  # CDPROBE_MAX_GPUS: the stride of a cell array
ERR_TIMEOUT = -5
CELL, RANK = "cell", "rank"  # an n x n matrix [s][d] of a MAX_GPUS-strided array, or a list over ranks [s]
SIZED = True  # each kept entry is a list over the ladder's n_sizes


# When an entry (s, d) of a field is kept; elsewhere it is None.  d is None for a rank field.
def always(t, s, d):
    return True


def measured(t, s, d):
    return bool(t.measured[s if d is None else s * M + d])


def timed(t, s, d):
    k = s if d is None else s * M + d
    return bool(t.measured[k]) and t.status[k] != ERR_TIMEOUT


def checked(t, s, d):
    return bool(t.cell_measured[s * M + d]) and t.cell_status[s * M + d] != ERR_TIMEOUT


def local_row(t, s, d):
    return bool(t.row_mask >> s & 1)


def issued(t, s, d):
    # rank s issues a cell to every peer, and to itself only with a loop-back slice (then it copies n blocks)
    return bool(t.measured[s]) and (s != d or t.blocks[s] == t.n)


RULES = [  # (result type, field, shape, sized, kept where)
    ("Latency", "measured", CELL, False, always),
    ("Latency", "status", CELL, False, always),
    ("Latency", "ns_min", CELL, False, timed),
    ("Latency", "ns_median", CELL, False, timed),
    ("Latency", "ns_max", CELL, False, timed),
    ("Latency", "digest", CELL, False, measured),
    ("PingPong", "measured", CELL, False, always),
    ("PingPong", "status", CELL, False, always),
    ("PingPong", "ns_min", CELL, False, timed),
    ("PingPong", "ns_median", CELL, False, timed),
    ("PingPong", "ns_max", CELL, False, timed),
    ("PingPong", "digest", CELL, False, measured),
    ("Atomics", "native", CELL, False, local_row),
    ("Atomics", "measured", CELL, False, always),
    ("Atomics", "status", CELL, False, always),
    ("Atomics", "ns_min", CELL, False, timed),
    ("Atomics", "ns_median", CELL, False, timed),
    ("Atomics", "ns_max", CELL, False, timed),
    ("Atomics", "digest", CELL, False, measured),
    ("BwCurve", "measured", CELL, False, always),
    ("BwCurve", "status", CELL, False, always),
    ("BwCurve", "bad_sizes", CELL, False, timed),
    ("BwCurve", "t0_ns", CELL, False, timed),
    ("BwCurve", "peak_gbps", CELL, False, timed),
    ("BwCurve", "half_bytes", CELL, False, timed),
    ("BwCurve", "ns_min", CELL, SIZED, timed),
    ("BwCurve", "ns_median", CELL, SIZED, timed),
    ("BwCurve", "ns_max", CELL, SIZED, timed),
    ("BwCurve", "sum", CELL, SIZED, timed),
    ("BwCurve", "xr", CELL, SIZED, timed),
    ("Memcpy", "measured", CELL, False, always),
    ("Memcpy", "status", CELL, False, always),
    ("Memcpy", "bad_sizes", CELL, False, timed),
    ("Memcpy", "t0_ns", CELL, False, timed),
    ("Memcpy", "peak_gbps", CELL, False, timed),
    ("Memcpy", "half_bytes", CELL, False, timed),
    ("Memcpy", "ns_min", CELL, SIZED, timed),
    ("Memcpy", "ns_median", CELL, SIZED, timed),
    ("Memcpy", "ns_max", CELL, SIZED, timed),
    ("Memcpy", "sum", CELL, SIZED, timed),
    ("Memcpy", "xr", CELL, SIZED, timed),
    ("Memcpy", "bad_words", CELL, SIZED, timed),
    ("Memcpy", "first_bad", CELL, SIZED, timed),
    ("AllReduce", "measured", RANK, False, always),
    ("AllReduce", "status", RANK, False, always),
    ("AllReduce", "bad_sizes", RANK, False, timed),
    ("AllReduce", "t0_ns", RANK, False, timed),
    ("AllReduce", "peak_gbps", RANK, False, timed),
    ("AllReduce", "half_bytes", RANK, False, timed),
    ("AllReduce", "ns_min", RANK, SIZED, timed),
    ("AllReduce", "ns_median", RANK, SIZED, timed),
    ("AllReduce", "ns_max", RANK, SIZED, timed),
    ("AllReduce", "sum", RANK, SIZED, timed),
    ("AllReduce", "xr", RANK, SIZED, timed),
    ("AllReduce", "bad_words", RANK, SIZED, timed),
    ("AllReduce", "first_bad", RANK, SIZED, timed),
    ("AllToAll", "measured", RANK, False, always),
    ("AllToAll", "status", RANK, False, always),
    ("AllToAll", "blocks", RANK, False, measured),
    ("AllToAll", "t0_ns", RANK, False, timed),
    ("AllToAll", "peak_gbps", RANK, False, timed),
    ("AllToAll", "half_bytes", RANK, False, timed),
    ("AllToAll", "ns_min", RANK, SIZED, timed),
    ("AllToAll", "ns_median", RANK, SIZED, timed),
    ("AllToAll", "ns_max", RANK, SIZED, timed),
    ("AllToAll", "cell_measured", CELL, False, always),
    ("AllToAll", "cell_status", CELL, False, always),
    ("AllToAll", "bad_sizes", CELL, False, checked),
    ("AllToAll", "bad_words", CELL, SIZED, checked),
    ("AllToAll", "first_bad", CELL, SIZED, checked),
    ("AllToAll", "sum", CELL, SIZED, checked),
    ("AllToAll", "xr", CELL, SIZED, checked),
    ("CeAllToAll", "measured", RANK, False, always),
    ("CeAllToAll", "status", RANK, False, always),
    ("CeAllToAll", "blocks", RANK, False, measured),
    ("CeAllToAll", "t0_ns", RANK, False, measured),
    ("CeAllToAll", "peak_gbps", RANK, False, measured),
    ("CeAllToAll", "half_bytes", RANK, False, measured),
    ("CeAllToAll", "ns_min", RANK, SIZED, measured),
    ("CeAllToAll", "ns_median", RANK, SIZED, measured),
    ("CeAllToAll", "ns_max", RANK, SIZED, measured),
    ("CeAllToAll", "cell_measured", CELL, False, always),
    ("CeAllToAll", "cell_status", CELL, False, always),
    ("CeAllToAll", "bad_sizes", CELL, False, checked),
    ("CeAllToAll", "copy_ns_median", CELL, SIZED, issued),
    ("CeAllToAll", "bad_words", CELL, SIZED, checked),
    ("CeAllToAll", "first_bad", CELL, SIZED, checked),
    ("CeAllToAll", "sum", CELL, SIZED, checked),
    ("CeAllToAll", "xr", CELL, SIZED, checked),
]
TYPES = {"Latency": "LatencyT", "PingPong": "PingPongT", "Atomics": "AtomicsT", "BwCurve": "BwCurveT",
         "Memcpy": "MemcpyT", "AllReduce": "AllReduceT", "AllToAll": "AllToAllT", "CeAllToAll": "CeAllToAllT"}


def random_result(a, struct_type, rng, nrng):
    """A result of `struct_type` with random contents: finite floats, n of 1 to 16, n_sizes of 0 to 24, measured
    entries at one of four densities (any nonzero byte), statuses that often time out, and rank block counts that
    often equal n."""
    t = struct_type()
    for name, _ in struct_type._fields_:
        v = getattr(t, name)
        if isinstance(v, (int, float)):
            setattr(t, name, rng.getrandbits(16) if isinstance(v, int) else rng.uniform(0.0, 1e3))
            continue
        arr = np.ctypeslib.as_array(v).reshape(-1)
        if arr.dtype.kind == "f":
            arr[:] = nrng.uniform(-1e6, 1e6, arr.size)
        elif arr.dtype.kind in "iu":
            info = np.iinfo(arr.dtype)
            arr[:] = nrng.integers(info.min, info.max, arr.size, dtype=arr.dtype, endpoint=True)
    t.n = rng.randint(1, M)
    if hasattr(t, "n_sizes"):
        t.n_sizes = rng.randint(0, a.BWCURVE_MAX_SIZES)
    for name in ("measured", "cell_measured"):
        if hasattr(t, name):
            density = rng.choice((0.0, 0.5, 0.9, 1.0))
            arr = getattr(t, name)
            for k in range(len(arr)):
                arr[k] = rng.randint(1, 255) if rng.random() < density else 0
    for name in ("status", "cell_status"):
        if hasattr(t, name):
            arr = getattr(t, name)
            for k in range(len(arr)):
                arr[k] = rng.choice((a.OK, a.ERR_TIMEOUT, a.ERR_TIMEOUT, a.ERR_INTEGRITY, a.ERR_UNSUPPORTED, 3))
    if hasattr(t, "blocks"):
        for r in range(M):
            t.blocks[r] = rng.choice((t.n, t.n, t.n - 1, 0, rng.getrandbits(32)))
    return t


def expected(t, field, shape, sized, keep):
    a = getattr(t, field)

    def entry(k):
        if sized:
            return list(a[k])[:t.n_sizes]
        return bool(a[k]) if field in ("measured", "cell_measured") else a[k]

    if shape == RANK:
        return [entry(s) if keep(t, s, None) else None for s in range(t.n)]
    return [[entry(s * M + d) if keep(t, s, d) else None for d in range(t.n)] for s in range(t.n)]


@pytest.mark.parametrize("kind", list(TYPES))
def test_from_c_keeps_each_field_where_the_table_says(pkg, kind):
    a = pkg.abi
    assert a.MAX_GPUS == M and a.ERR_TIMEOUT == ERR_TIMEOUT
    cls, struct_type = getattr(pkg, kind), getattr(a, TYPES[kind])
    rules = [r[1:] for r in RULES if r[0] == kind]
    struct_fields = {f for f, _ in struct_type._fields_}
    # every field of the result is in the table, or is the ladder, the raw struct or a scalar copied from it
    ruled = {f for f, *_ in rules}
    rest = [f.name for f in dataclasses.fields(cls) if f.name not in ruled | {"sizes", "raw"}]
    assert ruled <= {f.name for f in dataclasses.fields(cls)} and set(rest) <= struct_fields, kind
    rng, nrng = random.Random(kind), np.random.default_rng(sum(kind.encode()))
    for _ in range(60):
        t = random_result(a, struct_type, rng, nrng)
        m = cls.from_c(t)
        assert m.raw is t
        for f in rest:
            v = getattr(m, f)
            assert v == (bool(getattr(t, f)) if type(v) is bool else getattr(t, f)), f
        if "size" in struct_fields:
            assert m.sizes == list(t.size)[:t.n_sizes]
        for field, shape, sized, keep in rules:
            got = getattr(m, field)
            assert got == expected(t, field, shape, sized, keep), (kind, field, t.n)
            if field in ("measured", "cell_measured"):
                assert all(type(x) is bool for x in (got if shape == RANK else sum(got, []))), field


ENCODERS = [  # (encoder, its fields as (argument, shift, width, bias), its mode argument and count, whether it checks)
    ("memcpy_fault", [("issuer", 40, 8, 1), ("target", 32, 8, 1), ("k", 24, 8, 1), ("word", 0, 24, 0)],
     ("mode", 2), True),
    ("ce_alltoall_fault", [("issuer", 40, 8, 1), ("target", 32, 8, 1), ("k", 24, 8, 1), ("arg", 0, 24, 0)],
     ("mode", 3), True),
    ("alltoall_fault", [("sender", 40, 8, 1), ("receiver", 32, 8, 1), ("k", 24, 8, 1), ("word", 0, 24, 0)],
     None, False),
    ("allreduce_fault", [("rank", 32, 16, 1), ("k", 24, 8, 1), ("word", 0, 24, 0)], ("drop", 2), True),
    ("allreduce_twoshot_fault", [("receiver", 32, 16, 1), ("k", 24, 8, 1), ("word", 0, 24, 0)], ("drop", 2), False),
    ("allreduce_ll_fault", [("sender", 40, 8, 1), ("receiver", 32, 8, 1), ("k", 24, 8, 1), ("arg", 0, 24, 0)],
     ("mode", 3), True),
    ("allreduce_ring_fault", [("phase", 40, 1, 0), ("sender", 32, 8, 1), ("k", 24, 8, 1), ("arg", 0, 24, 0)],
     ("mode", 3), True),
    ("allreduce_push_fault", [("rank", 32, 16, 1), ("k", 24, 8, 1), ("word", 0, 24, 0)], ("mode", 4), True),
    ("allreduce_nvls_fault", [("k", 24, 8, 1), ("word", 0, 24, 0)], ("mode", 2), True),
    ("atomics_fault", [("issuer", 16, 16, 1), ("target", 0, 16, 1)], None, False),
    ("pingpong_fault", [("initiator", 32, 16, 1), ("target", 16, 16, 1), ("trip", 0, 16, 0)], None, False),
]


@pytest.mark.parametrize("name,fields,mode,checks", ENCODERS, ids=[e[0] for e in ENCODERS])
def test_fault_packing_at_each_field_edge(pkg, name, fields, mode, checks):
    encode = getattr(pkg.abi, name)
    zero = {arg: 0 for arg, *_ in fields}

    def packed(args, m=0):
        word = m << 48
        for arg, shift, _, bias in fields:
            word |= (args[arg] + bias) << shift
        return word

    assert encode(**zero) == packed(zero)
    for arg, shift, width, bias in fields:
        top = (1 << width) - 1 - bias  # the largest value whose field fits
        for v in (0, 1, top):
            args = zero | {arg: v}
            got = encode(**args)
            assert got == packed(args) and (got >> shift) & ((1 << width) - 1) == v + bias, (arg, v)
        for v in (-1, top + 1):
            args = zero | {arg: v}
            if checks:
                with pytest.raises(ValueError, match=f"^{name}: "):
                    encode(**args)
            else:  # packed as given, whatever the width
                assert encode(**args) == packed(args), (arg, v)
    if mode is not None:
        arg, count = mode
        for m in range(count):
            assert encode(**zero, **{arg: bool(m) if arg == "drop" else m}) == packed(zero, m)
        if arg == "mode":
            for m in (-1, count):
                with pytest.raises(ValueError, match=f"^{name}: "):
                    encode(**zero, mode=m)
