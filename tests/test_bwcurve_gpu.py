"""cdprobe_bwcurve on the GPU: every run cell's (S, X) at every size equals the oracle's for that prefix, a word
corrupted at rest fails exactly the sizes that cover it, cells whose mapping is down are skipped, the call needs no run
and disturbs none, the times are plausible and bounded, and two processes agree.  Several ranks share one device where
a test needs N > 1."""
import functools
import textwrap

import pytest

import bwcurve_ref as ref
from conftest import ROOT
from harness import run_children

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
LOCAL_DIAG = 0x04
SIMULATE_MIG = 0x200
MODE_SLICED, MODE_FULL = 1, 2
ERR_ARG, ERR_UNSUPPORTED, ERR_STATE, ERR_INTEGRITY = -2, -8, -9, -10
GIB = 1 << 30
HBM_GBPS = 3350.0  # H100 SXM data sheet


def open_same(pkg, n, flags=0, nbytes=1 << 20, mode=MODE_SLICED):
    return pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, mode=mode, flags=SAME | flags, ctas=8,
                               timeout_ms=20000))


@functools.lru_cache(maxsize=None)
def want(oracle, target, first_word, n_words):
    return oracle.src_checksum(SEED, target, first_word, n_words)


def slice_first_word(n, i, j, bpp, full):
    """Word index in j's source buffer where the slice issuer i reads begins (cell_slice in plan.h)."""
    if full:
        return 0
    slot = (n - 1) if i == j else (i if i < j else i - 1)
    return slot * (bpp // 8)


def assert_clean(bw, oracle, i, j, bpp, full=False):
    assert bw.measured[i][j] and bw.status[i][j] == 0 and bw.bad_sizes[i][j] == 0, (i, j, bw.status[i][j])
    first = slice_first_word(bw.n, i, j, bpp, full)
    for k, s in enumerate(bw.sizes):
        assert 0 < bw.ns_min[i][j][k] <= bw.ns_median[i][j][k] <= bw.ns_max[i][j][k], (i, j, s)
        assert (bw.sum[i][j][k], bw.xr[i][j][k]) == want(oracle, j, first, s // 8), (i, j, s)
    assert (bw.t0_ns[i][j], bw.peak_gbps[i][j], bw.half_bytes[i][j]) == ref.summary(bw.sizes, bw.ns_median[i][j])


def assert_all_clean(bw, oracle, bpp, diag, full=False, skip=()):
    assert bw.sizes == ref.ladder(bpp)
    for i in range(bw.n):
        for j in range(bw.n):
            if i == j and not diag:
                assert not bw.measured[i][j] and bw.status[i][j] == 0 and bw.ns_median[i][j] is None
            elif (i, j) not in skip:
                assert_clean(bw, oracle, i, j, bpp, full)


def assert_fits_in_call(bw):
    """Each local rank's timed reps run one after another, so their least times must fit the call's wall clock."""
    for i in range(bw.n):
        busy = sum(bw.reps * t for j in range(bw.n) if bw.ns_min[i][j] for t in bw.ns_min[i][j])
        assert busy / 1e6 <= bw.ms, (i, busy, bw.ms)


@pytest.mark.parametrize("path", [0, 1, 2], ids=["tma", "ldst16", "ldst32"])
@pytest.mark.parametrize("nbytes", [4 << 20, GIB], ids=["4MiB", "1GiB"])
def test_loopback_every_size_clean(pkg, oracle, nbytes, path):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, timeout_ms=20000)) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        bw = p.BwCurve()
        assert (bw.n, bw.row_mask, bw.reps, bw.path, bw.call_seq) == (1, 1, 8, path, 1)
        assert_all_clean(bw, oracle, nbytes, True)
        assert_fits_in_call(bw)
        bw2 = p.BwCurve(reps=3)
        assert (bw2.reps, bw2.call_seq) == (3, 2)
        assert_all_clean(bw2, oracle, nbytes, True)
        if nbytes == GIB:
            k = bw.sizes.index(GIB)
            assert GIB / bw.ns_min[0][0][k] <= 1.1 * HBM_GBPS, bw.ns_min[0][0][k]
            # both beyond the 50 MB L2: twice the bytes take about twice the time
            ratio = bw.ns_median[0][0][k] / bw.ns_median[0][0][bw.sizes.index(GIB // 2)]
            assert 1.6 <= ratio <= 2.4, ratio


@pytest.mark.parametrize("mode", [MODE_SLICED, MODE_FULL], ids=["sliced", "full"])
@pytest.mark.parametrize("flags", [0, LOCAL_DIAG], ids=["", "local-diag"])
@pytest.mark.parametrize("n", [2, 3, 4, 5, 8])
def test_same_device_every_cell_clean(pkg, oracle, n, flags, mode):
    nbytes = 1 << 20
    with open_same(pkg, n, flags, nbytes, mode) as p:
        bpp = pkg.plan(n, nbytes, mode, flags).bytes_per_pair
        bw = p.BwCurve(reps=4)
        assert (bw.n, bw.row_mask, bw.reps, bw.call_seq) == (n, (1 << n) - 1, 4, 1)
        assert_all_clean(bw, oracle, bpp, bool(flags & LOCAL_DIAG), mode == MODE_FULL)
        assert_fits_in_call(bw)
        assert p.BwCurve(reps=2).call_seq == 2


@pytest.mark.parametrize("path", [0, 1, 2], ids=["tma", "ldst16", "ldst32"])
def test_a_corrupt_word_fails_exactly_the_sizes_that_cover_it(pkg, oracle, path):
    n, nbytes = 2, (1 << 20) + 5 * 1024 + 128  # bpp is not a whole number of 16 KiB granules
    with open_same(pkg, n, nbytes=nbytes) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        bpp = pkg.plan(n, nbytes, MODE_SLICED).bytes_per_pair
        sizes = ref.ladder(bpp)
        i, j = 0, 1
        base = slice_first_word(n, i, j, bpp, False) * 8  # the slice i reads, in j's source buffer
        last_partial = bpp // 16384 * 16384 + 1000
        for o in (40, 200000, last_partial):
            assert bpp // 16384 * 16384 <= last_partial < bpp
            p.Corrupt(j, base + o, 1 << 17)
            bw = p.BwCurve(reps=2)
            assert bw.measured[i][j] and bw.status[i][j] == ERR_INTEGRITY, o
            assert bw.bad_sizes[i][j] == sum(1 << k for k, s in enumerate(sizes) if s > o), (o, bw.bad_sizes[i][j])
            assert 0 < bw.ns_min[i][j][-1] <= bw.ns_max[i][j][-1]  # the times are still reported
            assert_all_clean(bw, oracle, bpp, False, skip={(i, j)})
            p.Corrupt(j, base + o, 1 << 17)  # restore
            assert_all_clean(p.BwCurve(reps=2), oracle, bpp, False)


def test_callable_before_the_first_run_and_disturbs_nothing(pkg, oracle):
    n, nbytes = 2, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        assert_all_clean(p.BwCurve(reps=2), oracle, nbytes, False)
        lat = p.Latency()
        r1 = p.Run()
        assert r1.reach == [[1] * n for _ in range(n)] and not r1.aborted
        bw = p.BwCurve(reps=2)
        assert bw.call_seq == 2
        assert_all_clean(bw, oracle, nbytes, False)
        for i, j in ((0, 1), (1, 0)):  # the run's regions are as it left them
            for op in ("read", "write"):
                d = p.Diagnose(op, i, j)
                assert d.bad_words == 0 and d.run_seq == r1.run_seq
        r2 = p.Run()
        assert r2.run_seq == r1.run_seq + 1 and r2.reach == r1.reach and not r2.aborted
        assert (r2.sum_read, r2.xor_read) == (r1.sum_read, r1.xor_read)
        words = r2.bytes_per_pair // 8
        for i, j in ((0, 1), (1, 0)):
            assert (r2.sum_write[i][j], r2.xor_write[i][j]) == oracle.write_checksum(SEED, i, j, r2.run_seq, words)
        assert p.Latency().digest == lat.digest
        pp = p.PingPong(trips=64, reps=2)
        assert all(pp.status[i][j] == 0 and pp.measured[i][j] for i in range(n) for j in range(n) if i != j)
        at = p.Atomics(pkg.abi.ATOMIC_FETCH_ADD, ops=64, reps=2)
        assert all(at.status[i][j] == 0 and at.measured[i][j] for i in range(n) for j in range(n) if i != j)


def test_a_mapping_that_is_down_skips_only_that_cell(pkg, oracle):
    n, nbytes = 4, 1 << 20
    with open_same(pkg, n) as p:
        bpp = pkg.plan(n, nbytes, MODE_SLICED).bytes_per_pair
        p.UnmapPeer(0, 1)
        bw = p.BwCurve(reps=2)
        assert not bw.measured[0][1] and bw.status[0][1] == ERR_STATE and bw.ns_median[0][1] is None
        assert bw.raw.sum[1][0] == 0
        assert_clean(bw, oracle, 1, 0, bpp)  # its reverse cell still runs
        assert_all_clean(bw, oracle, bpp, False, skip={(0, 1)})
        p.RemapPeer(0, 1)
        assert_all_clean(p.BwCurve(reps=2), oracle, bpp, False)


def test_simulated_mig_runs_no_pair(pkg):
    n = 2
    with open_same(pkg, n, flags=SIMULATE_MIG) as p:
        bw = p.BwCurve(reps=2)
        for i in range(n):
            for j in range(n):
                assert not bw.measured[i][j] and bw.ns_median[i][j] is None
                assert bw.status[i][j] == (ERR_UNSUPPORTED if i != j else 0)


def test_argument_errors_fill_the_output(pkg, oracle):
    a = pkg.abi
    with open_same(pkg, 2) as p:
        rc, t = p.bwcurve_raw(a.BWCURVE_MAX_REPS + 1)
        assert rc == ERR_ARG and (t.abi, t.n, t.reps, t.call_seq, t.row_mask, t.n_sizes) == (2, 2, 65, 0, 0, 0)
        assert sum(t.measured) == 0
        with pytest.raises(pkg.ProbeError):
            p.BwCurve(1 << 31)
        bw = p.BwCurve(reps=a.BWCURVE_MAX_REPS)  # the handle stays usable
        assert bw.call_seq == 1
        assert_all_clean(bw, oracle, 1 << 20, False)


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    cfg = m.Config(ordinals=[0], bytes=1 << 20, world_size=world, rank=rank, session=session, flags=0x40, ctas=8,
                   timeout_ms=30000)

    def dump(bw):
        return {"row_mask": bw.row_mask, "measured": bw.measured, "status": bw.status, "sum": bw.sum, "xr": bw.xr,
                "ns_min": bw.ns_min, "sizes": bw.sizes, "call_seq": bw.call_seq, "reps": bw.reps}

    with m.Open(cfg) as p:
        out = {"calls": [dump(p.BwCurve(reps=2)), dump(p.BwCurve(reps=3))]}
        rc, t = p.bwcurve_raw(2 + rank)  # the processes disagree
        out["mismatch"] = {"rc": rc, "call_seq": t.call_seq, "measured": sum(t.measured)}
        out["after"] = dump(p.BwCurve(reps=2))
        r = p.Run(gather=True)
        out["run"] = {"reach": r.reach, "aborted": r.aborted}
        # a handle made sticky: rank 1 never launches its kernel, rank 0's watchdog fires, both handles stay unusable
        p.SetOption(m.abi.OPT_TIMEOUT_MS, 300)
        if rank == 1:
            p.SetOption(m.abi.OPT_DEBUG_SKIP_RANK, 1)
        p.Run(allow_timeout=True)
        out["sticky"] = p.bwcurve_raw(2)[0]
    print("RESULT " + json.dumps(out))
    """
) % ROOT


def test_two_processes_agree_and_fill_their_own_rows(pkg, oracle):
    """Both processes drive GPU 0, so their contexts are time-sliced and the times only need to be positive."""
    world = 2
    outs = run_children(CHILD, world)
    bpp = 1 << 20
    for rank, o in enumerate(outs):
        other = 1 - rank
        assert [c["call_seq"] for c in o["calls"]] + [o["after"]["call_seq"]] == [1, 2, 3]
        assert o["mismatch"] == {"rc": ERR_ARG, "call_seq": 0, "measured": 0}
        for c in o["calls"] + [o["after"]]:
            assert c["row_mask"] == 1 << rank and c["sizes"] == ref.ladder(bpp)
            assert c["measured"][rank] == [j != rank for j in range(world)]
            assert c["measured"][other] == [False] * world and c["sum"][other] == [None] * world
            assert c["status"][rank][other] == 0 and all(t > 0 for t in c["ns_min"][rank][other])
            first = slice_first_word(world, rank, other, bpp, False)
            assert [[s, x] for s, x in zip(c["sum"][rank][other], c["xr"][rank][other])] == \
                [list(want(oracle, other, first, s // 8)) for s in c["sizes"]]
        assert o["run"]["reach"] == [[1] * world for _ in range(world)] and not o["run"]["aborted"]
        assert o["sticky"] == ERR_STATE
