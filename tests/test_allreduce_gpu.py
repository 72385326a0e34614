"""cdprobe_allreduce on the GPU: every row's output at every size has the (S, X) of the pattern's sum and passes the
word check, a word corrupted at rest fails exactly the sizes that cover it in every row, an armed fault fails exactly
one row and size, a mapping that is down stops every rank without waiting, two processes agree, the call needs no run
and disturbs none, and the times are ordered and bounded.  Several ranks share one device where a test needs N > 1,
with CTA counts that let their grids be resident together (every rank waits for every other at each rep)."""
import json
import subprocess
import sys
import textwrap
import uuid

import pytest

import allreduce_ref as ref
import atomics_ref
import pingpong_ref
from conftest import ROOT

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
SIMULATE_MIG = 0x200
MODE_REACH, MODE_SLICED, MODE_FULL = 0, 1, 2
ERR_ARG, ERR_UNSUPPORTED, ERR_STATE, ERR_INTEGRITY = -2, -8, -9, -10
U64_MAX = (1 << 64) - 1
GIB = 1 << 30
REF_MAX = 64 << 20  # sizes up to this get their (S, X) from the numpy reference; larger ones (N = 1) from the oracle


def open_same(pkg, n, flags=0, nbytes=1 << 20, mode=MODE_SLICED):
    return pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, mode=mode, flags=SAME | flags,
                               ctas=8 if n <= 8 else 4, timeout_ms=20000))


def want(oracle, n, sizes):
    small = tuple(s for s in sizes if s <= REF_MAX)
    got = dict(zip(small, ref.expected(SEED, n, small))) if small else {}
    for s in sizes:
        if s not in got:
            assert n == 1, "only the single-rank output is checked against the oracle beyond REF_MAX"
            got[s] = oracle.src_checksum(SEED, 0, 0, s // 8)
    return [got[s] for s in sizes]


def assert_row_clean(ar, r, expect):
    assert ar.measured[r] and ar.status[r] == 0 and ar.bad_sizes[r] == 0, (r, ar.status[r], ar.bad_sizes[r])
    for k, s in enumerate(ar.sizes):
        assert 0 < ar.ns_min[r][k] <= ar.ns_median[r][k] <= ar.ns_max[r][k], (r, s)
        assert (ar.sum[r][k], ar.xr[r][k]) == expect[k], (r, s)
        assert ar.bad_words[r][k] == 0 and ar.first_bad[r][k] == U64_MAX, (r, s)
    assert (ar.t0_ns[r], ar.peak_gbps[r], ar.half_bytes[r]) == ref.summary(ar.sizes, ar.ns_median[r])


def assert_fits_in_call(ar):
    """A rank's timed reps run one after another inside the call, so their least times must fit its wall clock."""
    for r in range(ar.n):
        if ar.ns_min[r]:
            busy = sum(ar.reps * t for t in ar.ns_min[r])
            assert busy / 1e6 <= ar.ms, (r, busy, ar.ms)
            assert max(ar.ns_median[r]) / 1e6 <= ar.ms


def assert_all_clean(ar, oracle, bpp, rows=None):
    assert ar.sizes == ref.ladder(bpp)
    expect = want(oracle, ar.n, ar.sizes)
    for r in (range(ar.n) if rows is None else rows):
        assert_row_clean(ar, r, expect)
    assert_fits_in_call(ar)


@pytest.mark.parametrize("path", [0, 1, 2], ids=["tma", "ldst16", "ldst32"])
@pytest.mark.parametrize("nbytes", [4 << 20, GIB], ids=["4MiB", "1GiB"])
def test_single_rank_every_size_clean(pkg, oracle, nbytes, path):
    """At N = 1 the output is a copy of the rank's own prefix."""
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, timeout_ms=20000)) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        ar = p.AllReduce()
        assert (ar.n, ar.row_mask, ar.reps, ar.path, ar.call_seq) == (1, 1, 8, path, 1)
        assert_all_clean(ar, oracle, nbytes)
        ar2 = p.AllReduce(reps=3)
        assert (ar2.reps, ar2.call_seq) == (3, 2)
        assert_all_clean(ar2, oracle, nbytes)


@pytest.mark.parametrize("mode", [MODE_SLICED, MODE_FULL, MODE_REACH], ids=["sliced", "full", "reach"])
@pytest.mark.parametrize("n", [2, 3, 4, 5, 8, 16])
def test_same_device_every_row_clean(pkg, oracle, n, mode):
    nbytes = 1 << 20
    with open_same(pkg, n, nbytes=nbytes, mode=mode) as p:
        bpp = pkg.plan(n, nbytes, mode).bytes_per_pair
        ar = p.AllReduce(reps=3)
        assert (ar.n, ar.row_mask, ar.reps, ar.call_seq) == (n, (1 << n) - 1, 3, 1)
        assert_all_clean(ar, oracle, bpp)
        # every rank holds the same output
        assert len({tuple(ar.sum[r]) for r in range(n)}) == 1
        assert p.AllReduce(reps=2).call_seq == 2


@pytest.mark.parametrize("path", [0, 1, 2], ids=["tma", "ldst16", "ldst32"])
def test_a_corrupt_word_fails_exactly_the_sizes_that_cover_it_in_every_row(pkg, oracle, path):
    n, nbytes = 3, (2 << 20) + 5 * 1024 + 256  # bytes_per_pair is not a whole number of 16 KiB granules
    with open_same(pkg, n, nbytes=nbytes) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        bpp = pkg.plan(n, nbytes, MODE_SLICED).bytes_per_pair
        sizes = ref.ladder(bpp)
        assert bpp % 16384 != 0
        last_partial = bpp // 16384 * 16384 + 1000
        x, mask = 2, 1 << 17
        for o in (40, 200000, last_partial):
            w = o // 8
            p.Corrupt(x, w * 8, mask)
            ar = p.AllReduce(reps=2)
            bits = sum(1 << k for k, s in enumerate(sizes) if s > 8 * w)
            expect = ref.expected_corrupted(SEED, n, tuple(sizes), x, w, mask)
            for r in range(n):
                assert ar.measured[r] and ar.status[r] == ERR_INTEGRITY and ar.bad_sizes[r] == bits, (o, r)
                for k, s in enumerate(sizes):
                    covered = s > 8 * w
                    assert ar.bad_words[r][k] == (1 if covered else 0), (o, r, s)
                    assert ar.first_bad[r][k] == (8 * w if covered else U64_MAX), (o, r, s)
                    assert (ar.sum[r][k], ar.xr[r][k]) == expect[k], (o, r, s)
                    assert 0 < ar.ns_min[r][k] <= ar.ns_max[r][k]  # the times are still reported
            p.Corrupt(x, w * 8, mask)  # restore
            assert_all_clean(p.AllReduce(reps=2), oracle, bpp)


def test_an_armed_fault_fails_exactly_one_row_and_size(pkg, oracle):
    n, nbytes = 3, 1 << 20
    a = pkg.abi
    with open_same(pkg, n, nbytes=nbytes) as p:
        bpp = pkg.plan(n, nbytes, MODE_SLICED).bytes_per_pair
        sizes = ref.ladder(bpp)
        expect = want(oracle, n, sizes)
        rank, k, word = 1, 3, sizes[3] // 8 - 5
        p.SetOption(a.OPT_ALLREDUCE_FAULT, a.allreduce_fault(rank, k, word))
        for reps in (2, 3, 1):
            ar = p.AllReduce(reps=reps)
            for r in range(n):
                if r != rank:
                    assert_row_clean(ar, r, expect)
                    continue
                assert ar.status[r] == ERR_INTEGRITY and ar.bad_sizes[r] == 1 << k, (reps, ar.bad_sizes[r])
                for q in range(len(sizes)):
                    found = reps == 1 and q == k  # a later clean rep overwrites the faulted output
                    assert ar.bad_words[r][q] == (1 if found else 0), (reps, q)
                    assert ar.first_bad[r][q] == (8 * word if found else U64_MAX), (reps, q)
                    if q != k or reps > 1:
                        assert (ar.sum[r][q], ar.xr[r][q]) == expect[q], (reps, q)
        # arming that names no rank, size or word of the call is refused, and refusing changes nothing
        seq = ar.call_seq
        for bad in (a.allreduce_fault(n, 0, 0), a.allreduce_fault(0, len(sizes), 0),
                    a.allreduce_fault(0, 0, sizes[0] // 8), (1 << 24) | 5, (1 << 32) | 5):
            p.SetOption(a.OPT_ALLREDUCE_FAULT, bad)
            rc, t = p.allreduce_raw(2)
            assert rc == ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0, hex(bad)
        p.SetOption(a.OPT_ALLREDUCE_FAULT, 0)
        ar = p.AllReduce(reps=2)
        assert ar.call_seq == seq + 1
        assert_all_clean(ar, oracle, bpp)


def test_a_mapping_that_is_down_stops_every_rank(pkg, oracle):
    n, nbytes = 4, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        bpp = pkg.plan(n, nbytes, MODE_SLICED).bytes_per_pair
        p.UnmapPeer(2, 1)
        ar = p.AllReduce(reps=2)
        assert ar.call_seq == 1 and ar.ms < 5000  # returned without waiting for a watchdog
        for r in range(n):
            assert not ar.measured[r] and ar.status[r] == ERR_STATE and ar.ns_median[r] is None
        assert sum(ar.raw.sum[r][0] for r in range(n)) == 0
        p.RemapPeer(2, 1)
        assert_all_clean(p.AllReduce(reps=2), oracle, bpp)


def test_simulated_mig_runs_no_rank(pkg):
    n = 2
    with open_same(pkg, n, flags=SIMULATE_MIG) as p:
        ar = p.AllReduce(reps=2)
        assert ar.ms < 5000
        for r in range(n):
            assert not ar.measured[r] and ar.ns_median[r] is None and ar.status[r] == ERR_UNSUPPORTED


def test_argument_errors_fill_the_output(pkg, oracle):
    a = pkg.abi
    with open_same(pkg, 2) as p:
        rc, t = p.allreduce_raw(a.ALLREDUCE_MAX_REPS + 1)
        assert rc == ERR_ARG and (t.abi, t.n, t.reps, t.call_seq, t.row_mask, t.n_sizes) == (2, 2, 65, 0, 0, 0)
        assert sum(t.measured) == 0
        with pytest.raises(pkg.ProbeError):
            p.AllReduce(1 << 31)
        ar = p.AllReduce(reps=a.ALLREDUCE_MAX_REPS)  # the handle stays usable
        assert ar.call_seq == 1
        assert_all_clean(ar, oracle, 1 << 20)


def test_callable_before_the_first_run_and_disturbs_nothing(pkg, oracle):
    n, nbytes = 2, 1 << 20
    a = pkg.abi
    with open_same(pkg, n, nbytes=nbytes) as p:
        assert_all_clean(p.AllReduce(reps=2), oracle, nbytes)
        r1 = p.Run()
        assert r1.reach == [[1] * n for _ in range(n)] and not r1.aborted
        diags = [(op, i, j, p.Diagnose(op, i, j)) for i, j in ((0, 1), (1, 0)) for op in ("read", "write")]
        lat = p.Latency()
        pp = p.PingPong(trips=64, reps=2)
        at = p.Atomics(a.ATOMIC_FETCH_ADD, ops=64, reps=2)
        bw = p.BwCurve(reps=2)
        ar = p.AllReduce(reps=2)
        assert ar.call_seq == 2
        assert_all_clean(ar, oracle, nbytes)
        # the last run's regions and every other measurement are as they were
        for op, i, j, d in diags:
            d2 = p.Diagnose(op, i, j)
            assert (d2.bad_words, d2.run_seq, d2.region_offset) == (d.bad_words, d.run_seq, d.region_offset) == \
                (0, r1.run_seq, d.region_offset)
        assert p.Latency().digest == lat.digest
        bw2 = p.BwCurve(reps=2)
        assert bw2.call_seq == 2 and (bw2.sum, bw2.xr, bw2.status) == (bw.sum, bw.xr, bw.status)
        pl = pkg.plan(n, nbytes, MODE_SLICED)
        pp2 = p.PingPong(trips=64, reps=2)
        at2 = p.Atomics(a.ATOMIC_FETCH_ADD, ops=64, reps=2)
        assert (pp2.call_seq, at2.call_seq) == (pp.call_seq + 1, at.call_seq + 1)
        for i in range(n):
            for j in range(n):
                if i == j:
                    continue
                assert pp2.status[i][j] == 0 and at2.status[i][j] == 0
                assert pp2.digest[i][j] == pingpong_ref.cell_digest(pp2.call_seq, pl.partner, pl.rounds, i, j, 64, 2)
                assert at2.digest[i][j] == atomics_ref.cell_digest(at2.call_seq, a.ATOMIC_FETCH_ADD, 64, 2)
        r2 = p.Run()
        assert r2.run_seq == r1.run_seq + 1 and r2.reach == r1.reach and not r2.aborted
        assert (r2.sum_read, r2.xor_read) == (r1.sum_read, r1.xor_read)
        words = r2.bytes_per_pair // 8
        for i, j in ((0, 1), (1, 0)):
            assert (r2.sum_write[i][j], r2.xor_write[i][j]) == oracle.write_checksum(SEED, i, j, r2.run_seq, words)


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world, n_local, what = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), sys.argv[5]
    flags = 0x40 | (0x10 if n_local > 1 else 0) | (0x200 if what == "mig" and rank == 1 else 0)
    cfg = m.Config(ordinals=[0] * n_local, bytes=1 << 20, world_size=world, rank=rank, session=session, flags=flags,
                   ctas=8, timeout_ms=30000)

    def dump(ar):
        return {"row_mask": ar.row_mask, "measured": ar.measured, "status": ar.status, "sum": ar.sum, "xr": ar.xr,
                "bad_words": ar.bad_words, "ns_min": ar.ns_min, "sizes": ar.sizes, "call_seq": ar.call_seq,
                "reps": ar.reps, "ms": ar.ms}

    with m.Open(cfg) as p:
        if what == "mig":
            print("RESULT " + json.dumps({"calls": [dump(p.AllReduce(reps=2))]}))
            sys.exit(0)
        out = {"calls": [dump(p.AllReduce(reps=2)), dump(p.AllReduce(reps=3))]}
        rc, t = p.allreduce_raw(2 + rank)  # the processes disagree
        out["mismatch"] = {"rc": rc, "call_seq": t.call_seq, "measured": sum(t.measured)}
        out["after"] = dump(p.AllReduce(reps=2))
        r = p.Run(gather=True)
        out["run"] = {"reach": r.reach, "aborted": r.aborted}
    print("RESULT " + json.dumps(out))
    """
) % ROOT


def run_processes(world, n_local, what):
    session = f"ar-{uuid.uuid4().hex[:12]}"
    procs = [subprocess.Popen([sys.executable, "-c", CHILD, session, str(r), str(world), str(n_local), what],
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(world)]
    outs = []
    for pr in procs:
        so, se = pr.communicate(timeout=600)
        assert pr.returncode == 0, se[-2000:]
        outs.append(json.loads([l for l in so.splitlines() if l.startswith("RESULT ")][-1][7:]))
    return outs


@pytest.mark.parametrize("n_local", [1, 2], ids=["2x1", "2x2"])
def test_two_processes_agree_and_fill_their_own_rows(pkg, n_local):
    """Both processes drive GPU 0, so their contexts are time-sliced and the times only need to be positive."""
    world = 2
    n = world * n_local
    outs = run_processes(world, n_local, "full")
    sizes = ref.ladder(pkg.plan(n, 1 << 20, MODE_SLICED).bytes_per_pair)
    expect = [list(sx) for sx in ref.expected(SEED, n, tuple(sizes))]
    masks = [o["calls"][0]["row_mask"] for o in outs]
    assert masks[0] & masks[1] == 0 and masks[0] | masks[1] == (1 << n) - 1
    for rank, o in enumerate(outs):
        mine = set(range(rank * n_local, (rank + 1) * n_local))
        assert [c["call_seq"] for c in o["calls"]] + [o["after"]["call_seq"]] == [1, 2, 3]
        assert o["mismatch"] == {"rc": ERR_ARG, "call_seq": 0, "measured": 0}
        for c in o["calls"] + [o["after"]]:
            assert c["row_mask"] == sum(1 << r for r in mine) and c["sizes"] == sizes
            for r in range(n):
                assert c["measured"][r] == (r in mine), r
                if r in mine:
                    assert c["status"][r] == 0 and all(t > 0 for t in c["ns_min"][r])
                    assert [[s, x] for s, x in zip(c["sum"][r], c["xr"][r])] == expect, r
                    assert c["bad_words"][r] == [0] * len(sizes)
                else:
                    assert c["sum"][r] is None
        assert o["run"]["reach"] == [[1] * n for _ in range(n)] and not o["run"]["aborted"]


def test_one_process_with_no_peer_mappings_stops_both():
    """A peer mapping cannot be dropped in one process of a multi-process domain (cdprobe_unmap_peer refuses), so the
    process whose mappings are down is one whose ranks are (simulated) MIG instances: neither process runs, both
    report the status of the domain's first down cell, and neither waits for a watchdog."""
    outs = run_processes(2, 2, "mig")
    for rank, o in enumerate(outs):
        c = o["calls"][0]
        assert c["call_seq"] == 1 and c["ms"] < 5000
        for r in range(4):
            assert not c["measured"][r]
            assert c["status"][r] == (ERR_UNSUPPORTED if r // 2 == rank else 0), (rank, r)
