"""cdprobe_pingpong on the GPU: every exchanged cell's digest equals the restatement in tests/pingpong_ref.py, so a
round trip that returned the wrong words cannot pass; the times are plausible; pairs whose mapping is down are not
exchanged; the skip-ahead fault fails exactly its cell; the call needs no run and disturbs none.  Several ranks share
one device where a test needs N > 1."""
import textwrap

import pytest

import pingpong_ref as ref
from conftest import ROOT
from harness import run_children

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
SIMULATE_MIG = 0x200
ERR_ARG, ERR_UNSUPPORTED, ERR_STATE, ERR_INTEGRITY = -2, -8, -9, -10


def open_same(pkg, n, flags=0, nbytes=1 << 20):
    return pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME | flags, ctas=8, timeout_ms=20000))


def want(pkg, pp, i, j, fault_trip=None):
    pl = pkg.plan(pp.n, 1 << 20, 1)
    return ref.cell_digest(pp.call_seq, pl.partner, pl.rounds, i, j, pp.trips, pp.reps, fault_trip)


def assert_clean(pkg, pp, i, j):
    assert pp.measured[i][j] and pp.status[i][j] == 0, (i, j, pp.status[i][j])
    assert 0 < pp.ns_min[i][j] <= pp.ns_median[i][j] <= pp.ns_max[i][j], (i, j)
    assert 100 <= pp.ns_median[i][j] <= 100000, (i, j, pp.ns_median[i][j])  # plausibility, not a performance claim
    assert pp.digest[i][j] == want(pkg, pp, i, j), (i, j)


def assert_all_clean(pkg, pp, skip=()):
    for i in range(pp.n):
        for j in range(pp.n):
            if i == j:
                assert not pp.measured[i][j] and pp.status[i][j] == 0 and pp.digest[i][j] is None
            elif (i, j) not in skip:
                assert_clean(pkg, pp, i, j)


@pytest.mark.parametrize("fenced", [False, True], ids=["plain", "fenced"])
@pytest.mark.parametrize("n", [2, 3, 4, 5, 8])
def test_every_cell_clean(pkg, n, fenced):
    """Odd n: every rank idles in one round, and its partners of the rounds either side reach it late or early."""
    with open_same(pkg, n) as p:
        pp = p.PingPong(fenced=fenced)
        assert (pp.n, pp.row_mask, pp.trips, pp.reps, pp.fenced, pp.call_seq) == (n, (1 << n) - 1, 256, 8, fenced, 1)
        assert_all_clean(pkg, pp)
        assert pp.ms > 0
        pp2 = p.PingPong(trips=32, reps=3, fenced=fenced)
        assert (pp2.trips, pp2.reps, pp2.call_seq) == (32, 3, 2)
        assert_all_clean(pkg, pp2)


def test_single_rank_measures_nothing(pkg):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 20)) as p:
        pp = p.PingPong()
        assert (pp.n, pp.row_mask, pp.call_seq) == (1, 1, 1)
        assert pp.measured == [[False]] and pp.status == [[0]] and pp.ns_median == [[None]]
        assert p.Run().verdict


def test_callable_before_the_first_run_and_disturbs_nothing(pkg, oracle):
    n, nbytes = 2, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        lat = p.Latency()
        assert_all_clean(pkg, p.PingPong())

        def check_run(seq):
            """A run that passes with the oracle's checksums, and whose run_seq counts runs only."""
            r = p.Run()
            assert r.reach == [[1] * n for _ in range(n)] and not r.aborted
            assert seq is None or r.run_seq == seq
            words = r.bytes_per_pair // 8
            for i in range(n):
                for j in range(n):
                    if i != j:
                        assert (r.sum_read[i][j], r.xor_read[i][j]) == oracle.expected_read(SEED, n, nbytes, 1, i, j)
                        assert (r.sum_write[i][j], r.xor_write[i][j]) == oracle.write_checksum(SEED, i, j, r.run_seq,
                                                                                               words)
            return r.run_seq

        first = check_run(None)
        assert_all_clean(pkg, p.PingPong(fenced=True))
        for i, j in ((0, 1), (1, 0)):  # the run's regions are as it left them
            for op in ("read", "write"):
                d = p.Diagnose(op, i, j)
                assert d.bad_words == 0 and d.run_seq == first
        assert p.Latency().digest == lat.digest
        check_run(first + 1)  # directly after a pingpong: Ctrl and its flags are untouched
        assert_all_clean(pkg, p.PingPong(trips=16, reps=2))
        check_run(first + 2)


def test_a_mapping_that_is_down_skips_the_pair(pkg):
    n = 4
    with open_same(pkg, n) as p:
        p.UnmapPeer(0, 1)
        r = p.Run()
        assert r.status[0][1] == ERR_STATE
        pp = p.PingPong(trips=64, reps=2)
        for i, j in ((0, 1), (1, 0)):
            assert not pp.measured[i][j] and pp.status[i][j] == r.status[0][1]
            assert pp.ns_median[i][j] is None and pp.digest[i][j] is None and pp.raw.digest[i * 16 + j] == 0
        assert_all_clean(pkg, pp, skip={(0, 1), (1, 0)})
        p.RemapPeer(0, 1)
        assert_all_clean(pkg, p.PingPong(trips=64, reps=2))


def test_simulated_mig_measures_nothing(pkg):
    n = 2
    with open_same(pkg, n, flags=SIMULATE_MIG) as p:
        pp = p.PingPong()
        for i in range(n):
            for j in range(n):
                assert not pp.measured[i][j] and pp.ns_median[i][j] is None
                if i != j:
                    assert pp.status[i][j] == ERR_UNSUPPORTED


def test_skip_ahead_echo_fails_exactly_its_cell(pkg):
    n, trips, reps = 4, 16, 2
    with open_same(pkg, n) as p:
        for i, j, trip in ((1, 3, 5), (3, 0, 0), (2, 1, trips - 2)):
            p.SetOption(pkg.abi.OPT_PINGPONG_FAULT, pkg.abi.pingpong_fault(i, j, trip))
            pp = p.PingPong(trips=trips, reps=reps)
            assert pp.measured[i][j] and pp.status[i][j] == ERR_INTEGRITY, (i, j, pp.status[i][j])
            assert pp.digest[i][j] == want(pkg, pp, i, j, fault_trip=trip) != want(pkg, pp, i, j)
            assert 0 < pp.ns_min[i][j] <= pp.ns_median[i][j] <= pp.ns_max[i][j]
            assert_all_clean(pkg, pp, skip={(i, j)})
            p.SetOption(pkg.abi.OPT_PINGPONG_FAULT, 0)
            assert_all_clean(pkg, p.PingPong(trips=trips, reps=reps))
        # the echo must stay inside its rep, and the cell must exist
        for value in (pkg.abi.pingpong_fault(1, 3, trips - 1), pkg.abi.pingpong_fault(1, 3, trips),
                      pkg.abi.pingpong_fault(2, 2, 0), pkg.abi.pingpong_fault(0, n, 0), pkg.abi.pingpong_fault(n, 0, 0)):
            p.SetOption(pkg.abi.OPT_PINGPONG_FAULT, value)
            rc, t = p.pingpong_raw(trips, reps, 0)
            assert rc == ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0, hex(value)
        # with one timed rep, the initiator must catch up before the leg ends: trips - 2 is refused too
        p.SetOption(pkg.abi.OPT_PINGPONG_FAULT, pkg.abi.pingpong_fault(1, 3, trips - 2))
        assert p.pingpong_raw(trips, 1, 0)[0] == ERR_ARG
        p.SetOption(pkg.abi.OPT_PINGPONG_FAULT, pkg.abi.pingpong_fault(1, 3, trips - 3))  # an earlier trip is accepted
        pp = p.PingPong(trips=trips, reps=1, fenced=True)
        assert pp.status[1][3] == ERR_INTEGRITY and pp.digest[1][3] == want(pkg, pp, 1, 3, fault_trip=trips - 3)
        assert_all_clean(pkg, pp, skip={(1, 3)})
        p.SetOption(pkg.abi.OPT_PINGPONG_FAULT, 0)
        assert_all_clean(pkg, p.PingPong(trips=trips, reps=reps))


def test_argument_errors_fill_the_output(pkg):
    a = pkg.abi
    with open_same(pkg, 2) as p:
        first = p.PingPong(trips=1, reps=1)  # the smallest exchange
        assert_all_clean(pkg, first)
        for trips, reps, fenced in ((a.PINGPONG_MAX_TRIPS + 1, 0, 0), (0, a.PINGPONG_MAX_REPS + 1, 0), (0, 0, 2),
                                    (1 << 31, 1 << 31, 1)):
            rc, t = p.pingpong_raw(trips, reps, fenced)
            assert rc == a.ERR_ARG, (trips, reps, fenced)
            assert (t.abi, t.n, t.call_seq, t.row_mask) == (2, 2, 0, 0) and sum(t.measured) == 0
            assert (t.trips, t.reps, t.fenced) == (trips or a.PINGPONG_DEFAULT_TRIPS, reps or a.PINGPONG_DEFAULT_REPS,
                                                   fenced)
        with pytest.raises(pkg.ProbeError):
            p.PingPong(trips=a.PINGPONG_MAX_TRIPS + 1)
        big = p.PingPong(trips=a.PINGPONG_MAX_TRIPS, reps=1)  # the largest trip field
        assert big.call_seq == first.call_seq + 1
        assert_all_clean(pkg, big)
        last = p.PingPong(trips=8, reps=a.PINGPONG_MAX_REPS, fenced=True)  # the largest rep field
        assert last.call_seq == 3
        assert_all_clean(pkg, last)


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    cfg = m.Config(ordinals=[0], bytes=1 << 20, world_size=world, rank=rank, session=session, flags=0x40, ctas=8,
                   timeout_ms=30000)

    def dump(pp):
        return {"row_mask": pp.row_mask, "measured": pp.measured, "status": pp.status, "digest": pp.digest,
                "ns_min": pp.ns_min, "ns_median": pp.ns_median, "trips": pp.trips, "reps": pp.reps,
                "call_seq": pp.call_seq}

    with m.Open(cfg) as p:
        out = {"calls": [dump(p.PingPong(trips=4, reps=2))]}
        r = p.Run(gather=True)
        out["run"] = {"reach": r.reach, "aborted": r.aborted, "run_seq": r.run_seq}
        out["calls"].append(dump(p.PingPong(trips=4, reps=2)))
        rc, t = p.pingpong_raw(4 if rank == 0 else 8, 2, 0)
        out["mismatch"] = {"rc": rc, "call_seq": t.call_seq, "measured": sum(t.measured)}
        out["calls"].append(dump(p.PingPong(trips=4, reps=2)))
    print("RESULT " + json.dumps(out))
    """
) % ROOT


def test_two_processes_fill_their_own_rows(pkg):
    """Both processes drive GPU 0, so their contexts are time-sliced and every round trip may wait for a context
    switch: the counts stay small and the times only need to be positive."""
    world = 2
    outs = run_children(CHILD, world)
    pl = pkg.plan(world, 1 << 20, 1)
    for rank, o in enumerate(outs):
        other = 1 - rank
        assert [c["call_seq"] for c in o["calls"]] == [1, 2, 3]
        for c in o["calls"]:
            assert c["row_mask"] == 1 << rank
            assert c["measured"][rank] == [j != rank for j in range(world)]
            assert c["measured"][other] == [False] * world and c["digest"][other] == [None] * world
            assert c["status"][rank][other] == 0 and 0 < c["ns_min"][rank][other] <= c["ns_median"][rank][other]
            assert c["digest"][rank][other] == ref.cell_digest(c["call_seq"], pl.partner, pl.rounds, rank, other,
                                                                c["trips"], c["reps"])
        assert o["run"]["reach"] == [[1] * world for _ in range(world)] and not o["run"]["aborted"]
        assert o["mismatch"] == {"rc": ERR_ARG, "call_seq": 0, "measured": 0}
