"""cdprobe_atomics on the GPU: every run cell's digest equals the restatement in tests/atomics_ref.py, so atomics that
lost, duplicated or misplaced an update cannot pass; the times are plausible; cells whose mapping is down are not run;
the armed fault fails exactly its cell; the call is one-sided, needs no run and disturbs none.  Several ranks share
one device where a test needs N > 1."""
import textwrap

import pytest

import atomics_ref as ref
from conftest import ROOT
from harness import run_children

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
LOCAL_DIAG = 0x04
SIMULATE_MIG = 0x200
ERR_ARG, ERR_UNSUPPORTED, ERR_STATE, ERR_INTEGRITY = -2, -8, -9, -10
KINDS = [ref.FETCH_ADD, ref.CAS, ref.CONTENDED]
KIND_IDS = ["fetch_add", "cas", "contended"]


def open_same(pkg, n, flags=0, nbytes=1 << 20):
    return pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME | flags, ctas=8, timeout_ms=20000))


def has_diag(n, flags):
    return n == 1 or bool(flags & LOCAL_DIAG)


def assert_clean(at, i, j):
    assert at.measured[i][j] and at.status[i][j] == 0, (i, j, at.status[i][j])
    assert at.native[i][j] == 1, (i, j)
    assert 0 < at.ns_min[i][j] <= at.ns_median[i][j] <= at.ns_max[i][j], (i, j)
    assert 0.05 <= at.ns_median[i][j] <= 100000, (i, j, at.ns_median[i][j])  # plausibility, not a performance claim
    assert at.digest[i][j] == ref.cell_digest(at.call_seq, at.kind, at.ops, at.reps), (i, j)


def assert_all_clean(at, diag, skip=()):
    for i in range(at.n):
        for j in range(at.n):
            if i == j and not diag:
                assert not at.measured[i][j] and at.status[i][j] == 0 and at.digest[i][j] is None
            elif (i, j) not in skip:
                assert_clean(at, i, j)


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("n,flags", [(1, 0), (2, 0), (3, 0), (4, 0), (5, 0), (8, 0), (4, LOCAL_DIAG)],
                         ids=["n1", "n2", "n3", "n4", "n5", "n8", "n4-local-diag"])
def test_every_cell_clean(pkg, n, flags, kind):
    with open_same(pkg, n, flags) as p:
        at = p.Atomics(kind)
        assert (at.n, at.row_mask, at.kind, at.ops, at.reps, at.call_seq) == (n, (1 << n) - 1, kind, 1024, 8, 1)
        assert at.lanes == (32 if kind == ref.CONTENDED else 1)
        assert_all_clean(at, has_diag(n, flags))
        assert at.ms > 0
        at2 = p.Atomics(kind, ops=100, reps=3)
        assert (at2.ops, at2.reps, at2.call_seq) == (100, 3, 2)
        assert_all_clean(at2, has_diag(n, flags))


def test_callable_before_the_first_run_and_disturbs_nothing(pkg, oracle):
    n, nbytes = 2, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        for kind in KINDS:
            assert_all_clean(p.Atomics(kind, ops=256, reps=2), False)
        lat = p.Latency()

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
        at = p.Atomics(ref.CONTENDED)
        assert at.call_seq == 4
        assert_all_clean(at, False)
        for i, j in ((0, 1), (1, 0)):  # the run's regions are as it left them
            for op in ("read", "write"):
                d = p.Diagnose(op, i, j)
                assert d.bad_words == 0 and d.run_seq == first
        assert p.Latency().digest == lat.digest
        pp = p.PingPong(trips=64, reps=2)
        assert all(pp.status[i][j] == 0 and pp.measured[i][j] for i in range(n) for j in range(n) if i != j)
        check_run(first + 1)  # directly after an atomics call: Ctrl, the pingpong lines and the slots are untouched
        assert_all_clean(p.Atomics(ref.CAS, ops=64, reps=2), False)
        check_run(first + 2)


def test_a_mapping_that_is_down_skips_only_that_cell(pkg):
    n = 4
    with open_same(pkg, n) as p:
        p.UnmapPeer(0, 1)
        r = p.Run()
        assert r.status[0][1] == ERR_STATE
        for kind in KINDS:
            at = p.Atomics(kind, ops=128, reps=2)
            assert not at.measured[0][1] and at.status[0][1] == r.status[0][1]
            assert at.ns_median[0][1] is None and at.digest[0][1] is None and at.raw.digest[1] == 0
            assert_clean(at, 1, 0)  # one-sided: the other direction still runs
            assert_all_clean(at, False, skip={(0, 1)})
        p.RemapPeer(0, 1)
        for kind in KINDS:
            assert_all_clean(p.Atomics(kind, ops=128, reps=2), False)


def test_simulated_mig_pairs_are_not_run(pkg):
    n = 2
    with open_same(pkg, n, flags=SIMULATE_MIG) as p:
        r = p.Run()
        at = p.Atomics(ref.FETCH_ADD)
        for i in range(n):
            for j in range(n):
                assert not at.measured[i][j] and at.ns_median[i][j] is None
                if i != j:
                    assert at.status[i][j] == r.status[i][j] == ERR_UNSUPPORTED


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_armed_fault_fails_exactly_its_cell(pkg, kind):
    n, ops, reps = 4, 200, 2
    with open_same(pkg, n) as p:
        for i, j in ((1, 3), (3, 0), (2, 1)):
            p.SetOption(pkg.abi.OPT_ATOMICS_FAULT, pkg.abi.atomics_fault(i, j))
            at = p.Atomics(kind, ops=ops, reps=reps)
            assert at.measured[i][j] and at.status[i][j] == ERR_INTEGRITY, (i, j, at.status[i][j])
            assert 0 < at.ns_min[i][j] <= at.ns_median[i][j] <= at.ns_max[i][j]
            if kind != ref.CONTENDED:
                assert at.digest[i][j] == ref.cell_digest(at.call_seq, kind, ops, reps, fault=True) \
                    != ref.cell_digest(at.call_seq, kind, ops, reps)
            assert_all_clean(at, False, skip={(i, j)})
            p.SetOption(pkg.abi.OPT_ATOMICS_FAULT, 0)
            assert_all_clean(p.Atomics(kind, ops=ops, reps=reps), False)
        # the armed cell must exist: a rank past n, rank 0 (the encoding is 1-based), or a diagonal without a loop-back
        for value in (pkg.abi.atomics_fault(0, n), pkg.abi.atomics_fault(n, 0), pkg.abi.atomics_fault(2, 2), 1, 1 << 16,
                      (1 << 32) | 0x10001):
            p.SetOption(pkg.abi.OPT_ATOMICS_FAULT, value)
            rc, t = p.atomics_raw(kind, ops, reps)
            assert rc == ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0, hex(value)
            assert (t.abi, t.n, t.kind, t.ops, t.reps) == (2, n, kind, ops, reps)
        p.SetOption(pkg.abi.OPT_ATOMICS_FAULT, 0)
        assert_all_clean(p.Atomics(kind, ops=ops, reps=reps), False)  # the handle stays usable


def test_fault_on_the_loopback_cell(pkg):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 20)) as p:
        p.SetOption(pkg.abi.OPT_ATOMICS_FAULT, pkg.abi.atomics_fault(0, 0))
        for kind in KINDS:
            at = p.Atomics(kind, ops=64, reps=1)
            assert at.status[0][0] == ERR_INTEGRITY, kind
        p.SetOption(pkg.abi.OPT_ATOMICS_FAULT, 0)
        for kind in KINDS:
            assert_all_clean(p.Atomics(kind, ops=64, reps=1), True)


def test_argument_errors_fill_the_output(pkg):
    a = pkg.abi
    with open_same(pkg, 2) as p:
        first = p.Atomics(a.ATOMIC_FETCH_ADD, ops=1, reps=1)  # the smallest call
        assert_all_clean(first, False)
        for kind, ops, reps in ((3, 0, 0), (a.ATOMIC_CAS, a.ATOMICS_MAX_OPS + 1, 0),
                                (a.ATOMIC_CONTENDED, 0, a.ATOMICS_MAX_REPS + 1), (1 << 31, 1 << 31, 1 << 31)):
            rc, t = p.atomics_raw(kind, ops, reps)
            assert rc == a.ERR_ARG, (kind, ops, reps)
            assert (t.abi, t.n, t.call_seq, t.row_mask) == (2, 2, 0, 0) and sum(t.measured) == 0
            assert (t.kind, t.ops, t.reps) == (kind, ops or a.ATOMICS_DEFAULT_OPS, reps or a.ATOMICS_DEFAULT_REPS)
        with pytest.raises(pkg.ProbeError):
            p.Atomics(3)
        big = p.Atomics(a.ATOMIC_CONTENDED, ops=a.ATOMICS_MAX_OPS, reps=1)  # the largest increment count
        assert big.call_seq == first.call_seq + 1
        assert_all_clean(big, False)
        last = p.Atomics(a.ATOMIC_CAS, ops=8, reps=a.ATOMICS_MAX_REPS)  # the largest rep field
        assert last.call_seq == 3
        assert_all_clean(last, False)


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    cfg = m.Config(ordinals=[0], bytes=1 << 20, world_size=world, rank=rank, session=session, flags=0x40, ctas=8,
                   timeout_ms=30000)

    def dump(at):
        return {"row_mask": at.row_mask, "measured": at.measured, "status": at.status, "digest": at.digest,
                "native": at.native, "ns_min": at.ns_min, "ns_median": at.ns_median, "kind": at.kind, "ops": at.ops,
                "reps": at.reps, "call_seq": at.call_seq}

    with m.Open(cfg) as p:
        out = {"calls": [dump(p.Atomics(k, ops=64, reps=2)) for k in range(3)]}
        r = p.Run(gather=True)
        out["run"] = {"reach": r.reach, "aborted": r.aborted, "run_seq": r.run_seq}
        if rank == 0:  # a call only this process makes: nothing waits for the other
            out["solo"] = dump(p.Atomics(0, ops=64, reps=2))
        r = p.Run(gather=True)
        out["run2"] = {"reach": r.reach, "aborted": r.aborted, "run_seq": r.run_seq}
    print("RESULT " + json.dumps(out))
    """
) % ROOT


def test_two_processes_fill_their_own_rows(pkg):
    """Both processes drive GPU 0, so their contexts are time-sliced and the times only need to be positive."""
    world = 2
    outs = run_children(CHILD, world)
    for rank, o in enumerate(outs):
        other = 1 - rank
        calls = o["calls"] + ([o["solo"]] if rank == 0 else [])
        assert [c["call_seq"] for c in calls] == list(range(1, len(calls) + 1))
        for c in calls:
            assert c["row_mask"] == 1 << rank
            assert c["measured"][rank] == [j != rank for j in range(world)]
            assert c["measured"][other] == [False] * world and c["digest"][other] == [None] * world
            assert c["native"][rank][other] == 2 and c["native"][other] == [None] * world
            assert c["status"][rank][other] == 0 and 0 < c["ns_min"][rank][other] <= c["ns_median"][rank][other]
            assert c["digest"][rank][other] == ref.cell_digest(c["call_seq"], c["kind"], c["ops"], c["reps"])
        for run in (o["run"], o["run2"]):
            assert run["reach"] == [[1] * world for _ in range(world)] and not run["aborted"]
        assert o["run2"]["run_seq"] == o["run"]["run_seq"] + 1
