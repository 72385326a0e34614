"""Rep records where the rest of the suite could not see a wrong value, each found by a mutant of tests/mutants.py
that no other test killed:
  * pingpong's and the atomics' digests over an odd number of round trips or ops and of reps.  At the default counts
    (256 trips, 1024 ops, multiples of 4 from an aligned start) every rep's xor of echoes or returns is 0, the same as
    the xor of the pings or of any regrouping of the lanes' returns, and at an even number of reps the reps cancel too,
    so a digest of the wrong words passes;
  * rep times of short reps: a rep stamped late by a constant hides in the C-versus-8C comparison of 2048-trip reps
    and in the ladder's lower bound at its HBM floor;
  * the two-shot's armed fault in timed rep 1 of three reps, where the older tests run one."""
import pytest

import atomics_ref
import pingpong_ref

pytestmark = pytest.mark.gpu

SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE


def open_same(pkg, n, nbytes=1 << 20):
    return pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME if n > 1 else 0, ctas=8, timeout_ms=20000))


@pytest.mark.parametrize("trips", [1, 5, 33])
@pytest.mark.parametrize("fenced", [False, True], ids=["plain", "fenced"])
def test_pingpong_digest_over_an_odd_number_of_trips(pkg, trips, fenced):
    n = 3
    with open_same(pkg, n) as p:
        pp = p.PingPong(trips=trips, reps=2, fenced=fenced)
        pl = pkg.plan(n, 1 << 20, 1)
        for i in range(n):
            for j in range(n):
                if i == j:
                    continue
                want = pingpong_ref.cell_digest(pp.call_seq, pl.partner, pl.rounds, i, j, trips, 2)
                assert want != 0, (i, j)  # the check below can tell a wrong echo from a right one
                assert pp.status[i][j] == 0 and pp.digest[i][j] == want, (i, j, pp.status[i][j], pp.digest[i][j])


@pytest.mark.parametrize("ops", [1, 5, 33])
@pytest.mark.parametrize("kind", [0, 1, 2], ids=["fetch_add", "cas", "contended"])
def test_atomics_digest_over_an_odd_number_of_ops(pkg, kind, ops):
    """The contended kind's 32 x ops returns of a rep are one aligned block whose xor is 0 at any ops; at an odd ops
    each lane's share no longer cancels on its own, so a digest that regroups the lanes' xors is no longer 0."""
    with open_same(pkg, 2) as p:
        at = p.Atomics(kind=kind, ops=ops, reps=2)
        want = atomics_ref.cell_digest(at.call_seq, at.kind, at.ops, at.reps)
        assert (want != 0) == (kind != 2)
        for i, j in ((0, 1), (1, 0)):
            assert at.measured[i][j] and at.status[i][j] == 0, (i, j, at.status[i][j])
            assert at.digest[i][j] == want, (i, j)


def test_short_pingpong_reps_are_not_padded(pkg):
    """Per round trip, reps of 16 trips and of 256 trips agree within a factor of 2: a constant added to every rep
    (100 us against about 25 us of 16 round trips) does not."""
    with open_same(pkg, 2) as p:
        short, long_ = (p.PingPong(trips=t, reps=5) for t in (16, 256))
        for i, j in ((0, 1), (1, 0)):
            assert short.status[i][j] == long_.status[i][j] == 0
            ratio = short.ns_median[i][j] / long_.ns_median[i][j]
            assert 0.5 <= ratio <= 2.0, (i, j, short.ns_median[i][j], long_.ns_median[i][j])


def test_short_bwcurve_reps_are_not_padded(pkg):
    """At N = 1 the ladder's smallest size, 4 KiB of local HBM, takes a rep of a few us (1.2-1.5 us on an H100 at
    700 W, profiles/h100_bwcurve_n1.json); under 50 us is a plausibility bound, not a performance claim."""
    with open_same(pkg, 1, nbytes=4 << 20) as p:
        bw = p.BwCurve(reps=3)
        assert bw.status[0][0] == 0 and bw.sizes[0] == 4096
        assert 0 < bw.ns_median[0][0][0] < 50000, bw.ns_median[0][0]
        assert bw.t0_ns[0][0] == bw.ns_median[0][0][0]


def test_twoshot_fault_acts_in_timed_rep_1_of_3_only(pkg):
    a = pkg.abi
    n, k, word = 3, 2, 1000
    with open_same(pkg, n, nbytes=2 << 20) as p:
        assert p.Info().bytes_per_pair == 1 << 20
        p.SetOption(a.OPT_ALLREDUCE_TWOSHOT_FAULT, a.allreduce_twoshot_fault(1, k, word))
        ar = p.AllReduceTwoShot(reps=3)
        p.SetOption(a.OPT_ALLREDUCE_TWOSHOT_FAULT, 0)
        for r in range(n):
            for kk in range(len(ar.sizes)):
                hit = (r, kk) == (1, k)
                assert ar.bad_words[r][kk] == (1 if hit else 0), (r, kk, ar.bad_words[r][kk])
                if hit:
                    assert ar.first_bad[r][kk] == 8 * word
            assert ar.bad_sizes[r] == (1 << k if r == 1 else 0), r
