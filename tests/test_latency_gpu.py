"""cdprobe_latency on the GPU: every chased cell's digest equals the restatement in tests/latency_ref.py, so a chase
that read the wrong words cannot pass; the times are plausible; cells whose mapping is down are never read; the call
needs no run and disturbs none.  Several ranks share one device where a test needs N > 1."""
import textwrap

import pytest

import latency_ref as ref
from conftest import ROOT
from harness import run_children

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
LOCAL_DIAG = 0x04
SIMULATE_MIG = 0x200
ERR_INTEGRITY = -10


def first_word(oracle, n, mode, i, j, bpp):
    """Index of the cell's word 0 in j's source buffer: the slice of i's slot in j (the diagonal slot n - 1), slice 0
    in full mode."""
    slot = n - 1 if i == j else oracle.lib().cdoracle_slot(i, j)
    return ref.first_word(0 if mode == 2 else slot, bpp)


def want_digest(oracle, lat, n, mode, i, j, words=None):
    bpp = lat.region_bytes
    return ref.digest(SEED, i, j, first_word(oracle, n, mode, i, j, bpp), bpp // ref.LINE_BYTES, lat.hops, lat.reps,
                      words)


def assert_clean(lat, i, j):
    assert lat.measured[i][j] and lat.status[i][j] == 0, (i, j, lat.status[i][j])
    assert 0 < lat.ns_min[i][j] <= lat.ns_median[i][j] <= lat.ns_max[i][j], (i, j)
    assert 50 <= lat.ns_median[i][j] <= 50000, (i, j, lat.ns_median[i][j])  # plausibility, not a performance claim


@pytest.mark.parametrize("nbytes", [128, 1 << 20, 1 << 30], ids=["128B", "1MiB", "1GiB"])
def test_loopback_chase_digest_and_times(pkg, oracle, nbytes):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes)) as p:
        lat = p.Latency()
        assert (lat.n, lat.row_mask, lat.hops, lat.reps, lat.region_bytes) == (1, 1, 1024, 8, nbytes)
        assert_clean(lat, 0, 0)
        assert lat.digest[0][0] == want_digest(oracle, lat, 1, 1, 0, 0) and lat.ms > 0
        lat2 = p.Latency(hops=100, reps=3)
        assert (lat2.hops, lat2.reps) == (100, 3)
        assert_clean(lat2, 0, 0)
        assert lat2.digest[0][0] == want_digest(oracle, lat2, 1, 1, 0, 0)


def test_callable_before_the_first_run_and_disturbs_nothing(pkg, oracle):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 20)) as p:
        lat = p.Latency()
        assert_clean(lat, 0, 0)
        r1 = p.Run()
        assert r1.verdict
        bpp = r1.bytes_per_pair
        assert (r1.sum_read[0][0], r1.xor_read[0][0]) == oracle.src_checksum(SEED, 0, 0, bpp // 8)
        assert (r1.sum_write[0][0], r1.xor_write[0][0]) == oracle.write_checksum(SEED, 0, 0, r1.run_seq, bpp // 8)
        assert p.Latency().digest[0][0] == lat.digest[0][0]
        for op in ("read", "write"):  # the run's regions are as it left them
            d = p.Diagnose(op, 0, 0)
            assert d.bad_words == 0 and d.run_seq == r1.run_seq
        r2 = p.Run()
        assert r2.verdict and r2.run_seq == r1.run_seq + 1
        assert (r2.sum_write[0][0], r2.xor_write[0][0]) == oracle.write_checksum(SEED, 0, 0, r2.run_seq, bpp // 8)


@pytest.mark.parametrize("flags", [0, LOCAL_DIAG], ids=["no-diag", "local-diag"])
@pytest.mark.parametrize("mode", [1, 2], ids=["sliced", "full"])
def test_same_device_every_cell(pkg, oracle, mode, flags):
    n = 4
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=4 << 20, mode=mode, flags=SAME | flags, ctas=8,
                             timeout_ms=20000)) as p:
        lat = p.Latency(hops=512, reps=4)
        assert lat.row_mask == (1 << n) - 1 and lat.region_bytes == p.Info().bytes_per_pair
        for i in range(n):
            for j in range(n):
                if i == j and not flags & LOCAL_DIAG:
                    assert not lat.measured[i][j] and lat.status[i][j] == 0 and lat.ns_median[i][j] is None
                    assert lat.digest[i][j] is None
                    continue
                assert_clean(lat, i, j)
                assert lat.digest[i][j] == want_digest(oracle, lat, n, mode, i, j), (i, j)
        r = p.Run()  # ranks sharing one device: reachability is judged, not the NVLink bandwidth gate
        assert r.reach == [[1] * n for _ in range(n)] and not r.aborted


def test_a_mapping_that_is_down_is_not_read(pkg, oracle):
    n = 2
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=1 << 20, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        p.UnmapPeer(0, 1)
        r = p.Run()
        assert r.status[0][1] != 0
        lat = p.Latency()
        assert not lat.measured[0][1] and lat.status[0][1] == r.status[0][1]
        assert lat.ns_min[0][1] is None and lat.digest[0][1] is None and lat.raw.digest[1] == 0
        assert_clean(lat, 1, 0)
        assert lat.digest[1][0] == want_digest(oracle, lat, n, 1, 1, 0)
        p.RemapPeer(0, 1)
        lat = p.Latency()
        for i, j in ((0, 1), (1, 0)):
            assert_clean(lat, i, j)
            assert lat.digest[i][j] == want_digest(oracle, lat, n, 1, i, j)


def test_a_corrupted_word_on_the_path_fails_the_cell(pkg, oracle):
    nbytes = 1 << 20
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes)) as p:
        lines = nbytes // ref.LINE_BYTES
        k = ref.loaded_word(SEED, 0, 0, 0, lines, rep=2, hop=10)
        mask = 0x0123456789ABCDEF
        p.Corrupt(0, 8 * k, mask)
        lat = p.Latency()
        assert lat.measured[0][0] and lat.status[0][0] == ERR_INTEGRITY
        bad = {k: ref.src_word(SEED, 0, k) ^ mask}
        assert lat.digest[0][0] == want_digest(oracle, lat, 1, 1, 0, 0, bad)
        assert lat.digest[0][0] != want_digest(oracle, lat, 1, 1, 0, 0)
        p.Corrupt(0, 8 * k, mask)
        lat = p.Latency()
        assert_clean(lat, 0, 0)
        assert lat.digest[0][0] == want_digest(oracle, lat, 1, 1, 0, 0)


def test_simulated_mig_pairs_are_not_read(pkg):
    n = 2
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=1 << 20, flags=SAME | SIMULATE_MIG, ctas=8, timeout_ms=20000)) as p:
        r = p.Run()
        lat = p.Latency()
        for i in range(n):
            for j in range(n):
                assert not lat.measured[i][j] and lat.ns_median[i][j] is None
                if i != j:
                    assert lat.status[i][j] == r.status[i][j] != 0


def test_errors_fill_the_output(pkg):
    a = pkg.abi
    with pkg.Open(pkg.Config(ordinals=[0, 0], bytes=1 << 20, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        for hops, reps in ((a.LATENCY_MAX_HOPS + 1, 0), (0, a.LATENCY_MAX_REPS + 1), (1 << 31, 1 << 31)):
            rc, t = p.latency_raw(hops, reps)
            assert rc == a.ERR_ARG, (hops, reps)
            assert (t.abi, t.n, t.region_bytes) == (2, 2, p.Info().bytes_per_pair) and sum(t.measured) == 0
            assert (t.hops, t.reps) == (hops or a.LATENCY_DEFAULT_HOPS, reps or a.LATENCY_DEFAULT_REPS)
        with pytest.raises(pkg.ProbeError):
            p.Latency(hops=a.LATENCY_MAX_HOPS + 1)
        rc, t = p.latency_raw(1, 1)  # the smallest chase
        assert rc == a.OK and (t.hops, t.reps) == (1, 1) and t.measured[1] and t.measured[16]
        rc, t = p.latency_raw(a.LATENCY_MAX_HOPS // 64, a.LATENCY_MAX_REPS)
        assert rc == a.OK and t.reps == 64 and t.status[1] == 0


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    cfg = m.Config(ordinals=[0], bytes=1 << 20, world_size=world, rank=rank, session=session, flags=0x40, ctas=8,
                   timeout_ms=30000)
    with m.Open(cfg) as p:
        out = []
        for _ in range(2):
            lat = p.Latency()
            out.append({"row_mask": lat.row_mask, "measured": lat.measured, "status": lat.status, "digest": lat.digest,
                        "ns_min": lat.ns_min, "ns_median": lat.ns_median, "hops": lat.hops, "reps": lat.reps,
                        "bpp": lat.region_bytes})
            r = p.Run(gather=True)
            out[-1].update(reach=r.reach, aborted=r.aborted, run_seq=r.run_seq, verdict=r.verdict,
                           slow_pairs=r.slow_pairs, unreachable_pairs=r.unreachable_pairs)
    print("RESULT " + json.dumps(out))
    """
) % ROOT


def test_two_processes_fill_their_own_rows(pkg, oracle):
    """Both processes drive GPU 0, so their contexts are time-sliced: the chases' times then include slices of the
    other context and only need to be positive, and the probe's bandwidth verdict is not judged (as in the other
    two-process tests); every pair must stay reachable around the latency calls."""
    world = 2
    outs = run_children(CHILD, world, timeout=300)
    for rank, per_call in enumerate(outs):
        other = 1 - rank
        for o in per_call:
            assert o["row_mask"] == 1 << rank
            assert o["measured"][rank] == [False if j == rank else True for j in range(world)]
            assert o["measured"][other] == [False] * world and o["digest"][other] == [None] * world
            assert o["status"][rank][other] == 0 and 0 < o["ns_min"][rank][other] <= o["ns_median"][rank][other]
            assert o["reach"] == [[1] * world for _ in range(world)] and not o["aborted"], o
            lines = o["bpp"] // ref.LINE_BYTES
            first = first_word(oracle, world, 1, rank, other, o["bpp"])
            assert o["digest"][rank][other] == ref.digest(SEED, rank, other, first, lines, o["hops"], o["reps"])
        assert [o["run_seq"] for o in per_call] == [per_call[0]["run_seq"], per_call[0]["run_seq"] + 1]
    assert [o["reach"] for o in outs[0]] == [o["reach"] for o in outs[1]]  # after cdprobe_gather
