"""The write verify rejects a corrupted landing slot, on every schedule and data path.

A write cell passes when the owner re-reads its landing slot (K4), finds the (S, X) the writer published, and routes
that verdict back to the writer's row.  cdprobe_corrupt_landing xors words into the slot after the write has completed
and before any rank verifies it, with the writer's published (S, X) untouched: a fault in transit.  Each test runs to
completion with exactly the armed cell failing, the writer's checksum still equal to the oracle's, and
cdprobe_diagnose's whole report on the slot equal to the CPU reference (tests/word_ref.py).  No test here aborts a run."""
import json
import random
import subprocess
import sys
import textwrap
import uuid

import pytest

import word_ref as ref
from conftest import ROOT, gpu_count
from test_words_gpu import assert_report, observed, region_offset, want_dict

pytestmark = pytest.mark.gpu

NGPU = gpu_count()
SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
LOCAL_DIAG = 0x04
G = ref.GRANULE_WORDS


def same_device(pkg, n, nbytes, flags=0):
    return pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME | flags, ctas=8, timeout_ms=20000))


def flip_mask(rng):
    return rng.choice((1 << rng.randrange(64), rng.getrandbits(64) | 1))


def assert_only_write_cell_fails(r, i, j, n, diag, ops=3):
    """reach_write[i][j] == 0 and every other probed bit is 1; the run completed."""
    ones = [[1] * n for _ in range(n)]
    want_w = [row[:] for row in ones]
    want_w[i][j] = 0
    ctx = (i, j, r.reach_read, r.reach_write)
    assert r.reach_write == want_w, ctx
    assert r.reach_read == (ones if ops & 1 else [[0 if (a == b and diag) else 1 for b in range(n)] for a in range(n)]), ctx
    assert not r.aborted and r.slow_pairs == 0, ctx
    if i != j:
        assert r.unreachable_pairs == 1 and not r.verdict, ctx
    elif n == 1:
        assert r.unreachable_pairs == 0 and not r.verdict, ctx
    else:  # in a multi-rank domain the loop-back cell is reported, not gated
        assert r.unreachable_pairs == 0 and r.verdict, ctx


def check_failing_cell(p, oracle, r, i, j, faults, nbytes, diag=False, ops=3):
    """The cell fails alone, its writer generated the oracle's pattern, and the slot holds that pattern with exactly
    `faults` xored in, read at rest by the target and through the issuer's mapping."""
    n = r.n
    assert_only_write_cell_fails(r, i, j, n, diag, ops)
    W = r.bytes_per_pair // 8
    assert (r.sum_write[i][j], r.xor_write[i][j]) == oracle.write_checksum(SEED, i, j, r.run_seq, W), (i, j)
    spec = ref.write_spec(SEED, n, i, j, r.run_seq, W)
    want = want_dict(spec, observed(spec, faults), "write", i, r.run_seq,
                     region_offset(oracle, n, nbytes, 1, diag, "write", i, j))
    for reader in sorted({i, j}):
        assert_report(p.Diagnose("write", i, j, reader=reader), want, (i, j, reader))
    return want


def check_clean(p, r, n, diag=False):
    want = [[1] * n for _ in range(n)]
    assert r.reach_write == want and r.verdict and not r.aborted and r.unreachable_pairs == 0
    for i in range(n):
        for j in range(n):
            if i != j or diag:
                assert p.Diagnose("write", i, j, reader=j).bad_words == 0, (i, j)


# ---- exactly one cell fails, every ordered cell, every data path ---------------------------------------------------
@pytest.mark.parametrize("n", [2, 3, 4, 5, 8])
def test_one_corrupted_landing_fails_exactly_its_cell(pkg, oracle, n):
    nbytes = 256 << 10
    rng = random.Random(n)
    with same_device(pkg, n, nbytes) as p:
        W = p.Run().bytes_per_pair // 8
        for path in (0, 1, 2):
            p.SetOption(pkg.abi.OPT_PATH, path)
            todo = [(i, j) for i in range(n) for j in range(n) if i != j]
            if n == 8 and path:
                todo = rng.sample(todo, 10)
            for i, j in todo:
                faults = [(rng.randrange(W), flip_mask(rng))]
                p.CorruptLanding(i, j, faults)  # replaces the previous cell's arming
                r = p.Run()
                check_failing_cell(p, oracle, r, i, j, faults, nbytes)
            p.CorruptLanding(0, 1, [])
            check_clean(p, p.Run(), n)


# ---- N = 1: the streamed pass, and the phase walk of a write-only probe --------------------------------------------
LOOPBACK = [(nb, path) for nb in (128, 8192 + 128, 16384 * 3 + 640, 1 << 20) for path in (0, 1, 2)] + [(1 << 30, 0)]


@pytest.mark.parametrize("nbytes,path", LOOPBACK)
def test_loopback_corrupted_landing(pkg, oracle, nbytes, path):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes)) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        assert p.Run().verdict
        W = nbytes // 8
        tail = (W - 1) // 1024 * 1024  # first word of the last 8 KiB unit
        idx = sorted({0, W - 1, tail + (W - tail) // 2})
        faults = [(k, 1 << (k % 64) | 1 << 63) for k in idx]
        p.CorruptLanding(0, 0, faults)
        check_failing_cell(p, oracle, p.Run(), 0, 0, faults, nbytes, diag=True)
        assert_only_write_cell_fails(p.Run(), 0, 0, 1, True)  # armed until disarmed
        p.CorruptLanding(0, 0, [])
        r = p.Run()
        check_clean(p, r, 1, diag=True)
        assert r.reach_read == [[1]]


@pytest.mark.parametrize("path", [0, 1, 2])
def test_loopback_write_only_takes_the_phase_walk(pkg, oracle, path):
    nbytes = 16384 * 3 + 640
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, ops=2)) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        assert p.Run().verdict
        assert [t["job0"] for t in p.Trace()] == ["write", "verify"]
        faults = [(0, 1 << 5), (nbytes // 8 - 1, 0xF0F0)]
        p.CorruptLanding(0, 0, faults)
        check_failing_cell(p, oracle, p.Run(), 0, 0, faults, nbytes, diag=True, ops=2)
        p.CorruptLanding(0, 0, [])
        check_clean(p, p.Run(), 1, diag=True)


# ---- every schedule ------------------------------------------------------------------------------------------------
SCHEDULES = [("unidirectional", 0x80, None), ("serial-verify", 0x100, None), ("overlap-verify-3", 0x20, 3),
             ("pair-barriers", 0x800, None), ("all-rank-barriers", 0x400, None), ("local-diag", LOCAL_DIAG, None)]


@pytest.mark.parametrize("flags,verify_ctas", [s[1:] for s in SCHEDULES], ids=[s[0] for s in SCHEDULES])
def test_corrupted_landing_on_every_schedule(pkg, oracle, flags, verify_ctas):
    n, nbytes = 4, 1 << 20
    diag = bool(flags & LOCAL_DIAG)
    rng = random.Random(flags)
    with same_device(pkg, n, nbytes, flags) as p:
        if verify_ctas:
            p.SetOption(pkg.abi.OPT_VERIFY_CTAS, verify_ctas)
        W = p.Run().bytes_per_pair // 8
        todo = [(i, j) for i in range(n) for j in range(n) if i != j or diag]
        for m, (i, j) in enumerate(todo):
            p.SetOption(pkg.abi.OPT_PATH, m % 3)
            faults = [(rng.randrange(W), flip_mask(rng))]
            p.CorruptLanding(i, j, faults)
            check_failing_cell(p, oracle, p.Run(), i, j, faults, nbytes, diag=diag)
        p.CorruptLanding(0, 0 if diag else 1, [])
        check_clean(p, p.Run(), n, diag)


# ---- every class of bad word, on the device ------------------------------------------------------------------------
def test_every_kind_in_one_write_cell(pkg, oracle):
    """Cell 0 -> 1 of N = 3 after 9 runs: ZERO, DISPLACED (this run's word from another index), STALE (the same writer
    1 and 8 runs back), FOREIGN (rank 2's salt into rank 1) and single- and multi-bit FLIPs in one slot."""
    n, nbytes = 3, 512 << 10
    with same_device(pkg, n, nbytes) as p:
        for _ in range(9):
            r = p.Run()
        W = r.bytes_per_pair // 8
        s = r.run_seq + 1  # the run the fault goes into

        def word(writer, seq, k):
            return int(ref.write_words(ref.write_salt(SEED, writer, 1, seq), k, 1)[0])

        def becomes(k, obs):  # the mask that turns word k of this run's pattern into `obs`
            return word(0, s, k) ^ obs

        faults = [(0, becomes(0, 0)),                                   # ZERO
                  (3 * G + 17, becomes(3 * G + 17, word(0, s, 5))),     # DISPLACED: this run's word 5
                  (4 * G, becomes(4 * G, word(0, s - 1, 4 * G))),       # STALE: the run before
                  (9 * G + 1, becomes(9 * G + 1, word(0, s - 8, 77))),  # STALE: 8 runs back
                  (10 * G + 2047, becomes(10 * G + 2047, word(2, s, 10 * G))),  # FOREIGN: rank 2's word
                  (W - 1, becomes(W - 1, word(2, s, W - 1))),           # FOREIGN, in the last word
                  (11 * G + 3, 1 << 40),                                # FLIP, one bit
                  (12 * G + 9, 0x00FF00000000F00F)]                     # FLIP, many bits
        p.CorruptLanding(0, 1, faults)
        r = p.Run()
        assert r.run_seq == s
        want = check_failing_cell(p, oracle, r, 0, 1, faults, nbytes)
        assert want["kind_count"] == [2, 1, 1, 2, 2]  # flip, zero, displaced, stale, foreign
        assert sorted(x["run_seq"] for x in want["sample"] if x["kind"] == ref.STALE) == [s - 8, s - 1]
        p.CorruptLanding(0, 1, [])
        check_clean(p, p.Run(), n)


# ---- the write side of the (S, X) blind spot -----------------------------------------------------------------------
def test_write_checksum_blind_spot_on_the_device(pkg, oracle):
    """Mirrors the read side: two words of one granule swapped, or one word each of granules 1 and 64 (fold6 1 both),
    pass the write verify; one word each of granules 0 and 1 swapped changes X only, and two words of one granule xored
    with the same mask change S only, and both fail it."""
    nbytes = 2 << 20
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes)) as p:
        r = p.Run()
        W = r.bytes_per_pair // 8
        assert W == 128 * G and r.verdict

        def arm_swap(a, b):
            s = r.run_seq + 1
            e = ref.write_words(ref.write_salt(SEED, 0, 0, s), 0, W)
            m = int(e[a] ^ e[b])
            p.CorruptLanding(0, 0, [(a, m), (b, m)])
            return [(a, m), (b, m)]

        for a, b in ((3 * G + 5, 3 * G + 2000), (1 * G + 7, 64 * G + 7)):
            faults = arm_swap(a, b)
            r = p.Run()
            assert r.reach_write[0][0] == 1 and r.verdict, (a, b)
            d = p.Diagnose("write", 0, 0)
            assert d.bad_words == 2 and d.kinds["displaced"] == 2, (a, b)
            assert [(x["offset"], x["word"]) for x in d.samples] == [(8 * a, b), (8 * b, a)]
            spec = ref.write_spec(SEED, 1, 0, 0, r.run_seq, W)
            assert_report(d, want_dict(spec, observed(spec, faults), "write", 0, r.run_seq,
                                       region_offset(oracle, 1, nbytes, 1, True, "write", 0, 0)), (a, b))
        faults = arm_swap(7, G + 7)  # fold6 0 and 1: X changes, S does not
        r = p.Run()
        check_failing_cell(p, oracle, r, 0, 0, faults, nbytes, diag=True)
        # the same one-bit mask on two words of a granule: X does not change, and S does when the bit is equal in both
        a, b = 5 * G + 1, 5 * G + 2
        e = ref.write_words(ref.write_salt(SEED, 0, 0, r.run_seq + 1), a, 2)
        bit = next(t for t in range(64) if (int(e[0]) >> t & 1) == (int(e[1]) >> t & 1))
        faults = [(a, 1 << bit), (b, 1 << bit)]
        p.CorruptLanding(0, 0, faults)
        r = p.Run()
        check_failing_cell(p, oracle, r, 0, 0, faults, nbytes, diag=True)
        p.CorruptLanding(0, 0, [])
        check_clean(p, p.Run(), 1, diag=True)


# ---- a read fault and a write fault in one run ---------------------------------------------------------------------
def test_read_and_write_faults_fail_their_own_cells(pkg, oracle):
    n, nbytes = 2, 1 << 20
    with same_device(pkg, n, nbytes) as p:
        W = p.Run().bytes_per_pair // 8
        p.Corrupt(0, 8 * 100, 1 << 3)  # rank 0's slice 0: what rank 1 reads
        faults = [(W // 2, 1 << 50)]
        p.CorruptLanding(0, 1, faults)
        r = p.Run()
        assert r.reach_read == [[1, 1], [0, 1]] and r.reach_write == [[1, 0], [1, 1]]
        assert r.unreachable_pairs == 2 and not r.verdict and not r.aborted and r.slow_pairs == 0
        assert (r.sum_write[0][1], r.xor_write[0][1]) == oracle.write_checksum(SEED, 0, 1, r.run_seq, W)
        d = p.Diagnose("read", 1, 0)
        assert d.bad_words == 1 and d.first_bad == 8 * 100 and d.bit_flips[3] == 1
        spec = ref.write_spec(SEED, n, 0, 1, r.run_seq, W)
        want = want_dict(spec, observed(spec, faults), "write", 0, r.run_seq,
                         region_offset(oracle, n, nbytes, 1, False, "write", 0, 1))
        assert_report(p.Diagnose("write", 0, 1, reader=1), want)
        assert p.Diagnose("write", 1, 0, reader=0).bad_words == 0
        p.Corrupt(0, 8 * 100, 1 << 3)
        p.CorruptLanding(0, 1, [])
        check_clean(p, p.Run(), n)


# ---- two processes on one GPU --------------------------------------------------------------------------------------
CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, nbytes, k, mask = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5])
    cfg = m.Config(ordinals=[0], bytes=nbytes, world_size=2, rank=rank, session=session, flags=0x40, ctas=8,
                   timeout_ms=30000)
    with m.Open(cfg) as p:
        p.Run(gather=True)
        if rank == 0:
            p.CorruptLanding(0, 1, [(k, mask)])
        r = p.Run(gather=True)
        d = p.Diagnose("write", 0, 1, reader=rank)  # rank 1 at rest, rank 0 through the imported handle
        raw = {f: getattr(d.raw, f) for f, _ in d.raw._fields_ if f not in ("ms", "reader", "kind_count", "bit_flips", "sample")}
        raw["kind_count"] = list(d.raw.kind_count)
        raw["bit_flips"] = list(d.raw.bit_flips)
        raw["sample"] = [{f: getattr(s, f) for f, _ in s._fields_} for s in d.raw.sample]
        if rank == 0:
            p.CorruptLanding(0, 1, [])
        r2 = p.Run(gather=True)
        out = {"reach_read": r.reach_read, "reach_write": r.reach_write, "verdict": r.verdict, "aborted": r.aborted,
               "unreachable": r.unreachable_pairs, "run_seq": r.run_seq, "bpp": r.bytes_per_pair,
               "sum_write": r.sum_write[0][1], "xor_write": r.xor_write[0][1], "diag": raw,
               "after": {"reach": r2.reach, "verdict": r2.verdict}}
    print("RESULT " + json.dumps(out))
    """
) % ROOT


def test_two_processes_one_gpu(pkg, oracle):
    nbytes, k, mask = 1 << 20, 12345, 0x8000000000000001
    session = f"lf-{uuid.uuid4().hex[:12]}"
    procs = [subprocess.Popen([sys.executable, "-c", CHILD, session, str(r), str(nbytes), str(k), str(mask)],
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(2)]
    outs = []
    for pr in procs:
        so, se = pr.communicate(timeout=300)
        assert pr.returncode == 0, se[-2000:]
        outs.append(json.loads([l for l in so.splitlines() if l.startswith("RESULT ")][-1][7:]))
    for rank, o in enumerate(outs):
        assert o["reach_read"] == [[1, 1], [1, 1]] and o["reach_write"] == [[1, 0], [1, 1]], rank
        assert not o["verdict"] and not o["aborted"] and o["unreachable"] == 1, rank
        assert o["after"] == {"reach": [[1, 1], [1, 1]], "verdict": True}, rank
    o = outs[0]
    W = o["bpp"] // 8
    assert (o["sum_write"], o["xor_write"]) == oracle.write_checksum(SEED, 0, 1, o["run_seq"], W)
    spec = ref.write_spec(SEED, 2, 0, 1, o["run_seq"], W)
    want = want_dict(spec, observed(spec, [(k, mask)]), "write", 0, o["run_seq"],
                     region_offset(oracle, 2, nbytes, 1, False, "write", 0, 1))
    for rank, o in enumerate(outs):
        assert o["diag"] == want, rank


# ---- real NVLink ---------------------------------------------------------------------------------------------------
@pytest.mark.skipif(NGPU < 2, reason="needs >= 2 GPUs")
def test_real_peer_corrupted_landing(pkg, oracle):
    n, nbytes = 2, 16 << 20
    with pkg.Open(pkg.Config(ordinals=[0, 1], bytes=nbytes, timeout_ms=20000)) as p:
        W = p.Run().bytes_per_pair // 8
        for path in (0, 1, 2):
            p.SetOption(pkg.abi.OPT_PATH, path)
            faults = [(0, 1), (W - 1, 1 << 63), (W // 3, 0xDEADBEEF)]
            p.CorruptLanding(0, 1, faults)
            check_failing_cell(p, oracle, p.Run(), 0, 1, sorted(faults), nbytes)
        p.CorruptLanding(0, 1, [])
        check_clean(p, p.Run(), n)


# ---- arming errors -------------------------------------------------------------------------------------------------
def test_arming_errors(pkg):
    a = pkg.abi
    with same_device(pkg, 2, 1 << 20) as p:
        W = p.Run().bytes_per_pair // 8
        p.CorruptLanding(0, 1, [(3, 1)])
        for local, target, faults in [(2, 1, [(3, 1)]),                       # local rank out of range
                                      (0, 2, [(3, 1)]),                       # target out of range
                                      (0, 1, [(k, 1) for k in range(9)]),     # more than 8 words
                                      (0, 1, [(W, 1)]),                       # one past the slot
                                      (0, 1, [(5, 1), (5, 2)]),               # a repeated word
                                      (0, 1, [(5, 0)]),                       # a zero mask
                                      (0, 0, [(5, 1)])]:                      # no loop-back slot at n = 2
            assert p.corrupt_landing_raw(local, target, faults) == a.ERR_ARG, (local, target, faults)
        assert p._lib.cdprobe_corrupt_landing(p._h, 0, 1, 1, None, None) == a.ERR_ARG
        with pytest.raises(pkg.ProbeError):
            p.CorruptLanding(0, 1, [(W, 1)])
        # a refused call leaves the earlier arming in place
        r = p.Run()
        assert_only_write_cell_fails(r, 0, 1, 2, False)
        # arming another cell replaces it
        p.CorruptLanding(1, 0, [(3, 1)])
        assert_only_write_cell_fails(p.Run(), 1, 0, 2, False)
        p.CorruptLanding(1, 0, [])
        check_clean(p, p.Run(), 2)
        # an unmapped target
        p.UnmapPeer(0, 1)
        assert p.corrupt_landing_raw(0, 1, [(3, 1)]) == a.ERR_STATE
        p.RemapPeer(0, 1)
        check_clean(p, p.Run(), 2)
