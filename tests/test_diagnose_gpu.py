"""cdprobe_diagnose on the GPU: clean regions stay clean, injected faults are counted, located and classified exactly,
the samples are deterministic, and the call disturbs nothing.  Several ranks share one device where a test needs N > 1."""
import ctypes as C

import pytest

from conftest import gpu_count

pytestmark = pytest.mark.gpu

NGPU = gpu_count()
SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
U64_MAX = (1 << 64) - 1
GRANULE = 16384
KINDS = ("flip", "zero", "displaced", "stale", "foreign")


def kinds(**kw):
    return {k: kw.get(k, 0) for k in KINDS}


def report(d):
    """Everything a diagnosis says about the bytes (not who read them, nor how long it took)."""
    raw = d.raw
    return ({f: getattr(raw, f) for f, _ in raw._fields_ if f not in ("reader", "ms", "kind_count", "bit_flips", "sample")},
            list(raw.kind_count), list(raw.bit_flips), d.samples)


@pytest.mark.parametrize("path", [0, 1, 2], ids=["tma", "ldst", "ldst32"])
def test_clean_regions_after_a_passing_run(pkg, oracle, path):
    nbytes = 1 << 30
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes)) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        r = p.Run()
        assert r.verdict
        for op in ("read", "write"):
            d = p.Diagnose(op, 0, 0)
            assert d.bad_words == 0 and d.raw.n_samples == 0 and d.samples == [] and d.bad_granules == 0
            assert d.raw.first_bad == U64_MAX and d.first_bad is None and d.bytes == r.bytes_per_pair
            assert d.run_seq == r.run_seq and d.kinds == kinds() and d.bit_flips == [0] * 64 and d.ms > 0
        # diagnosing disturbs nothing: the next run passes with the oracle's checksums
        r2 = p.Run()
        assert r2.verdict
        bpp = r2.bytes_per_pair
        assert (r2.sum_read[0][0], r2.xor_read[0][0]) == oracle.src_checksum(SEED, 0, 0, bpp // 8)
        assert (r2.sum_write[0][0], r2.xor_write[0][0]) == oracle.write_checksum(SEED, 0, 0, r2.run_seq, bpp // 8)


def test_flipped_bits_are_counted_located_and_sampled(pkg, oracle):
    L = oracle.lib()
    with pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 20)) as p:
        assert p.Run().verdict
        faults = [(4096 + 8, 1 << 17), (4096 + 64, 1 << 17), (3 * GRANULE + 128, 0xFF00)]  # granules 0 and 3
        for off, mask in faults:
            p.Corrupt(0, off, mask)
        r = p.Run()
        assert r.reach_read[0][0] == 0 and not r.verdict
        d = p.Diagnose("read", 0, 0)
        assert (d.bad_words, d.bad_granules, d.first_bad, d.last_bad) == (3, 2, 4096 + 8, 3 * GRANULE + 128)
        assert d.kinds == kinds(flip=3) and d.zero_words == 0
        assert d.bit_flips == [2 if b == 17 else 1 if 8 <= b <= 15 else 0 for b in range(64)]
        assert [s["offset"] for s in d.samples] == [off for off, _ in faults]
        for s, (off, mask) in zip(d.samples, faults):
            exp = L.cdoracle_src_word(SEED, 0, off // 8)
            assert (s["expected"], s["observed"], s["kind"], s["rank"]) == (exp, exp ^ mask, "flip", -1)
        for off, mask in faults:
            p.Corrupt(0, off, mask)
        assert p.Run().verdict
        assert p.Diagnose("read", 0, 0).bad_words == 0


def test_read_cell_kinds(pkg, oracle):
    """N = 4 ranks on one device: on the slice rank 2 reads from rank 0, a ZERO, two DISPLACED (one from another
    slice, one from its own) and a FOREIGN word (rank 3's).  The issuer and the owner see the same report."""
    L = oracle.lib()
    n = 4
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=1 << 20, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        bpp = p.Info().bytes_per_pair
        W = bpp // 8  # slice 1 of rank 0 (rank 2's slot among rank 0's peers) starts at word W

        def sw(rank, k):
            return L.cdoracle_src_word(SEED, rank, k)

        kz, kd, kd2, kf = 3, 2100, 2101, 5000
        p.Corrupt(0, bpp + 8 * kz, sw(0, W + kz))                        # -> 0
        p.Corrupt(0, bpp + 8 * kd, sw(0, W + kd) ^ sw(0, 7))             # -> word 7 (slice 0)
        p.Corrupt(0, bpp + 8 * kd2, sw(0, W + kd2) ^ sw(0, W + 10))      # -> word W + 10 (same slice)
        p.Corrupt(0, bpp + 8 * kf, sw(0, W + kf) ^ sw(3, W + kf))        # -> rank 3's word
        r = p.Run()
        exp = [[1] * n for _ in range(n)]
        exp[2][0] = 0
        assert r.reach_read == exp
        d = p.Diagnose("read", 2, 0)
        assert d.reader == 2 and d.region_offset == (2 << 20) + bpp and d.bytes == bpp
        assert d.bad_words == 4 and d.bad_granules == 3 and d.zero_words == 1
        assert d.kinds == kinds(zero=1, displaced=2, foreign=1) and d.bit_flips == [0] * 64
        assert [(s["offset"], s["kind"], s["rank"], s["word"]) for s in d.samples] == [
            (8 * kz, "zero", -1, 0), (8 * kd, "displaced", 0, 7), (8 * kd2, "displaced", 0, W + 10),
            (8 * kf, "foreign", 3, W + kf)]
        for s in d.samples:
            assert s["expected"] == sw(0, W + s["offset"] // 8)
        d0 = p.Diagnose("read", 2, 0, reader=0)
        assert d0.reader == 0 and report(d0) == report(d)


def test_write_cell_never_written_reads_zero(pkg):
    with pkg.Open(pkg.Config(ordinals=[0, 0], bytes=1 << 20, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        p.UnmapPeer(0, 1)
        r = p.Run()
        assert r.reach_write[0][1] == 0 and r.status[0][1] != 0
        d = p.Diagnose("write", 0, 1, reader=1)
        W = d.bytes // 8
        assert d.bad_words == W and d.zero_words == W and d.kinds == kinds(zero=W)
        assert d.first_bad == 0 and d.last_bad == d.bytes - 8 and d.bad_granules == -(-d.bytes // GRANULE)
        assert [s["offset"] for s in d.samples] == [8 * k for k in range(16)]
        rc, raw = p.diagnose_raw(pkg.abi.OP_WRITE, 0, 1, 0)  # rank 0's mapping of rank 1 is down: never read through it
        assert rc == pkg.abi.ERR_STATE and (raw.abi, raw.op, raw.issuer, raw.target, raw.reader) == (2, 2, 0, 1, 0)


def test_write_cell_that_missed_a_run_holds_the_previous_runs_pattern(pkg, oracle):
    L = oracle.lib()
    with pkg.Open(pkg.Config(ordinals=[0, 0], bytes=64 << 20, flags=SAME, ctas=16, timeout_ms=20000)) as p:
        r1 = p.Run()
        assert r1.verdict
        p.UnmapPeer(0, 1)
        r2 = p.Run()
        assert r2.reach_write[0][1] == 0
        d = p.Diagnose("write", 0, 1, reader=1)
        W = d.bytes // 8
        assert d.bytes == 64 << 20 and d.run_seq == r2.run_seq
        assert d.bad_words == W and d.kinds == kinds(stale=W) and d.bit_flips == [0] * 64 and d.bad_granules == W // 2048
        new, old = L.cdoracle_write_salt(SEED, 0, 1, r2.run_seq), L.cdoracle_write_salt(SEED, 0, 1, r1.run_seq)
        for k, s in enumerate(d.samples):
            assert (s["offset"], s["kind"], s["rank"], s["word"], s["run_seq"]) == (8 * k, "stale", 0, k, r1.run_seq)
            assert (s["expected"], s["observed"]) == (L.cdoracle_write_word(new, k), L.cdoracle_write_word(old, k))
        assert p.diagnose_raw(pkg.abi.OP_WRITE, 0, 1, 0)[0] == pkg.abi.ERR_STATE


def test_samples_are_the_lowest_offsets_in_order_and_repeatable(pkg):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=4 << 20)) as p:
        assert p.Run().verdict
        offs = [200 * GRANULE + 8 * k for k in range(0, 40, 2)] + [5 * GRANULE + 8 * k for k in (1, 9, 100, 2047)] + \
               [64 * k for k in range(10)] + [37 * GRANULE + 16 * 32 * 7]
        for o in offs:
            p.Corrupt(0, o, 1 << (o // 8 % 64))
        assert not p.Run().verdict
        d1, d2 = p.Diagnose("read", 0, 0), p.Diagnose("read", 0, 0)
        assert d1.bad_words == len(offs) and d1.raw.n_samples == 16 and d1.bad_granules == 4
        assert [s["offset"] for s in d1.samples] == sorted(offs)[:16]
        assert d1.samples[0]["offset"] == d1.first_bad and d1.last_bad == max(offs)
        assert sum(d1.bit_flips) == len(offs) and d1.kinds == kinds(flip=len(offs))
        d1.raw.ms = d2.raw.ms = 0.0
        assert bytes(d1.raw) == bytes(d2.raw)


def test_errors_fill_the_output(pkg):
    a = pkg.abi
    with pkg.Open(pkg.Config(ordinals=[0, 0], bytes=1 << 20, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        rc, d = p.diagnose_raw(a.OP_READ, 0, 1, 0)  # before the first run there is no pattern to compare with
        assert rc == a.ERR_STATE and (d.abi, d.op, d.issuer, d.target, d.reader) == (2, 1, 0, 1, 0)
        assert d.first_bad == U64_MAX and d.bad_words == 0
        assert p.Run().verdict
        for args, code in [((3, 0, 1, 0), a.ERR_ARG),   # bad op
                           ((0, 0, 1, 0), a.ERR_ARG),
                           ((a.OP_READ, 2, 1, 0), a.ERR_ARG),   # issuer >= n
                           ((a.OP_READ, 0, 5, 0), a.ERR_ARG),   # target >= n
                           ((a.OP_READ, 0, 1, 2), a.ERR_ARG),   # reader >= n
                           ((a.OP_WRITE, 0, 0, 0), a.ERR_ARG)]:  # no loop-back slot at n = 2
            rc, d = p.diagnose_raw(*args)
            assert rc == code, args
            assert (d.abi, d.op, d.issuer, d.target, d.reader) == (2, *args)
        with pytest.raises(pkg.ProbeError):
            p.Diagnose("read", 0, 9)
        assert p.Diagnose("read", 0, 1).bad_words == 0 and p.Diagnose("write", 1, 0).bad_words == 0
        assert p.Run().verdict


@pytest.mark.skipif(NGPU < 2, reason="needs >= 2 GPUs")
def test_fabric_reader_and_resting_reader_agree(pkg):
    with pkg.Open(pkg.Config(ordinals=[0, 1], bytes=1 << 20)) as p:
        assert p.Run().verdict
        p.Corrupt(1, 64, 1 << 5)  # rank 1's slice 0: what rank 0 reads over NVLink
        r = p.Run()
        assert r.reach_read[0][1] == 0
        over, rest = p.Diagnose("read", 0, 1, reader=0), p.Diagnose("read", 0, 1, reader=1)
        assert over.bad_words == 1 and over.first_bad == 64 and over.bit_flips[5] == 1
        assert report(over) == report(rest)
