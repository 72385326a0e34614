"""Probe memory word for word: after a run every cell's region holds exactly the pattern the spec names, in every path,
size, mode, schedule and process layout; cdprobe_diagnose's whole report equals a plain CPU reference
(tests/word_ref.py); and the (S, X) checksum's documented blind spots, on the device.

The probe's verdict and the parity suite compare checksums, and (S, X) cannot see a word stored at the wrong offset
inside its 16 KiB granule, nor a swap of two granules with the same fold6 class.  cdprobe_diagnose compares every
word, so a sweep of it over every cell is what catches a placement bug in a write path or in the source fill."""
import json
import random
import subprocess
import sys
import textwrap
import uuid

import numpy as np
import pytest

import word_ref as ref
from conftest import ROOT, gpu_count

pytestmark = pytest.mark.gpu

NGPU = gpu_count()
SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
LOCAL_DIAG = 0x04
G = ref.GRANULE_WORDS
VMM = 2 << 20       # allocation granule; Ctrl fills the first one, the source buffer starts at the second
OP = {"read": 1, "write": 2}


# ---- where a cell lives, restated from the plan ----------------------------------------------------------------
def region_offset(oracle, n, nbytes, mode, diag, op, i, j):
    """Byte offset of cell (op, i, j) in rank j's allocation: landing slot slot_of(i, j) (the diagonal at n - 1) for
    writes, the source slice of the same index for reads (slice 0 in full mode)."""
    pl = oracle.plan(n, nbytes, mode, diag)
    slot = n - 1 if i == j else oracle.lib().cdoracle_slot(i, j)
    if op == "read":
        return VMM + (0 if mode == 2 else slot) * pl.bytes_per_pair
    return VMM + -(-pl.src_bytes // VMM) * VMM + slot * pl.bytes_per_pair


def cells(n, diag):
    return [(i, j) for i in range(n) for j in range(n) if i != j or diag]


def report(d):
    """Everything a diagnosis says about the bytes (not who read them, nor how long it took)."""
    raw = d.raw
    return ({f: getattr(raw, f) for f, _ in raw._fields_ if f not in ("reader", "ms", "kind_count", "bit_flips", "sample")},
            list(raw.kind_count), list(raw.bit_flips), d.samples)


def sweep(p, oracle, r, nbytes, mode, where, diag=None, ops=3, issuer_reads=True):
    """Diagnose every cell of the plan for both ops, at rest (reader = target) and, when `issuer_reads`, again through
    the issuer's mapping, which must give the same report.  A write cell of a run without write jobs holds the zeros
    of open."""
    n = r.n
    diag = n == 1 if diag is None else diag
    W = r.bytes_per_pair // 8
    for op in ("read", "write"):
        for i, j in cells(n, diag):
            ctx = f"{where}: {op} cell {i} -> {j}"
            d = p.Diagnose(op, i, j, reader=j)
            assert d.bytes == r.bytes_per_pair and d.run_seq == r.run_seq, ctx
            assert d.region_offset == region_offset(oracle, n, nbytes, mode, diag, op, i, j), ctx
            if op == "write" and not ops & 2:
                assert d.bad_words == d.zero_words == W and d.kinds["zero"] == W, ctx
            else:
                assert d.bad_words == 0, (ctx, d.bad_words, d.kinds, d.first_bad, d.samples[:4])
            if issuer_reads and i != j:
                assert report(p.Diagnose(op, i, j, reader=i)) == report(d), ctx


# ---- a. every region holds the pattern, word for word ---------------------------------------------------------
@pytest.mark.parametrize("nbytes", [128, 8192, 8192 + 128, 16384 * 3 + 640, 1 << 20, (1 << 23) + 128 * 77])
def test_loopback_regions_every_path_and_tail(pkg, oracle, nbytes):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes)) as p:
        for path in (0, 1, 2):
            p.SetOption(pkg.abi.OPT_PATH, path)
            r = p.Run()
            assert r.verdict
            sweep(p, oracle, r, nbytes, 1, f"path {path}, {nbytes} bytes")


@pytest.mark.parametrize("ops", [1, 2, 3])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_loopback_regions_every_mode_and_op(pkg, oracle, mode, ops):
    nbytes = 4 << 20
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, mode=mode, ops=ops)) as p:
        r = p.Run()
        sweep(p, oracle, r, nbytes, mode, f"mode {mode}, ops {ops}", ops=ops)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("n", [2, 3, 4, 5, 8])
def test_same_device_regions_every_mode_and_path(pkg, oracle, n, mode):
    """Two runs per path: a slot the second run failed to rewrite would hold the first run's pattern (STALE)."""
    nbytes = 2 << 20
    cfg = pkg.Config(ordinals=[0] * n, bytes=nbytes, mode=mode, flags=SAME, ctas=8, timeout_ms=20000)
    with pkg.Open(cfg) as p:
        for path in (0, 1, 2):
            p.SetOption(pkg.abi.OPT_PATH, path)
            for run in (1, 2):
                r = p.Run()
                assert r.reach == [[1] * n for _ in range(n)] and not r.aborted
                sweep(p, oracle, r, nbytes, mode, f"n {n}, mode {mode}, path {path}, run {run}")


VARIANTS = [("unidirectional", 0x80, None), ("serial-verify", 0x100, None), ("overlap-verify", 0x20, 3),
            ("local-diag", LOCAL_DIAG, None)]


@pytest.mark.parametrize("flags,verify_ctas", [v[1:] for v in VARIANTS], ids=[v[0] for v in VARIANTS])
def test_same_device_regions_every_schedule_variant(pkg, oracle, flags, verify_ctas):
    n, nbytes = 4, 2 << 20
    diag = bool(flags & LOCAL_DIAG)
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME | flags, ctas=8, timeout_ms=20000)) as p:
        if verify_ctas:
            p.SetOption(pkg.abi.OPT_VERIFY_CTAS, verify_ctas)
        for path in (0, 1, 2):
            p.SetOption(pkg.abi.OPT_PATH, path)
            for run in (1, 2):
                r = p.Run()
                assert r.reach == [[1] * n for _ in range(n)] and not r.aborted
                sweep(p, oracle, r, nbytes, 1, f"flags {flags:#x}, path {path}, run {run}", diag=diag)


def raw_dict(raw):
    out = {f: getattr(raw, f) for f, _ in raw._fields_ if f not in ("ms", "reader", "kind_count", "bit_flips", "sample")}
    out["kind_count"] = list(raw.kind_count)
    out["bit_flips"] = list(raw.bit_flips)
    out["sample"] = [{f: getattr(s, f) for f, _ in s._fields_} for s in raw.sample]
    return out


def want_dict(spec, observed, op, issuer, run_seq, offset):
    """The whole cdprobe_diag_t the reference predicts, minus `ms` and `reader`."""
    rep = ref.expected_report(spec, observed)
    zero = {"offset": 0, "expected": 0, "observed": 0, "word": 0, "run_seq": 0, "kind": 0, "rank": 0}
    rep["sample"] = rep["sample"] + [zero] * (ref.SAMPLES - len(rep["sample"]))
    rep.update(abi=2, op=OP[op], issuer=issuer, target=spec.target, run_seq=run_seq, region_offset=offset,
               bytes=spec.n_words * 8)
    return rep


def assert_report(d, want, ctx=""):
    got = raw_dict(d.raw)
    assert set(got) == set(want)
    for k in want:
        assert got[k] == want[k], (ctx, k)


def test_solo_rank_regions(pkg, oracle):
    """Rank 0 runs alone: its slot in rank 1 holds this run's pattern although nobody verified it; rank 1 did not run,
    so its slot in rank 0 holds the previous run's pattern, every word STALE from that run."""
    n, nbytes = 2, 8 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        r1 = p.Run()
        assert r1.reach == [[1] * n for _ in range(n)]
        p.SetOption(pkg.abi.OPT_SOLO_RANK, 1)
        r2 = p.Run()
        assert r2.reach_write[0][1] == 0 and r2.reach_read[0][1] == 1
        W = r2.bytes_per_pair // 8
        d = p.Diagnose("write", 0, 1, reader=1)
        assert d.bad_words == 0 and d.run_seq == r2.run_seq
        assert p.Diagnose("read", 0, 1, reader=1).bad_words == 0
        d = p.Diagnose("write", 1, 0, reader=0)
        assert d.kinds["stale"] == d.bad_words == W and d.samples[0]["run_seq"] == r1.run_seq
        spec = ref.write_spec(SEED, n, 1, 0, r2.run_seq, W)
        old = ref.write_words(ref.write_salt(SEED, 1, 0, r1.run_seq), 0, W)
        assert_report(d, want_dict(spec, old, "write", 1, r2.run_seq,
                                   region_offset(oracle, n, nbytes, 1, False, "write", 1, 0)))
        p.SetOption(pkg.abi.OPT_SOLO_RANK, 0)
        r3 = p.Run()
        assert r3.reach == [[1] * n for _ in range(n)]
        sweep(p, oracle, r3, nbytes, 1, "after solo")


def test_copy_engine_scribble_then_one_run_leaves_every_slot_clean(pkg, oracle):
    n, nbytes = 2, 2 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        r1 = p.Run()
        p.CeCopy([(0, 1), (1, 0)], push=True, reps=2)  # each rank's source -> the other's landing slot
        W = r1.bytes_per_pair // 8
        for i, j in ((0, 1), (1, 0)):
            d = p.Diagnose("write", i, j, reader=j)
            spec = ref.write_spec(SEED, n, i, j, r1.run_seq, W)
            assert_report(d, want_dict(spec, ref.src_words(SEED, i, 0, W), "write", i, r1.run_seq,
                                       region_offset(oracle, n, nbytes, 1, False, "write", i, j)), (i, j))
        r2 = p.Run()
        assert r2.reach == [[1] * n for _ in range(n)]
        sweep(p, oracle, r2, nbytes, 1, "after ce_copy")


@pytest.mark.skipif(NGPU < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("mode", [1, 2], ids=["sliced", "full"])
def test_real_peers_regions_read_from_both_sides(pkg, oracle, mode):
    n, nbytes = min(NGPU, 8), 16 << 20
    with pkg.Open(pkg.Config(ordinals=list(range(n)), bytes=nbytes, mode=mode, timeout_ms=20000)) as p:
        for path in (0, 1, 2):
            p.SetOption(pkg.abi.OPT_PATH, path)
            r = p.Run()
            assert r.reach == [[1] * n for _ in range(n)] and not r.aborted
            sweep(p, oracle, r, nbytes, mode, f"{n} GPUs, mode {mode}, path {path}")


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world, ordinal, nbytes, flags = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]), int(sys.argv[6])
    cfg = m.Config(ordinals=[ordinal], bytes=nbytes, world_size=world, rank=rank, session=session, flags=flags,
                   ctas=int(sys.argv[7]), timeout_ms=30000)
    with m.Open(cfg) as p:
        info = p.Info()
        out = []
        for _ in range(2):
            r = p.Run(gather=True)
            diags = []
            for op in ("read", "write"):
                for i in range(world):
                    for j in range(world):
                        if i != j and rank in (i, j):  # this rank's own memory, and the peer's through the imported fd
                            d = p.Diagnose(op, i, j, reader=rank)
                            diags.append({"op": op, "i": i, "j": j, "bad": d.bad_words, "kinds": d.kinds,
                                          "bytes": d.bytes, "run_seq": d.run_seq, "offset": d.region_offset})
            out.append({"reach": r.reach, "run_seq": r.run_seq, "bpp": r.bytes_per_pair, "verdict": r.verdict,
                        "handle_type": info.handle_type, "diags": diags})
    print("RESULT " + json.dumps(out))
    """
) % ROOT


def run_world(world, ordinals, nbytes, flags, ctas):
    session = f"w-{uuid.uuid4().hex[:12]}"
    procs = [subprocess.Popen([sys.executable, "-c", CHILD, session, str(r), str(world), str(ordinals[r]), str(nbytes),
                               str(flags), str(ctas)], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
             for r in range(world)]
    outs = []
    for p in procs:
        so, se = p.communicate(timeout=300)
        assert p.returncode == 0, se[-2000:]
        outs.append(json.loads([l for l in so.splitlines() if l.startswith("RESULT ")][-1][7:]))
    return outs


def test_two_processes_regions_through_imported_handles(pkg, oracle):
    world, nbytes = 2, 1 << 20
    outs = run_world(world, [0, 0], nbytes, 0x40, 8)
    for rank, per_rank in enumerate(outs):
        for r in per_rank:
            assert r["handle_type"] == 1 and r["reach"] == [[1] * world for _ in range(world)]
            assert len(r["diags"]) == 4
            for d in r["diags"]:
                ctx = (rank, d)
                assert d["bad"] == 0 and d["bytes"] == r["bpp"] and d["run_seq"] == r["run_seq"], ctx
                assert d["offset"] == region_offset(oracle, world, nbytes, 1, False, d["op"], d["i"], d["j"]), ctx


# ---- b. the whole report against the CPU reference -----------------------------------------------------------------
def plant(p, local, src_base, spec, rng, idx, kinds, other_ranks=()):
    """xor a fault into word k of the region (source bytes from src_base) for every k in idx, cycling through `kinds`;
    returns the (k, mask) pairs."""
    exp = spec.expected()
    faults = []
    for m, k in enumerate(idx):
        kind = kinds[m % len(kinds)]
        e = int(exp[k])
        if kind == "flip":
            mask = rng.choice((1 << rng.randrange(64), 1 << 63, rng.getrandbits(64) | 1 << 63, rng.getrandbits(64) or 1))
        elif kind == "zero":
            mask = e
        elif kind == "displaced":
            kp = rng.randrange(spec.src_words)
            kp = kp if kp != spec.first_word + k else (kp + 1) % spec.src_words
            mask = e ^ int(ref.src_words(SEED, spec.target, kp, 1)[0])
        else:  # foreign
            mask = e ^ int(ref.src_words(SEED, rng.choice(other_ranks), rng.randrange(spec.src_words), 1)[0])
        p.Corrupt(local, src_base + 8 * k, mask)
        faults.append((k, mask))
    return faults


def observed(spec, faults):
    w = spec.expected().copy()
    for k, mask in faults:
        w[k] ^= np.uint64(mask)
    return w


def undo(p, local, src_base, faults):
    for k, mask in faults:
        p.Corrupt(local, src_base + 8 * k, mask)


def loopback_read_spec(r):
    W = r.bytes_per_pair // 8
    return ref.read_spec(SEED, 1, 0, 0, W, W)


@pytest.mark.parametrize("nbytes,n_faults", [(128, 6), (16384 * 3 + 640, 12), (1 << 20, 40)])
def test_diagnosis_equals_the_reference(pkg, oracle, nbytes, n_faults):
    rng = random.Random(nbytes)
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes)) as p:
        r = p.Run()
        assert r.verdict and p.Diagnose("read", 0, 0).bad_words == 0
        spec = loopback_read_spec(r)
        idx = sorted(set(rng.sample(range(spec.n_words), n_faults - 1)) | {spec.n_words - 1})  # the last word too
        faults = plant(p, 0, 0, spec, rng, idx, ["flip", "flip", "zero", "displaced"])
        d = p.Diagnose("read", 0, 0)
        assert_report(d, want_dict(spec, observed(spec, faults), "read", 0, r.run_seq, VMM), nbytes)
        assert d.kinds["flip"] and d.kinds["displaced"] and d.kinds["zero"]
        undo(p, 0, 0, faults)
        assert p.Diagnose("read", 0, 0).bad_words == 0 and p.Run().verdict


def test_foreign_words_on_a_same_device_slice(pkg, oracle):
    """N = 3 on one device: the slice rank 2 reads from rank 0 (slice 1) holds words of ranks 1 and 2 and of rank 0's
    other slice; the issuer's and the owner's reports both equal the reference."""
    n, nbytes = 3, 1 << 20
    rng = random.Random(3)
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        r = p.Run()
        assert r.reach == [[1] * n for _ in range(n)]
        W = r.bytes_per_pair // 8
        spec = ref.read_spec(SEED, n, 0, W, W, 2 * W)
        idx = sorted(rng.sample(range(W), 24))
        faults = plant(p, 0, 8 * W, spec, rng, idx, ["foreign", "foreign", "displaced", "zero", "flip"], (1, 2))
        want = want_dict(spec, observed(spec, faults), "read", 2, r.run_seq,
                         region_offset(oracle, n, nbytes, 1, False, "read", 2, 0))
        assert want["kind_count"][ref.FOREIGN] > 0
        for reader in (2, 0):
            assert_report(p.Diagnose("read", 2, 0, reader=reader), want, reader)
        undo(p, 0, 8 * W, faults)
        assert p.Diagnose("read", 2, 0).bad_words == 0 and p.Run().reach == [[1] * n for _ in range(n)]


def test_samples_need_many_chunks_of_the_granule_scan(pkg, oracle):
    """128 MiB (8192 granules), one fault every 300 granules from granule 1000: the 16 samples span 4500 granules,
    so the sample pass scans many 256-granule chunks from a start that is not granule 0."""
    nbytes = 128 << 20
    rng = random.Random(128)
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes)) as p:
        r = p.Run()
        assert r.verdict and p.Diagnose("read", 0, 0).bad_words == 0
        spec = loopback_read_spec(r)
        idx = [g * G + rng.randrange(G) for g in range(1000, 6701, 300)]
        assert len(idx) == 20
        faults = plant(p, 0, 0, spec, rng, idx, ["flip", "zero", "displaced"])
        d = p.Diagnose("read", 0, 0)
        assert_report(d, want_dict(spec, observed(spec, faults), "read", 0, r.run_seq, VMM))
        assert [s["offset"] for s in d.samples] == [8 * k for k in idx[:16]]
        undo(p, 0, 0, faults)
        assert p.Diagnose("read", 0, 0).bad_words == 0 and p.Run().verdict


def test_a_granule_with_every_word_flipped(pkg, oracle):
    rng = random.Random(2048)
    with pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 20)) as p:
        r = p.Run()
        assert r.verdict and p.Diagnose("read", 0, 0).bad_words == 0
        spec = loopback_read_spec(r)
        faults = plant(p, 0, 0, spec, rng, range(5 * G, 6 * G), ["flip"])
        d = p.Diagnose("read", 0, 0)
        assert d.bad_words == G and d.bad_granules == 1 and d.kinds["flip"] == G
        assert_report(d, want_dict(spec, observed(spec, faults), "read", 0, r.run_seq, VMM))
        undo(p, 0, 0, faults)
        assert p.Diagnose("read", 0, 0).bad_words == 0 and p.Run().verdict


def test_write_cell_that_missed_a_run_equals_the_reference(pkg, oracle):
    n, nbytes = 2, 1 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        r1 = p.Run()
        assert r1.reach == [[1] * n for _ in range(n)]
        p.UnmapPeer(0, 1)
        r2 = p.Run()
        assert r2.reach_write[0][1] == 0
        W = r2.bytes_per_pair // 8
        d = p.Diagnose("write", 0, 1, reader=1)
        assert d.kinds["stale"] == d.bad_words == W
        spec = ref.write_spec(SEED, n, 0, 1, r2.run_seq, W)
        old = ref.write_words(ref.write_salt(SEED, 0, 1, r1.run_seq), 0, W)
        assert_report(d, want_dict(spec, old, "write", 0, r2.run_seq,
                                   region_offset(oracle, n, nbytes, 1, False, "write", 0, 1)))


# ---- c. what (S, X) cannot see, on the device ------------------------------------------------------------------
def swap(p, words, a, b, n):
    """Swap words [a, a + n) and [b, b + n) of rank 0's source: xor a ^ b into both places."""
    for k in range(n):
        m = int(words[a + k] ^ words[b + k])
        p.Corrupt(0, 8 * (a + k), m)
        p.Corrupt(0, 8 * (b + k), m)


def test_checksum_blind_spot_on_the_device(pkg, oracle):
    """The documented limitation of (S, X), asserted so that a change to the checksum has to update it on purpose:
    two words swapped inside a granule, or granules 1 and 64 (fold6 1 both) swapped, pass the probe with the clean
    checksum, and only cdprobe_diagnose sees them.  Granules 0 and 1 (fold6 0 and 1) change X."""
    nbytes = 2 << 20
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes)) as p:
        r = p.Run()
        W = r.bytes_per_pair // 8
        clean = oracle.src_checksum(SEED, 0, 0, W)
        assert W == 128 * G and r.verdict and (r.sum_read[0][0], r.xor_read[0][0]) == clean
        spec = loopback_read_spec(r)
        words = spec.expected()
        for a, b, n in ((3 * G + 5, 3 * G + 2000, 1), (1 * G, 64 * G, G)):
            swap(p, words, a, b, n)
            r = p.Run()
            assert r.reach_read[0][0] == 1 and r.verdict, (a, b)
            assert (r.sum_read[0][0], r.xor_read[0][0]) == clean, (a, b)
            d = p.Diagnose("read", 0, 0)
            assert d.bad_words == 2 * n and d.kinds["displaced"] == 2 * n, (a, b)
            assert [(s["offset"], s["word"]) for s in d.samples] == \
                [(8 * (a + k), b + k) for k in range(min(n, 16))] + ([(8 * b, a)] if n == 1 else [])
            sw = words.copy()
            sw[a:a + n], sw[b:b + n] = words[b:b + n], words[a:a + n]
            assert_report(d, want_dict(spec, sw, "read", 0, r.run_seq, VMM), (a, b))
            swap(p, words, a, b, n)
        swap(p, words, 0, G, G)
        r = p.Run()
        assert r.reach_read[0][0] == 0 and not r.verdict
        assert r.sum_read[0][0] == clean[0] and r.xor_read[0][0] != clean[1]
        swap(p, words, 0, G, G)
        r = p.Run()
        assert r.verdict and (r.sum_read[0][0], r.xor_read[0][0]) == clean
        assert p.Diagnose("read", 0, 0).bad_words == 0
