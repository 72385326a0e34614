"""The probe, its diagnosis and every size-bound measurement word for word past 2 GiB and 4 GiB per pair, up to the
plan's ceiling of 16 GiB: the byte offsets where a 32-bit offset, unit count or ctypes argument would wrap.

Every expected value comes from a reference that streams (tests/large_ref.py), the oracle, or latency_ref's pure-Python
chase, never from a dense region in host memory.  Each test opens its own handle and first checks that the device has
the memory the plan and the measurement's areas need, with 4 GiB to spare, by arithmetic; on a busy card it skips and
names both numbers rather than allocate and hope.

A. N = 1, bytes_per_pair = 4 GiB + 8 KiB + 128: the last 8 KiB unit is 128 B, the last 16 KiB granule is partial, and
   the whole landing slot lies past 2^32 in the allocation.
B. Two ranks on one device, full mode with LOCAL_DIAG, bytes_per_pair = 2 GiB + 8 KiB + 128: in each rank's allocation
   landing slot 0 runs across 2^32 and slot 1 lies past it; the exchange area's blocks end past 2^32.
C. N = 1 at the ceiling, bytes_per_pair = 16 GiB: the last word index is 2^31 - 1."""
import functools

import pytest

import bwcurve_ref
import large_ref
import latency_ref
import word_ref as ref
from test_words_gpu import assert_report

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
GIB = 1 << 30
VMM = 2 << 20           # allocation granule; the control block fills the first one
HEADROOM = 4 * GIB      # free memory a test leaves to everything else on the device
SPARE = 64 << 20        # per rank: scratch records, granule tables and a diagnosis of a whole region
HBM_GBPS = 3350.0       # H100 SXM data sheet
SAME = 0x40 | 0x10      # ALLOW_SAME_DEVICE | NO_COOPERATIVE
LOCAL_DIAG = 0x04
MODE_SLICED, MODE_FULL = 1, 2
OP_READ, OP_WRITE = 1, 2
ERR_INTEGRITY = -10
U64_MAX = (1 << 64) - 1
G = ref.GRANULE_WORDS
UNIT_WORDS = 1024       # an 8 KiB unit
SAME_DEVICE_LINK_PEAK_GBPS = 1e-3  # ranks on one device: the verdict depends on the slots alone

A_BPP = (4 << 30) + 8192 + 128
B_BPP = (2 << 30) + 8192 + 128
C_BPP = 16 * GIB


def round_up(v, a):
    return -(-v // a) * a


# ---- the memory guard -----------------------------------------------------------------------------------------------
def alloc_bytes(pkg, n, nbytes, mode, flags):
    """One rank's probe allocation: the control granule, the source buffer and the landing slots, each rounded up to
    the VMM granule (plan.cc)."""
    pl = pkg.plan(n, nbytes, mode, flags)
    return VMM + round_up(pl.src_bytes, VMM) + round_up(pl.land_bytes, VMM)


def guard(pkg, n, nbytes, mode=MODE_SLICED, flags=0, extra=0):
    """Skip unless the device has the handle's need (n allocations, n x `extra` for a measurement's area or scratch,
    SPARE per rank) plus HEADROOM free."""
    import torch

    need = n * (alloc_bytes(pkg, n, nbytes, mode, flags) + extra + SPARE)
    free, _ = torch.cuda.mem_get_info(0)
    if free < need + HEADROOM:
        pytest.skip(f"needs {need} bytes plus {HEADROOM} spare on the device; {free} free")


def open_a(pkg):
    return pkg.Open(pkg.Config(ordinals=[0], bytes=A_BPP, timeout_ms=60000))


def open_b(pkg):
    return pkg.Open(pkg.Config(ordinals=[0, 0], bytes=B_BPP, mode=MODE_FULL, flags=SAME | LOCAL_DIAG, ctas=8,
                               timeout_ms=120000, link_peak_gbps=SAME_DEVICE_LINK_PEAK_GBPS))


# ---- references, each computed once per session ---------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def src_sums(rank, bpp):
    """(S, X) of every ladder prefix of rank's source words 0 .. bpp / 8 - 1."""
    return tuple(large_ref.prefix_sums(large_ref.src_fn(SEED, rank), bpp // 8, bwcurve_ref.ladder(bpp)))


@functools.lru_cache(maxsize=None)
def ar_sums(n, bpp, corrupt=None):
    return tuple(large_ref.allreduce_sums(SEED, n, bwcurve_ref.ladder(bpp), corrupt))


@functools.lru_cache(maxsize=None)
def oracle_src(oracle, rank, words):
    return oracle.src_checksum(SEED, rank, 0, words)


def region_offset(pkg, n, nbytes, mode, flags, op, i, j):
    """Byte offset of cell (op, i, j) in j's allocation: the source slice after the control granule, or the landing
    slot after the source buffer; the loop-back cell uses slot n - 1."""
    pl = pkg.plan(n, nbytes, mode, flags)
    slot = n - 1 if i == j else (i if i < j else i - 1)
    if op == "read":
        return VMM + (0 if mode == MODE_FULL else slot) * pl.bytes_per_pair
    return VMM + round_up(pl.src_bytes, VMM) + slot * pl.bytes_per_pair


def want_sparse(spec, faults, op, issuer, run_seq, offset):
    """The whole cdprobe_diag_t that large_ref.sparse_report predicts, minus `ms` and `reader`."""
    rep = large_ref.sparse_report(spec, faults)
    zero = {"offset": 0, "expected": 0, "observed": 0, "word": 0, "run_seq": 0, "kind": 0, "rank": 0}
    rep["sample"] = rep["sample"] + [zero] * (ref.SAMPLES - len(rep["sample"]))
    rep.update(abi=2, op=OP_READ if op == "read" else OP_WRITE, issuer=issuer, target=spec.target, run_seq=run_seq,
               region_offset=offset, bytes=spec.n_words * 8)
    return rep


def expected_words(spec, idx):
    return [int(spec.expected(k, 1)[0]) for k in idx]


def read_faults(spec, idx):
    """(k, observed) for each k of idx, cycling FLIP, ZERO and DISPLACED (a word from the far end of the buffer)."""
    out = []
    for m, (k, e) in enumerate(zip(idx, expected_words(spec, idx))):
        kind = m % 3
        if kind == 0:
            v = e ^ (1 << (k % 63)) ^ (1 << 63)
        elif kind == 1:
            v = 0
        else:
            v = int(ref.src_words(SEED, spec.target, spec.src_words - 1 - m, 1)[0])
        out.append((k, v))
    return out


def write_faults(spec, idx):
    """(k, observed) for each k of idx, cycling FLIP, ZERO, DISPLACED and STALE; spec.run_seq must be at least 2."""
    salt = ref.write_salt(SEED, spec.issuer, spec.target, spec.run_seq)
    old = ref.write_salt(SEED, spec.issuer, spec.target, spec.run_seq - 1)
    out = []
    for m, (k, e) in enumerate(zip(idx, expected_words(spec, idx))):
        kind = m % 4
        if kind == 0:
            v = e ^ (0xF0F0 << (k % 48))
        elif kind == 1:
            v = 0
        elif kind == 2:
            v = int(ref.write_words(salt, (k + 1 + m) % spec.n_words, 1)[0])
        else:
            v = int(ref.write_words(old, k, 1)[0])
        out.append((k, v))
    return out


def masks(spec, faults):
    """The xor masks that turn the pattern into the faults' observed words."""
    return [(k, e ^ v) for (k, v), e in zip(faults, expected_words(spec, [k for k, _ in faults]))]


def far_words(W):
    """Word indices at byte 2^31 and 2^32 and either side, inside the last (128-byte) unit, and the last word."""
    last_unit = W // UNIT_WORDS * UNIT_WORDS
    return sorted(k for k in {(1 << 28) - 1, 1 << 28, (1 << 29) - 1, 1 << 29, last_unit, last_unit + 7, W - 1} if k < W)


# ---- A. N = 1, 4 GiB + 8 KiB + 128 --------------------------------------------------------------------------------
def test_a_run_on_every_path(pkg, oracle):
    guard(pkg, 1, A_BPP)
    W = A_BPP // 8
    with open_a(pkg) as p:
        assert p.Info().bytes_per_pair == A_BPP
        for path in (0, 1, 2):
            p.SetOption(pkg.abi.OPT_PATH, path)
            r = p.Run()
            assert r.bytes_per_pair == A_BPP and r.verdict and r.reach == [[1]], path
            assert (r.sum_read[0][0], r.xor_read[0][0]) == oracle_src(oracle, 0, W), path
            assert (r.sum_write[0][0], r.xor_write[0][0]) == oracle.write_checksum(SEED, 0, 0, r.run_seq, W), path
            gbps = 3 * A_BPP / r.kernel_ms[0] / 1e6  # read + write + verify, bytes per ms -> GB/s
            assert gbps <= 1.1 * HBM_GBPS, (path, r.kernel_ms[0], gbps)


def test_a_diagnosis_locates_faults_past_2_31_and_2_32(pkg, oracle):
    guard(pkg, 1, A_BPP)
    W = A_BPP // 8
    idx = far_words(W)
    assert len(idx) == 7 and idx[-1] == W - 1
    with open_a(pkg) as p:
        r = p.Run()
        assert r.verdict
        for op in ("read", "write"):
            d = p.Diagnose(op, 0, 0)
            assert d.bad_words == 0 and d.bytes == A_BPP and d.run_seq == r.run_seq, op
            assert d.region_offset == region_offset(pkg, 1, A_BPP, MODE_SLICED, 0, op, 0, 0), op

        # at rest: the source buffer; only the read cell fails
        spec = ref.read_spec(SEED, 1, 0, 0, W, W)
        faults = read_faults(spec, idx)
        for k, m in masks(spec, faults):
            p.Corrupt(0, 8 * k, m)
        r = p.Run()
        assert (r.reach_read, r.reach_write, r.verdict, r.aborted) == ([[0]], [[1]], False, False)
        want = want_sparse(spec, faults, "read", 0, r.run_seq, region_offset(pkg, 1, A_BPP, MODE_SLICED, 0, "read", 0, 0))
        assert want["kind_count"][:3] == [3, 2, 2] and want["last_bad"] == A_BPP - 8
        assert_report(p.Diagnose("read", 0, 0), want, "read")
        assert p.Diagnose("write", 0, 0).bad_words == 0
        for k, m in masks(spec, faults):
            p.Corrupt(0, 8 * k, m)

        # in transit: the landing slot of the next run; only the write cell fails
        spec = ref.write_spec(SEED, 1, 0, 0, r.run_seq + 1, W)
        faults = write_faults(spec, idx)
        p.CorruptLanding(0, 0, masks(spec, faults))
        r = p.Run()
        assert r.run_seq == spec.run_seq
        assert (r.reach_read, r.reach_write, r.verdict, r.aborted) == ([[1]], [[0]], False, False)
        want = want_sparse(spec, faults, "write", 0, r.run_seq,
                           region_offset(pkg, 1, A_BPP, MODE_SLICED, 0, "write", 0, 0))
        assert want["kind_count"] == [2, 2, 2, 1, 0]
        assert_report(p.Diagnose("write", 0, 0), want, "write")
        assert p.Diagnose("read", 0, 0).bad_words == 0

        p.CorruptLanding(0, 0, [])
        r = p.Run()
        assert r.verdict
        assert (r.sum_read[0][0], r.xor_read[0][0]) == oracle_src(oracle, 0, W)
        assert p.Diagnose("read", 0, 0).bad_words == 0 and p.Diagnose("write", 0, 0).bad_words == 0


def test_a_latency_chase_reaches_past_2_32(pkg):
    """The chase's warm-up first loads a line past byte 2^32 at hop 60211 of this seed and region, so 2^16 hops."""
    guard(pkg, 1, A_BPP)
    hops, reps, lines = 1 << 16, 2, A_BPP // latency_ref.LINE_BYTES
    far = max(line for rep in range(reps + 1) for line, _ in latency_ref.chase(SEED, 0, 0, 0, lines, rep, hops))
    assert far * latency_ref.LINE_BYTES >= 1 << 32
    with open_a(pkg) as p:
        lat = p.Latency(hops=hops, reps=reps)
        assert (lat.hops, lat.reps, lat.region_bytes) == (hops, reps, A_BPP)
        assert lat.measured[0][0] and lat.status[0][0] == 0
        assert lat.digest[0][0] == latency_ref.digest(SEED, 0, 0, 0, lines, hops, reps)


def test_a_bwcurve_every_size_and_a_word_past_2_31_and_2_32(pkg):
    guard(pkg, 1, A_BPP)
    sizes = bwcurve_ref.ladder(A_BPP)
    want = list(src_sums(0, A_BPP))
    k4, k2 = sizes.index(4 * GIB), sizes.index(2 * GIB)
    with open_a(pkg) as p:
        for path in (0, 1, 2):
            p.SetOption(pkg.abi.OPT_PATH, path)
            bw = p.BwCurve(reps=2)
            assert bw.sizes == sizes and bw.path == path
            assert bw.status[0][0] == 0 and bw.bad_sizes[0][0] == 0, path
            assert list(zip(bw.sum[0][0], bw.xr[0][0])) == want, path
            assert 4 * GIB / bw.ns_min[0][0][k4] <= 1.1 * HBM_GBPS, (path, bw.ns_min[0][0][k4])
            ratio = bw.ns_median[0][0][-1] / bw.ns_median[0][0][k2]  # both far beyond the 50 MB L2
            assert 1.6 <= ratio <= 2.4, (path, ratio)
            for off, bits in (((1 << 32) + 8, 1 << (len(sizes) - 1)), ((1 << 31) + 8, 1 << k4 | 1 << (len(sizes) - 1))):
                p.Corrupt(0, off, 1 << 17)
                bw = p.BwCurve(reps=2)
                assert bw.status[0][0] == ERR_INTEGRITY and bw.bad_sizes[0][0] == bits, (path, off, bw.bad_sizes[0][0])
                for k, s in enumerate(sizes):
                    if s <= off:
                        assert (bw.sum[0][0][k], bw.xr[0][0][k]) == want[k], (path, off, s)
                p.Corrupt(0, off, 1 << 17)  # restore
            assert p.BwCurve(reps=1).bad_sizes[0][0] == 0


@pytest.mark.parametrize("op", [OP_READ, OP_WRITE], ids=["pull", "push"])
def test_a_memcpy_every_size_and_a_word_past_2_32(pkg, op):
    guard(pkg, 1, A_BPP, extra=round_up(A_BPP, VMM))  # the exchange area
    sizes = bwcurve_ref.ladder(A_BPP)
    want = list(src_sums(0, A_BPP))
    with open_a(pkg) as p:
        mc = p.Memcpy(op, reps=2)
        assert mc.sizes == sizes and mc.area_bytes == round_up(A_BPP, VMM)
        assert mc.status[0][0] == 0 and mc.bad_sizes[0][0] == 0
        assert mc.bad_words[0][0] == [0] * len(sizes) and mc.first_bad[0][0] == [U64_MAX] * len(sizes)
        assert list(zip(mc.sum[0][0], mc.xr[0][0])) == want
        off = (1 << 32) + 8 * 37
        p.Corrupt(0, off, 1 << 40)
        mc = p.Memcpy(op, reps=2)
        assert mc.status[0][0] == ERR_INTEGRITY and mc.bad_sizes[0][0] == 1 << (len(sizes) - 1)
        assert mc.first_bad[0][0][-1] == off and mc.bad_words[0][0][-1] > 0
        assert mc.first_bad[0][0][:-1] == [U64_MAX] * (len(sizes) - 1)
        assert list(zip(mc.sum[0][0], mc.xr[0][0]))[:-1] == want[:-1]
        p.Corrupt(0, off, 1 << 40)
        mc = p.Memcpy(op, reps=1)
        assert mc.bad_sizes[0][0] == 0 and list(zip(mc.sum[0][0], mc.xr[0][0])) == want


@pytest.mark.parametrize("op", [OP_READ, OP_WRITE], ids=["pull", "push"])
def test_a_ce_alltoall_every_size_and_a_word_past_2_32(pkg, op):
    """The copy-engine all-to-all's loop-back block at N = 1: every size clean; a source word past byte 2^32 fails
    only the last size, the one that covers it, with one bad word in the warm-up and one in the timed rep and its own
    byte offset as first_bad; restored, every size is clean again."""
    guard(pkg, 1, A_BPP, extra=round_up(A_BPP, VMM))  # the exchange area
    sizes = bwcurve_ref.ladder(A_BPP)
    want = list(src_sums(0, A_BPP))
    with open_a(pkg) as p:
        ca = p.CeAllToAll(op, reps=2)
        assert ca.sizes == sizes and ca.area_bytes == round_up(A_BPP, VMM) and ca.blocks == [1]
        assert ca.cell_measured == [[True]] and ca.cell_status == [[0]] and ca.bad_sizes == [[0]]
        assert ca.bad_words[0][0] == [0] * len(sizes) and ca.first_bad[0][0] == [U64_MAX] * len(sizes)
        assert list(zip(ca.sum[0][0], ca.xr[0][0])) == want
        off = (1 << 32) + 8 * 37
        assert sizes[-2] <= off < sizes[-1]
        p.Corrupt(0, off, 1 << 40)
        ca = p.CeAllToAll(op, reps=1)
        assert ca.cell_status[0][0] == ERR_INTEGRITY and ca.bad_sizes[0][0] == 1 << (len(sizes) - 1)
        assert ca.bad_words[0][0] == [0] * (len(sizes) - 1) + [2]
        assert ca.first_bad[0][0] == [U64_MAX] * (len(sizes) - 1) + [off]
        assert list(zip(ca.sum[0][0], ca.xr[0][0]))[:-1] == want[:-1]
        assert tuple(zip(ca.sum[0][0], ca.xr[0][0]))[-1] != want[-1]
        p.Corrupt(0, off, 1 << 40)
        ca = p.CeAllToAll(op, reps=1)
        assert ca.bad_sizes[0][0] == 0 and list(zip(ca.sum[0][0], ca.xr[0][0])) == want


def test_a_alltoall_row_clean_at_every_size(pkg):
    guard(pkg, 1, A_BPP, extra=round_up(A_BPP, VMM))
    sizes = bwcurve_ref.ladder(A_BPP)
    with open_a(pkg) as p:
        aa = p.AllToAll(reps=2)
        assert aa.sizes == sizes and aa.area_bytes == round_up(A_BPP, VMM)
        assert aa.measured == [True] and aa.status == [0] and aa.blocks == [1]
        assert aa.cell_measured == [[True]] and aa.cell_status == [[0]] and aa.bad_sizes == [[0]]
        assert aa.bad_words[0][0] == [0] * len(sizes) and aa.first_bad[0][0] == [U64_MAX] * len(sizes)


ALLREDUCES = {"oneshot": "AllReduce", "twoshot": "AllReduceTwoShot", "ring": "AllReduceRing", "push": "AllReducePush"}


@pytest.mark.parametrize("name", list(ALLREDUCES))
def test_a_allreduce_every_size_and_a_word_past_2_32(pkg, name):
    # the one-shot's output is in the scratch; the others' in an area of about the same size
    guard(pkg, 1, A_BPP, extra=round_up(A_BPP + 4 * (A_BPP // 8192 + 1), VMM))
    sizes = bwcurve_ref.ladder(A_BPP)
    want = ar_sums(1, A_BPP)
    reps = 2
    corrupt = (0, (1 << 29) + 3, 1 << 21)
    pred = ar_sums(1, A_BPP, corrupt)
    assert pred[-1].first_bad == 8 * corrupt[1] and all(w.bad_words == 0 for w in pred[:-1])
    with open_a(pkg) as p:
        call = getattr(p, ALLREDUCES[name])
        for path in (0, 1, 2):
            p.SetOption(pkg.abi.OPT_PATH, path)
            ar = call(reps=reps)
            assert ar.sizes == sizes and ar.status == [0] and ar.bad_sizes == [0], path
            assert [(s, x) for s, x in zip(ar.sum[0], ar.xr[0])] == [(w.sum, w.xr) for w in want], path
            assert ar.bad_words[0] == [0] * len(sizes) and ar.first_bad[0] == [U64_MAX] * len(sizes), path
            p.Corrupt(0, 8 * corrupt[1], corrupt[2])
            ar = call(reps=reps)
            assert ar.status == [ERR_INTEGRITY] and ar.bad_sizes == [1 << (len(sizes) - 1)], path
            assert [(s, x) for s, x in zip(ar.sum[0], ar.xr[0])] == [(w.sum, w.xr) for w in pred], path
            assert ar.bad_words[0] == [(reps + 1) * w.bad_words for w in pred], path  # every rep, the warm-up too
            assert ar.first_bad[0] == [w.first_bad for w in pred], path
            p.Corrupt(0, 8 * corrupt[1], corrupt[2])  # restore


def test_a_ll_ladder_stops_at_1_mib_and_runs_clean(pkg):
    guard(pkg, 1, A_BPP, extra=8 << 20)
    sizes = [s for s in bwcurve_ref.ladder(A_BPP) if s <= 1 << 20]
    assert sizes[-1] == 1 << 20
    with open_a(pkg) as p:
        ar = p.AllReduceLL(reps=2)
        assert ar.sizes == sizes and ar.path == pkg.abi.ALLREDUCE_PATH_LL
        assert ar.status == [0] and ar.bad_sizes == [0] and ar.bad_words[0] == [0] * len(sizes)
        want = large_ref.allreduce_sums(SEED, 1, sizes)
        assert [(s, x) for s, x in zip(ar.sum[0], ar.xr[0])] == [(w.sum, w.xr) for w in want]


# ---- B. two ranks on one device, 2 GiB + 8 KiB + 128, full mode with LOCAL_DIAG --------------------------------------
B_CELLS = [(i, j) for i in range(2) for j in range(2)]


def test_b_runs_and_diagnoses_across_2_32(pkg, oracle):
    n, W = 2, B_BPP // 8
    guard(pkg, n, B_BPP, MODE_FULL, LOCAL_DIAG)
    slot0 = region_offset(pkg, n, B_BPP, MODE_FULL, LOCAL_DIAG, "write", 0, 1)
    slot1 = region_offset(pkg, n, B_BPP, MODE_FULL, LOCAL_DIAG, "write", 1, 1)
    assert slot0 < 1 << 32 < slot0 + B_BPP == slot1
    with open_b(pkg) as p:
        assert p.Info().alloc_bytes == alloc_bytes(pkg, n, B_BPP, MODE_FULL, LOCAL_DIAG)
        for path in (0, 1, 2):
            p.SetOption(pkg.abi.OPT_PATH, path)
            r = p.Run()
            assert r.bytes_per_pair == B_BPP and r.reach == [[1, 1], [1, 1]] and r.verdict and not r.aborted, path
            for i, j in B_CELLS:
                assert (r.sum_read[i][j], r.xor_read[i][j]) == oracle_src(oracle, j, W), (path, i, j)
                assert (r.sum_write[i][j], r.xor_write[i][j]) == \
                    oracle.write_checksum(SEED, i, j, r.run_seq, W), (path, i, j)
        for op in ("read", "write"):
            for i, j in B_CELLS:
                d = p.Diagnose(op, i, j, reader=j)
                assert d.bad_words == 0 and d.bytes == B_BPP and d.run_seq == r.run_seq, (op, i, j)
                assert d.region_offset == region_offset(pkg, n, B_BPP, MODE_FULL, LOCAL_DIAG, op, i, j), (op, i, j)
                assert d.raw.first_bad == U64_MAX
                d2 = p.Diagnose(op, i, j, reader=i)
                d.raw.ms = d2.raw.ms = 0.0
                d.raw.reader = d2.raw.reader = 0
                assert bytes(d.raw) == bytes(d2.raw), (op, i, j)

        # rank 0's slot in rank 1, on the two words either side of byte 2^32 of rank 1's allocation
        k = ((1 << 32) - slot0) // 8
        spec = ref.write_spec(SEED, n, 0, 1, r.run_seq + 1, W)
        faults = [(k - 1, 0), (k, int(spec.expected(k, 1)[0]) ^ (1 << 63))]
        p.CorruptLanding(0, 1, masks(spec, faults))
        r = p.Run()
        assert r.reach_write == [[1, 0], [1, 1]] and r.reach_read == [[1, 1], [1, 1]] and not r.verdict
        assert (r.sum_write[0][1], r.xor_write[0][1]) == oracle.write_checksum(SEED, 0, 1, r.run_seq, W)
        want = want_sparse(spec, faults, "write", 0, r.run_seq, slot0)
        assert want["first_bad"] == (1 << 32) - 8 - slot0 and want["bad_granules"] == 2 - (k % G != 0)
        for reader in (1, 0):
            assert_report(p.Diagnose("write", 0, 1, reader=reader), want, reader)
        p.CorruptLanding(0, 1, [])
        r = p.Run()
        assert r.reach == [[1, 1], [1, 1]] and r.verdict
        assert p.Diagnose("write", 0, 1, reader=1).bad_words == 0


def test_b_bwcurve_memcpy_and_alltoall_every_cell(pkg):
    n = 2
    guard(pkg, n, B_BPP, MODE_FULL, LOCAL_DIAG, extra=round_up(n * B_BPP, VMM))  # the exchange area
    sizes = bwcurve_ref.ladder(B_BPP)
    with open_b(pkg) as p:
        bw = p.BwCurve(reps=2)
        assert bw.sizes == sizes
        for i, j in B_CELLS:  # full mode: every issuer reads the target's slice 0
            assert bw.measured[i][j] and bw.status[i][j] == 0 and bw.bad_sizes[i][j] == 0, (i, j)
            assert list(zip(bw.sum[i][j], bw.xr[i][j])) == list(src_sums(j, B_BPP)), (i, j)
        for op in (OP_READ, OP_WRITE):
            mc = p.Memcpy(op, reps=2)
            assert mc.sizes == sizes and mc.area_bytes == round_up(n * B_BPP, VMM)
            for g, j in B_CELLS:
                owner = g if op == OP_WRITE else j
                assert mc.measured[g][j] and mc.status[g][j] == 0 and mc.bad_sizes[g][j] == 0, (op, g, j)
                assert mc.bad_words[g][j] == [0] * len(sizes), (op, g, j)
                assert list(zip(mc.sum[g][j], mc.xr[g][j])) == list(src_sums(owner, B_BPP)), (op, g, j)
        aa = p.AllToAll(reps=2)
        assert aa.sizes == sizes and aa.status == [0, 0] and aa.blocks == [2, 2]
        for s, d in B_CELLS:
            assert aa.cell_measured[s][d] and aa.cell_status[s][d] == 0 and aa.bad_sizes[s][d] == 0, (s, d)
            assert aa.bad_words[s][d] == [0] * len(sizes) and aa.first_bad[s][d] == [U64_MAX] * len(sizes)


def test_b_loopback_slice_and_slot_1_lie_past_2_32(pkg):
    """Two ranks, sliced, LOCAL_DIAG, A's 4 GiB + 8 KiB + 128 per pair: the loop-back cells use source slice 1 and
    landing slot 1, whose offsets slot x bytes_per_pair pass 2^32 themselves, and every region but slice 0 lies past
    byte 2^32 of its rank's allocation."""
    n = 2
    guard(pkg, n, A_BPP, MODE_SLICED, LOCAL_DIAG)
    with pkg.Open(pkg.Config(ordinals=[0, 0], bytes=A_BPP, flags=SAME | LOCAL_DIAG, ctas=8, timeout_ms=120000,
                             link_peak_gbps=SAME_DEVICE_LINK_PEAK_GBPS)) as p:
        r = p.Run()
        assert r.bytes_per_pair == A_BPP and r.reach == [[1, 1], [1, 1]] and r.verdict and not r.aborted
        for op in ("read", "write"):
            for i, j in B_CELLS:
                off = region_offset(pkg, n, A_BPP, MODE_SLICED, LOCAL_DIAG, op, i, j)
                assert off > 1 << 32 or (op, i != j) == ("read", True), (op, i, j)  # only slice 0 lies below
                d = p.Diagnose(op, i, j, reader=j)
                assert d.region_offset == off and d.bytes == A_BPP and d.run_seq == r.run_seq, (op, i, j)
                assert d.bad_words == 0, (op, i, j, d.first_bad)


@pytest.mark.parametrize("op", [OP_READ, OP_WRITE], ids=["pull", "push"])
def test_b_memcpy_block_1_starts_past_2_32(pkg, op):
    """Two ranks, sliced, A's 4 GiB + 8 KiB + 128 per pair: block 1 of each exchange area, where rank 1's slice lands,
    starts past byte 2^32 of the area."""
    n = 2
    guard(pkg, n, A_BPP, extra=round_up(n * A_BPP, VMM))
    sizes = bwcurve_ref.ladder(A_BPP)
    with pkg.Open(pkg.Config(ordinals=[0, 0], bytes=A_BPP, flags=SAME, ctas=8, timeout_ms=120000,
                             link_peak_gbps=SAME_DEVICE_LINK_PEAK_GBPS)) as p:
        mc = p.Memcpy(op, reps=1)
        assert mc.sizes == sizes and mc.area_bytes == round_up(n * A_BPP, VMM)
        for g, j in ((0, 1), (1, 0)):
            owner = g if op == OP_WRITE else j
            assert mc.measured[g][j] and mc.status[g][j] == 0 and mc.bad_sizes[g][j] == 0, (g, j)
            assert mc.bad_words[g][j] == [0] * len(sizes), (g, j)
            assert list(zip(mc.sum[g][j], mc.xr[g][j])) == list(src_sums(owner, A_BPP)), (g, j)


def test_b_oneshot_allreduce_every_size(pkg):
    n = 2
    guard(pkg, n, B_BPP, MODE_FULL, LOCAL_DIAG, extra=round_up(B_BPP, VMM))  # each rank's output in its scratch
    sizes = bwcurve_ref.ladder(B_BPP)
    want = [(w.sum, w.xr) for w in ar_sums(n, B_BPP)]
    with open_b(pkg) as p:
        ar = p.AllReduce(reps=2)
        assert ar.sizes == sizes and ar.status == [0, 0] and ar.bad_sizes == [0, 0]
        for r in range(n):
            assert list(zip(ar.sum[r], ar.xr[r])) == want, r
            assert ar.bad_words[r] == [0] * len(sizes) and ar.first_bad[r] == [U64_MAX] * len(sizes), r


# ---- C. the plan's ceiling: N = 1, 16 GiB per pair ----------------------------------------------------------------
def test_c_the_ceiling_end_to_end(pkg, oracle):
    guard(pkg, 1, C_BPP)
    W = C_BPP // 8
    assert W - 1 == (1 << 31) - 1
    with pkg.Open(pkg.Config(ordinals=[0], bytes=C_BPP, timeout_ms=120000)) as p:
        r = p.Run()
        assert r.bytes_per_pair == C_BPP and r.verdict
        assert (r.sum_read[0][0], r.xor_read[0][0]) == oracle_src(oracle, 0, W)
        assert (r.sum_write[0][0], r.xor_write[0][0]) == oracle.write_checksum(SEED, 0, 0, r.run_seq, W)
        assert p.Diagnose("read", 0, 0).bad_words == 0 and p.Diagnose("write", 0, 0).bad_words == 0

        idx = [W - 2, W - 1]
        spec = ref.read_spec(SEED, 1, 0, 0, W, W)
        faults = read_faults(spec, idx)
        for k, m in masks(spec, faults):
            p.Corrupt(0, 8 * k, m)
        wspec = ref.write_spec(SEED, 1, 0, 0, r.run_seq + 1, W)
        wfaults = write_faults(wspec, idx)
        p.CorruptLanding(0, 0, masks(wspec, wfaults))
        r = p.Run()
        assert (r.reach_read, r.reach_write, r.verdict) == ([[0]], [[0]], False)
        assert_report(p.Diagnose("read", 0, 0),
                      want_sparse(spec, faults, "read", 0, r.run_seq, VMM), "read")
        assert_report(p.Diagnose("write", 0, 0),
                      want_sparse(wspec, wfaults, "write", 0, r.run_seq, VMM + round_up(C_BPP, VMM)), "write")
        for k, m in masks(spec, faults):
            p.Corrupt(0, 8 * k, m)
        p.CorruptLanding(0, 0, [])

        bw = p.BwCurve(reps=2)
        assert len(bw.sizes) == 23 and bw.sizes == bwcurve_ref.ladder(C_BPP) and bw.sizes[-1] == C_BPP
        assert bw.status[0][0] == 0 and bw.bad_sizes[0][0] == 0
        assert list(zip(bw.sum[0][0], bw.xr[0][0])) == list(src_sums(0, C_BPP))


def test_c_open_refuses_more_than_16_gib_and_allocates_nothing(pkg):
    import torch

    free0, _ = torch.cuda.mem_get_info(0)
    for nbytes in (C_BPP + 128, C_BPP + 255):
        with pytest.raises(pkg.ProbeError) as e:
            pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes))
        assert e.value.code == pkg.abi.ERR_ARG, nbytes
    free1, _ = torch.cuda.mem_get_info(0)
    assert free1 >= free0 - (256 << 20), (free0, free1)  # others share the device: allow its own churn, not 16 GiB


@pytest.mark.parametrize("op", [OP_READ, OP_WRITE], ids=["pull", "push"])
def test_b_ce_alltoall_block_1_starts_past_2_32(pkg, op):
    """Two ranks, sliced, A's 4 GiB + 8 KiB + 128 per pair, both copying at once: block 1 of each exchange area starts
    past byte 2^32 of the area, and every block is clean at every size with its source slice's (S, X)."""
    n = 2
    guard(pkg, n, A_BPP, extra=round_up(n * A_BPP, VMM))
    sizes = bwcurve_ref.ladder(A_BPP)
    with pkg.Open(pkg.Config(ordinals=[0, 0], bytes=A_BPP, flags=SAME, ctas=8, timeout_ms=120000,
                             link_peak_gbps=SAME_DEVICE_LINK_PEAK_GBPS)) as p:
        ca = p.CeAllToAll(op, reps=1)
        assert ca.sizes == sizes and ca.area_bytes == round_up(n * A_BPP, VMM)
        assert ca.measured == [True, True] and ca.status == [0, 0] and ca.blocks == [1, 1]
        for g, j in ((0, 1), (1, 0)):
            src = g if op == OP_WRITE else j
            assert ca.cell_measured[g][j] and ca.cell_status[g][j] == 0 and ca.bad_sizes[g][j] == 0, (g, j)
            assert ca.bad_words[g][j] == [0] * len(sizes) and ca.first_bad[g][j] == [U64_MAX] * len(sizes), (g, j)
            assert list(zip(ca.sum[g][j], ca.xr[g][j])) == list(src_sums(src, A_BPP)), (g, j)
