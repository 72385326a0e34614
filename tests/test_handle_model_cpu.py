"""Pins tests/handle_model.py against hand-built cases, without a GPU: the (S, X) of a slice with corrupted words, the
latency chase over overridden words, what a landing slot holds after a history of runs, unmaps and landing faults
(and so what cdprobe_diagnose must report on it), the counters and the unmapped-pair rule, the all-reduce under
corruptions (also cancelling ones) and faults against a direct recomputation, its skip rule, and the all-to-all's
sticky exchange area; the same for the two-shot, LL, ring and push all-reduces (each protocol's faults at edge words,
drop and unstored modes included, against whole-array recomputations from their references) and for memcpy (a
corrupted source word fails exactly the cells and sizes that copy it), with their refusals, counters, skip rules and
sticky areas, the exchange area shared by memcpy and the all-to-all in both orders; and for the copy-engine all-to-all
(its blocks are memcpy's, checked by their owners: corruptions, edge faults of every mode, its refusals and their
precedence, the queue limit of every process, its all-or-nothing down rule and its own counter)."""
import ctypes as C
import random

import numpy as np
import pytest

import handle_model as hm
import allreduce_ll_ref
import allreduce_push_ref
import allreduce_ref
import allreduce_ring_ref
import alltoall_ref
import bwcurve_ref
import ce_alltoall_ref
import latency_ref
import memcpy_ref
import word_ref as ref

SEED = hm.SEED
G = ref.GRANULE_WORDS


def checksum_of(oracle, words):
    a = np.ascontiguousarray(words, dtype=np.uint64)
    s, x = C.c_uint64(), C.c_uint64()
    oracle.lib().cdoracle_checksum(a.ctypes.data_as(C.POINTER(C.c_uint64)), len(a), C.byref(s), C.byref(x))
    return s.value, x.value


def no_schedule(*args):
    raise AssertionError("the model needs no phase table here")


@pytest.mark.parametrize("first,words", [(0, 3 * G + 640), (5 * G + 16, 2 * G), (1000, 77)])
def test_corrupted_checksum_equals_the_checksum_of_the_corrupted_words(oracle, first, words):
    rng = random.Random(first + words)
    rank = 2
    region = ref.src_words(SEED, rank, first, words)
    tail = words // G * G
    picks = {first, first + words - 1, first + tail + (words - tail) // 2, first + rng.randrange(words)}
    cases = [{k: rng.getrandbits(64) | 1} for k in sorted(picks)]
    cases.append({k: 1 << rng.randrange(64) for k in picks})                     # several words, several granules
    cases.append({first - 1: 0xFF, first + words: 0xFF00})                      # outside the slice: no change
    base = oracle.src_checksum(SEED, rank, first, words)
    for corr in cases:
        obs = region.copy()
        for k, m in corr.items():
            if first <= k < first + words:
                obs[k - first] ^= np.uint64(m)
        assert hm.corrupted_checksum(base, SEED, rank, first, words, corr) == checksum_of(oracle, obs), corr
    assert hm.corrupted_checksum(base, SEED, rank, first, words, cases[-1]) == base


def plain_chase_digest(table, i, j, lines, hops, reps):
    """The chase restated over a word table (numpy), independently of latency_ref.chase."""
    d = 0
    for r in range(reps + 1):
        line = latency_ref.start_line(SEED, i, j, r, lines)
        for h in range(hops):
            v = int(table[latency_ref.LINE_WORDS * line])
            d ^= v
            line = latency_ref.next_line(v, h, lines)
    return d


def test_latency_over_overridden_words(oracle):
    n, nbytes = 1, 64 << 10
    m = hm.HandleModel(oracle, no_schedule, n, nbytes, sm_count=132)
    lines, hops, reps = m.bpp // latency_ref.LINE_BYTES, 40, 2
    first = m.first_word(0, 0)
    table = latency_ref.region_words(SEED, 0, first, lines)
    clean = m.latency(hops, reps)[(0, 0)]
    assert clean == dict(measured=True, digest=plain_chase_digest(table, 0, 0, lines, hops, reps), status=0)
    # a word the chase loads: the path and the digest change, and the cell is an integrity failure
    k = latency_ref.loaded_word(SEED, 0, 0, first, lines, 1, 7)
    mask = 0x5A5A << 20
    m.corrupt_word(0, k, mask)
    bad = table.copy()
    bad[k - first] ^= np.uint64(mask)
    got = m.latency(hops, reps)[(0, 0)]
    assert got["digest"] == plain_chase_digest(bad, 0, 0, lines, hops, reps) != clean["digest"]
    assert got["status"] == hm.ERR_INTEGRITY
    # a word no hop loads (not the first of its line): same digest, clean
    m.corrupt_word(0, k, mask)
    assert m.corrupt == {}
    m.corrupt_word(0, k + 1, mask)
    assert m.latency(hops, reps)[(0, 0)] == clean


def test_slot_history_maps_to_the_word_ref_report(oracle):
    n, nbytes = 3, 1 << 20
    m = hm.HandleModel(oracle, no_schedule, n, nbytes, sm_count=132)
    W = m.W
    m.unmapped.add((0, 1))                          # down from the start: slot (0, 1) and (1, 0) never written
    r = m.run()
    assert r["run_seq"] == hm.FIRST_RUN_SEQ
    assert r["cells"][(0, 1)]["reach_write"] == r["cells"][(1, 0)]["reach_read"] == 0
    assert r["cells"][(0, 1)]["status"] == hm.ERR_STATE and r["cells"][(1, 0)]["status"] == 0
    spec, obs = m.diagnose("write", 0, 1)
    rep = ref.expected_report(spec, obs)
    assert rep["bad_words"] == rep["zero_words"] == W and rep["kind_count"][ref.ZERO] == W
    assert not m.maps(0, 1) and m.maps(1, 0) and m.maps(1, 1)
    m.unmapped.discard((0, 1))
    faults = [(0, 1 << 3), (W - 1, 0xF0F0)]
    m.arm(0, 2, faults)
    r = m.run()
    seq = r["run_seq"]
    assert r["cells"][(0, 2)]["reach_write"] == 0 and r["cells"][(0, 1)]["reach_write"] == 1
    rep = ref.expected_report(*m.diagnose("write", 0, 2))
    assert rep["bad_words"] == 2 and rep["kind_count"][ref.FLIP] == 2 and rep["first_bad"] == 0
    assert ref.expected_report(*m.diagnose("write", 0, 1))["bad_words"] == 0
    m.arm(1, 0, [])                                 # disarms the one arming of this handle
    m.unmapped.add((2, 0))                          # writer 0 -> 2 misses one run: its slot is one run stale
    m.run()
    rep = ref.expected_report(*m.diagnose("write", 0, 2))
    assert rep["kind_count"][ref.STALE] == W - 2 and rep["kind_count"][ref.FLIP] == 2
    assert all(s["run_seq"] == seq for s in rep["sample"] if s["kind"] == ref.STALE)
    m.unmapped.discard((2, 0))
    m.run()
    for i, j in m.cells():
        for op in ("read", "write"):
            assert ref.expected_report(*m.diagnose(op, i, j))["bad_words"] == 0, (op, i, j)


def test_counters_and_the_unmapped_rule_of_the_measurements(oracle):
    n, nbytes = 3, 1 << 20
    m = hm.HandleModel(oracle, no_schedule, n, nbytes, sm_count=132)
    m.unmapped.add((2, 0))
    seq, pp = m.pingpong()
    assert seq == 1 and pp[(2, 0)] == pp[(0, 2)] == dict(measured=False, status=hm.ERR_STATE)
    assert pp[(0, 1)] == dict(measured=True, status=0)
    seq, at = m.atomics()
    assert seq == 1 and at[(2, 0)] == dict(measured=False, status=hm.ERR_STATE) and at[(0, 2)]["measured"]
    assert m.pingpong()[0] == 2 and m.atomics()[0] == 2
    # bwcurve: a corrupted word fails exactly the sizes whose prefix covers it
    k = 3 * G + 1
    first = m.first_word(0, 1)
    m.corrupt_word(1, first + k, 1 << 9)
    seq, sizes, bw = m.bwcurve()
    assert seq == 1 and sizes[-1] == m.bpp
    want_bad = sum(1 << b for b, s in enumerate(sizes) if s // 8 > k)
    assert bw[(0, 1)]["bad_sizes"] == want_bad and bw[(0, 1)]["status"] == hm.ERR_INTEGRITY
    assert bw[(0, 1)]["sx"][0] == oracle.src_checksum(SEED, 1, first, sizes[0] // 8)
    assert bw[(2, 1)]["bad_sizes"] == 0 and bw[(2, 0)] == dict(measured=False, status=hm.ERR_STATE)


def test_phase_table_idles_the_jobs_of_an_unmapped_pair(pkg, oracle):
    n, nbytes = 4, 1 << 20
    m = hm.HandleModel(oracle, hm.schedule_fn(pkg.abi.load_library(), pkg.abi), n, nbytes, sm_count=132, ctas=8)
    full = {g: m.phase_table(g) for g in range(n)}
    m.unmapped.add((1, 2))
    for g in range(n):
        tab = m.phase_table(g)
        assert len(tab) == len(full[g])
        for ph, was in zip(tab, full[g]):
            if g in (1, 2) and was["job0"] in ("read", "write", "warm") and was["peer0"] == 3 - g:
                assert (ph["job0"], ph["peer0"]) == ("-", g)
            else:
                assert (ph["job0"], ph["peer0"]) == (was["job0"], was["peer0"])
    # the N = 1 streamed pass, and the serial verify at N = 1
    m1 = hm.HandleModel(oracle, m._schedule, 1, nbytes, sm_count=132)
    assert m1.phase_table(0) == [{"job0": "write", "peer0": 0, "job1": "-", "peer1": 0},
                                 {"job0": "read", "peer0": 0, "job1": "verify", "peer1": 0}]
    m1.set_flag(hm.FLAG_OVERLAP_VERIFY, False)
    assert [ph["job0"] for ph in m1.phase_table(0)] == ["write", "read", "verify"]


# ---- the all-reduce and the all-to-all -------------------------------------------------------------------------
def allreduce_direct(n, sizes, corrupt, fault=None, reps=1):
    """The all-reduce restated over whole word arrays (numpy): per size, (S, X) of the output of the last rep, and the
    bad words and first bad offset over every rep (the warm-up, then `reps` timed reps), given the corruptions at rest
    {(rank, word): mask} and a fault (k, word, drop) of this row in timed rep 1: the word + 1, or its 8 KiB unit 0s."""
    W = sizes[-1] // 8
    src = [ref.src_words(SEED, j, 0, W) for j in range(n)]
    clean = sum(src[1:], src[0].copy())
    for (r, k), m in corrupt.items():
        if k < W:
            src[r][k] ^= np.uint64(m)
    at_rest = sum(src[1:], src[0].copy())
    out = []
    for k, s in enumerate(sizes):
        outs = [at_rest[:s // 8].copy() for _ in range(reps + 1)]
        if fault is not None and fault[0] == k:
            if fault[2]:
                outs[1][fault[1] // 1024 * 1024:(fault[1] // 1024 + 1) * 1024] = 0
            else:
                outs[1][fault[1]] += np.uint64(1)
        bad = [np.flatnonzero(w != clean[:s // 8]) for w in outs]
        first = min((int(b[0]) for b in bad if len(b)), default=None)
        out.append((allreduce_ref.checksum(outs[-1]), sum(len(b) for b in bad),
                    ref.U64_MAX if first is None else 8 * first))
    return out


def test_allreduce_under_one_corruption_equals_the_reference(oracle):
    n = 3
    m = hm.HandleModel(oracle, no_schedule, n, 1 << 20, sm_count=132)
    sizes = bwcurve_ref.ladder(m.bpp)
    for rank, word, mask in ((0, 0, 1), (2, 3 * G + 7, 1 << 63), (1, m.W - 1, 0xFFFF), (1, m.W + 5, 0xF0)):
        m.corrupt_word(rank, word, mask)
        got = m.allreduce(1)
        want = allreduce_ref.expected_corrupted(SEED, n, tuple(sizes), rank, word, mask)
        bits = 0 if word >= m.W else sum(1 << k for k, s in enumerate(sizes) if s // 8 > word)
        for g in range(n):
            row = got["rows"][g]
            assert row["sx"] == want and row["bad_sizes"] == bits, (rank, word, g)
            assert row["status"] == (hm.ERR_INTEGRITY if bits else 0)
            assert row["bad_words"] == [2 * ((bits >> k) & 1) for k in range(len(sizes))]  # the warm-up and rep 1
            assert row["first_bad"] == [8 * word if (bits >> k) & 1 else ref.U64_MAX for k in range(len(sizes))]
        m.corrupt_word(rank, word, mask)  # restore
        assert m.allreduce(1)["rows"][0]["sx"] == list(allreduce_ref.expected(SEED, n, tuple(sizes)))


def test_allreduce_under_several_corruptions_and_a_fault_equals_a_direct_recomputation(oracle):
    n = 3
    m = hm.HandleModel(oracle, no_schedule, n, 1 << 20, sm_count=132)
    sizes = bwcurve_ref.ladder(m.bpp)
    rng = random.Random(5)
    corrupt = {(0, 5): 1 << 40, (1, 5): 0x3, (2, 4 * G - 1): rng.getrandbits(64) | 1, (1, m.W - 1): 1 << 7,
               (0, 2 * m.W + 3): 0xFF}
    # a pair whose deltas cancel on word c: rank 2's change undoes rank 0's, so the sum there is clean
    c = 3 * G + 100
    wa, wb = hm.src_word(SEED, 0, c), hm.src_word(SEED, 2, c)
    da = ((wa ^ 0x1234) - wa) & hm.M64
    corrupt[(0, c)] = 0x1234
    corrupt[(2, c)] = wb ^ ((wb - da) & hm.M64)
    for (r, k), mask in corrupt.items():
        m.corrupt_word(r, k, mask)
    want = allreduce_direct(n, sizes, corrupt)
    got = m.allreduce(1)["rows"]
    for g in range(n):
        assert [(sx, b, f) for sx, b, f in zip(got[g]["sx"], got[g]["bad_words"], got[g]["first_bad"])] == want, g
    # the cancelled word is clean: a prefix ending just past it has exactly the bad words of the others
    k = next(k for k, s in enumerate(sizes) if s // 8 > c)
    assert want[k][1] == 2 * len({w for (r, w) in corrupt if w < min(sizes[k] // 8, m.W)} - {c})  # warm-up, rep 1
    # an armed fault on row 1, size 2, on a corrupted word: timed rep 1 adds 1 to the corrupted sum, or (drop) stores
    # nothing of its unit; then a drop on row 2 in the last, partial unit of the last size
    fk, last = 2, len(sizes) - 1
    for g0, k0, w0, drop in ((1, fk, 5, False), (1, fk, 5, True), (2, last, m.W - 1, True)):
        m.arm_measure(m.ar_fault, 0, (int(drop) << 48) | ((g0 + 1) << 32) | ((k0 + 1) << 24) | w0)
        for reps in (1, 3):
            got = m.allreduce(reps)["rows"]
            for g in range(n):
                want = allreduce_direct(n, sizes, corrupt, (k0, w0, drop) if g == g0 else None, reps)
                assert [(sx, b, f) for sx, b, f in zip(got[g]["sx"], got[g]["bad_words"], got[g]["first_bad"])] == \
                    want, (g0, k0, drop, reps, g)
            # the size fails even when its last rep is clean
            assert got[g0]["bad_sizes"] == got[(g0 + 1) % n]["bad_sizes"] | 1 << k0


def test_allreduce_skip_rule_refusals_and_counters(oracle):
    n = 3
    m = hm.HandleModel(oracle, no_schedule, n, 1 << 20, sm_count=132)
    sizes = bwcurve_ref.ladder(m.bpp)
    assert m.allreduce(2)["call_seq"] == 1
    for bad in ((4 << 32) | (1 << 24), (1 << 24) | 5, (1 << 32) | ((len(sizes) + 1) << 24),
                (1 << 32) | (1 << 24) | sizes[0] // 8, 1 << 32, (1 << 49) | (1 << 32) | (1 << 24),
                (1 << 63) | (1 << 48) | (1 << 32) | (1 << 24)):
        m.arm_measure(m.ar_fault, 0, bad)
        assert m.allreduce(2) is None, hex(bad)
    assert m.ar_calls == 1
    m.arm_measure(m.ar_fault, 0, 0)
    assert m.ar_fault == {}
    m.unmapped.add((2, 1))
    got = m.allreduce(2)
    assert got["call_seq"] == 2 and got["rows"] == {g: dict(measured=False, status=hm.ERR_STATE) for g in range(n)}
    assert (m.bw_calls, m.pp_calls, m.at_calls, m.a2a_calls, m.runs) == (0, 0, 0, 0, 0)
    # a refusal is checked before the mapping verdict
    m.arm_measure(m.ar_fault, 0, 1 << 32)
    assert m.allreduce(2) is None and m.ar_calls == 2
    m.arm_measure(m.ar_fault, 0, 0)
    m.unmapped.discard((2, 1))
    got = m.allreduce(2)
    assert got["call_seq"] == 3 and all(r["status"] == 0 and r["bad_sizes"] == 0 for r in got["rows"].values())


def test_alltoall_sticky_area_fault_and_counters(oracle):
    n = 3
    m = hm.HandleModel(oracle, no_schedule, n, 1 << 20, sm_count=132)
    sizes = bwcurve_ref.ladder(m.bpp)
    # a refused call builds no area
    m.arm_measure(m.a2a_fault, 0, (1 << 40) | (1 << 32) | (1 << 24))  # the diagonal, which N = 3 does not have
    assert m.alltoall(1) is None and m.area_down is None and m.a2a_calls == 0
    m.arm_measure(m.a2a_fault, 0, 0)
    m.unmapped.add((0, 2))
    m.corrupt_word(1, 3, 1 << 5)                                       # source corruptions do not touch it
    for step in ("first", "remapped", "again"):
        got = m.alltoall(1)
        assert got["sizes"] == sizes and m.area_down == {(0, 2)}, step
        assert got["cells"][(0, 2)] == dict(cell_measured=False, cell_status=hm.ERR_STATE), step
        assert [got["ranks"][g]["blocks"] for g in range(n)] == [1, 2, 2], step
        assert all(r["measured"] for r in got["ranks"].values())
        for (s, d), c in got["cells"].items():
            if (s, d) != (0, 2):
                assert c["cell_status"] == 0 and c["bad_sizes"] == 0
                assert c["sx"] == [allreduce_ref.checksum(alltoall_ref.block_words(SEED, s, d, got["call_seq"], k, 1,
                                                                                      sz // 8))
                                   for k, sz in enumerate(sizes)]
        m.unmapped.discard((0, 2))                                     # remap: the area stays unmapped for (0, 2)
    assert m.a2a_calls == 3 and (m.ar_calls, m.bw_calls) == (0, 0)
    # an armed fault fails exactly its cell and size; with reps = 1 the folded rep is the faulted one
    fk, fw = len(sizes) - 1, m.W - 1
    m.arm_measure(m.a2a_fault, 0, (3 << 40) | (1 << 32) | ((fk + 1) << 24) | fw)
    for reps in (1, 2):
        got = m.alltoall(reps)
        c = got["cells"][(2, 0)]
        assert c["bad_sizes"] == 1 << fk and c["cell_status"] == hm.ERR_INTEGRITY
        assert c["bad_words"][fk] == 1 and c["first_bad"][fk] == 8 * fw
        words = alltoall_ref.block_words(SEED, 2, 0, got["call_seq"], fk, reps, sizes[fk] // 8)
        if reps == 1:
            words[fw] ^= np.uint64(1)
        assert c["sx"][fk] == allreduce_ref.checksum(words)
        assert all(o["bad_sizes"] == 0 for key, o in got["cells"].items() if key not in ((2, 0), (0, 2)))


# ---- the two-shot, LL, ring and push all-reduces, and memcpy ----------------------------------------------------
EDGE_BPP = 57 * 8192 + 384  # a partial last unit in a partial last granule: ladder 4096 ... 262144, 467328
LADDERS = {"ts": bwcurve_ref.ladder, "ll": allreduce_ll_ref.ladder, "ring": bwcurve_ref.ladder,
           "push": bwcurve_ref.ladder}


def edge_model(oracle, n=3):
    m = hm.HandleModel(oracle, no_schedule, n, EDGE_BPP * max(n - 1, 1), sm_count=132)
    assert m.bpp == EDGE_BPP
    return m


def call(m, name, reps):
    return {"ts": m.twoshot, "ll": m.ll, "ring": m.ring, "push": m.push}[name](reps)


def sources(n, W, corrupt):
    srcs = [ref.src_words(SEED, j, 0, W) for j in range(n)]
    for (r, k), mask in corrupt.items():
        if k < W:
            srcs[r][k] ^= np.uint64(mask)
    return srcs


def ring_rep1(srcs, g, s, fault):
    """Row g after timed rep 1 of a ring fault (sender, word, phase, mode), over whole arrays (test_allreduce_ring_gpu's
    restatement, on the sources at rest)."""
    n, nw = len(srcs), s // 8
    sender, word, phase, mode = fault
    out = sum(x[:nw] for x in srcs)
    if mode == 2 or g not in allreduce_ring_ref.failing_rows(n, sender, phase, s, word):
        return out
    u0, u1 = word // 1024 * 1024, min(word // 1024 * 1024 + 1024, nw)
    if phase == 1 and mode == 0:
        out[word] ^= np.uint64(1)
        return out
    c = allreduce_ring_ref.chunk_of(s, n, word)
    part = sum(srcs[j][:nw] for j in allreduce_ring_ref.partial_ranks(n, sender, c)) if sender != c else None
    if phase == 1:
        out[u0:u1] = 0 if part is None else part[u0:u1]
    elif mode == 0:
        p = int(part[word])
        out[word] = np.uint64((int(out[word]) + (p ^ 1) - p) % (1 << 64))
    else:
        out[u0:u1] -= part[u0:u1]
    return out


def rep1_direct(name, srcs, g, k, s, fault, call_seq):
    """Row g's output after timed rep 1 of size s, with `fault` (the option's fields, as the per-protocol suites name
    them) or None, over whole arrays."""
    nw = s // 8
    out = sum(x[:nw] for x in srcs)
    if fault is None or fault[0] != k:
        return out
    f = fault[1:]
    if name == "ts":
        recv, word, drop = f
        if g == recv:
            if drop:
                out[word // 1024 * 1024:word // 1024 * 1024 + 1024] = 0
            else:
                out[word] ^= np.uint64(1)
        return out
    if name == "ll":
        sender, recv, word, mode = f
        if g == recv and mode == 0:
            v = int(srcs[sender][word]) + allreduce_ll_ref.salt(SEED, sender, allreduce_ll_ref.flag(call_seq, k, 1))
            out[word] = np.uint64((int(out[word]) + (v ^ 1) - v) % (1 << 64))
        return out
    if name == "ring":
        return ring_rep1(srcs, g, s, f)
    mode, rank, word = f
    return allreduce_push_ref.rep([x[:nw] for x in srcs], s, (mode, rank, word))[g]


def ar_direct(name, n, sizes, corrupt, g, fault=None, reps=1, call_seq=1):
    """Per size of row g: ((S, X) of the last timed rep, bad words, first bad offset, whether the size fails), from
    whole arrays: every rep checked (the LL: only the last, with a mode-2 word read as 0 in every rep of its size)."""
    W = sizes[-1] // 8
    clean = sum(ref.src_words(SEED, j, 0, W) for j in range(n))
    srcs = sources(n, W, corrupt)
    rest = sum(srcs[1:], srcs[0].copy())
    out = []
    for k, s in enumerate(sizes):
        nw = s // 8
        outs = [rest[:nw].copy() for _ in range(reps + 1)]
        outs[1] = rep1_direct(name, srcs, g, k, s, fault, call_seq)
        want = allreduce_ref.checksum(clean[:nw])
        if name == "ll":
            seen = outs[-1].copy()
            if fault is not None and fault[0] == k and fault[-1] == 2 and fault[2] == g:
                seen[fault[3]] = 0
            bad = [np.flatnonzero(seen != clean[:nw])]
        else:
            bad = [np.flatnonzero(o != clean[:nw]) for o in outs]
        n_bad = sum(len(b) for b in bad)
        first = min((int(b[0]) for b in bad if len(b)), default=None)
        fails = bool(n_bad) or any(allreduce_ref.checksum(o) != want for o in outs)
        out.append((allreduce_ref.checksum(outs[-1]), n_bad, ref.U64_MAX if first is None else 8 * first, fails))
    return out


def model_rows(got, n):
    return {g: [(sx, b, f, bool((got["rows"][g]["bad_sizes"] >> k) & 1))
                for k, (sx, b, f) in enumerate(zip(got["rows"][g]["sx"], got["rows"][g]["bad_words"],
                                                   got["rows"][g]["first_bad"]))] for g in range(n)}


@pytest.mark.parametrize("name", ["ts", "ll", "ring", "push"])
def test_ladder_allreduce_under_one_corruption_equals_the_reference(oracle, name):
    n = 3
    m = edge_model(oracle, n)
    sizes = LADDERS[name](m.bpp)
    for rank, word, mask in ((0, 0, 1), (2, 3 * G + 7, 1 << 63), (1, m.W - 1, 0xFFFF), (1, m.W + 5, 0xF0)):
        m.corrupt_word(rank, word, mask)
        got = call(m, name, 2)
        assert got["sizes"] == sizes
        want = allreduce_ref.expected_corrupted(SEED, n, tuple(sizes), rank, word, mask)
        bits = 0 if word >= m.W else sum(1 << k for k, s in enumerate(sizes) if s // 8 > word)
        checked = 1 if name == "ll" else 3  # the LL checks the last rep's words; the others every rep's
        for g in range(n):
            row = got["rows"][g]
            assert row["sx"] == want and row["bad_sizes"] == bits, (rank, word, g)
            assert row["status"] == (hm.ERR_INTEGRITY if bits else 0)
            assert row["bad_words"] == [checked * ((bits >> k) & 1) for k in range(len(sizes))]
            assert row["first_bad"] == [8 * word if (bits >> k) & 1 else ref.U64_MAX for k in range(len(sizes))]
        m.corrupt_word(rank, word, mask)  # restore
        assert call(m, name, 1)["rows"][0]["sx"] == list(allreduce_ref.expected(SEED, n, tuple(sizes)))


def edge_faults(name, n, sizes, W):
    """(option value, fault as ar_direct takes it) at the edges: word 0 of size 0, the last word of the last, partial
    unit, and each protocol's drop or unstored mode."""
    last = len(sizes) - 1
    Wl = sizes[last] // 8
    if name == "ts":
        a = lambda recv, k, w, drop=False: (int(drop) << 48) | ((recv + 1) << 32) | ((k + 1) << 24) | w
        cases = [(0, 0, 0, False), (n - 1, last, Wl - 1, False), (1, last, Wl - 1, True), (2, 0, 0, True)]
        return [(a(r, k, w, d), (k, r, w, d)) for r, k, w, d in cases]
    if name == "ll":
        a = lambda s, r, k, w, mode=0: (mode << 48) | ((s + 1) << 40) | ((r + 1) << 32) | ((k + 1) << 24) | w
        cases = [(0, 1, 0, 0, 0), (2, 0, last, Wl - 1, 0), (1, 1, 0, 0, 2), (2, 2, last, Wl - 1, 2),
                 (0, 2, 1, 10, 1)]
        return [(a(*c), (c[2], c[0], c[1], c[3], c[4])) for c in cases]
    if name == "ring":
        a = lambda s, k, w, ph, mode: (mode << 48) | (ph << 40) | ((s + 1) << 32) | ((k + 1) << 24) | w
        out = []
        for k, w in ((0, 0), (last, Wl - 1)):
            for ph in (0, 1):
                for mode in (0, 1):
                    c = allreduce_ring_ref.chunk_of(sizes[k], n, w)
                    s = next(s for s in range(n) if c in allreduce_ring_ref.pushes(n, s, ph))
                    out.append((a(s, k, w, ph, mode), (k, s, w, ph, mode)))
        return out
    a = lambda r, k, w, mode: (mode << 48) | ((r + 1) << 32) | ((k + 1) << 24) | w
    out = []
    for k, w in ((0, 0), (last, Wl - 1)):
        for mode in range(4):
            r = 1
            if mode == 3 and allreduce_push_ref.word_owner(sizes[k], n, w) == r:
                r = 2
            out.append((a(r, k, w, mode), (k, mode, r, w)))
    return out


@pytest.mark.parametrize("name", ["ts", "ll", "ring", "push"])
def test_ladder_allreduce_under_cancelling_corruptions_and_edge_faults_equals_a_direct_recomputation(oracle, name):
    n = 3
    m = edge_model(oracle, n)
    sizes = LADDERS[name](m.bpp)
    W = m.W
    corrupt = {(0, 5): 1 << 40, (1, 5): 0x3, (2, 4 * G - 1): 0x55 << 9, (1, W - 1): 1 << 7, (0, 2 * W + 3): 0xFF,
               (2, 1): 1 << 3}
    c = 3 * G + 100  # rank 2's change undoes rank 0's: the sum there is clean
    wa, wb = hm.src_word(SEED, 0, c), hm.src_word(SEED, 2, c)
    corrupt[(0, c)] = 0x1234
    corrupt[(2, c)] = wb ^ ((wb - (((wa ^ 0x1234) - wa) & hm.M64)) & hm.M64)
    for (r, k), mask in corrupt.items():
        m.corrupt_word(r, k, mask)
    got = model_rows(call(m, name, 1), n)
    for g in range(n):
        assert got[g] == ar_direct(name, n, sizes, corrupt, g), g
    opt = name + "_fault"
    for value, fault in edge_faults(name, n, sizes, W):
        m.arm_measure(getattr(m, opt), 0, value)
        for reps in (1, 3):
            out = call(m, name, reps)
            assert out is not None, hex(value)
            got = model_rows(out, n)
            for g in range(n):
                assert got[g] == ar_direct(name, n, sizes, corrupt, g, fault, reps, out["call_seq"]), \
                    (hex(value), reps, g)
    m.arm_measure(getattr(m, opt), 0, 0)


REFUSED = {
    "ts": lambda n, sizes: [((n + 1) << 32) | (1 << 24), (1 << 24) | 5, (1 << 32) | ((len(sizes) + 1) << 24),
                            (1 << 32) | (1 << 24) | sizes[0] // 8, 1 << 32, (1 << 49) | (1 << 32) | (1 << 24)],
    "ll": lambda n, sizes: [(1 << 40) | (1 << 32) | (1 << 24), (3 << 48) | (1 << 40) | (2 << 32) | (1 << 24),
                            (2 << 48) | (1 << 40) | (2 << 32) | (1 << 24), (1 << 40) | (2 << 32) | (1 << 24) | sizes[0] // 8,
                            (1 << 48) | (1 << 40) | (2 << 32) | (1 << 24) | 10_000_000, ((n + 1) << 40) | (1 << 32) | (1 << 24),
                            (1 << 40) | (2 << 32) | ((len(sizes) + 1) << 24)],
    "ring": lambda n, sizes: [(3 << 48) | (1 << 32) | (1 << 24), (2 << 40) | (1 << 32) | (1 << 24),
                              ((n + 1) << 32) | (1 << 24), (1 << 32) | ((len(sizes) + 1) << 24),
                              (3 << 32) | (1 << 24),  # size 0 is one unit, rank 2's, which it never pushes in phase 0
                              (2 << 48) | (1 << 32) | (1 << 24) | 10_000_000],
    "push": lambda n, sizes: [(4 << 48) | (1 << 32) | (1 << 24), ((n + 1) << 32) | (1 << 24),
                              (1 << 32) | ((len(sizes) + 1) << 24), (1 << 32) | (1 << 24) | sizes[0] // 8,
                              (3 << 48) | (3 << 32) | (1 << 24)],  # mode 3 to the word's owner, rank 2
}


@pytest.mark.parametrize("name", ["ts", "ll", "ring", "push"])
def test_ladder_allreduce_refusals_counters_skip_rule_and_sticky_area(oracle, name):
    n = 3
    m = hm.HandleModel(oracle, no_schedule, n, 1 << 20, sm_count=132)
    sizes = LADDERS[name](m.bpp)
    calls, opt = name + "_calls", name + "_fault"
    for bad in REFUSED[name](n, sizes):
        m.arm_measure(getattr(m, opt), 0, bad)
        assert call(m, name, 2) is None, hex(bad)
    assert getattr(m, calls) == 0 and m.ar_area_down[name] is None  # a refused call builds no area
    m.arm_measure(getattr(m, opt), 0, 0)
    assert call(m, name, 2)["call_seq"] == 1 and m.ar_area_down[name] == frozenset()
    m.unmapped.add((2, 1))  # any down pair stops every rank
    got = call(m, name, 2)
    assert got["call_seq"] == 2 and got["rows"] == {g: dict(measured=False, status=hm.ERR_STATE) for g in range(n)}
    m.unmapped.discard((2, 1))
    assert all(r["status"] == 0 and r["measured"] for r in call(m, name, 2)["rows"].values())
    assert (m.ar_calls, m.a2a_calls, m.mc_calls, m.bw_calls) == (0, 0, 0, 0)
    assert all(getattr(m, o + "_calls") == 0 for o in LADDERS if o != name)
    # an area built while a pair is down keeps every rank off after the remap, until the handle is closed; each
    # measurement's area is its own
    m2 = hm.HandleModel(oracle, no_schedule, n, 1 << 20, sm_count=132)
    m2.unmapped.add((0, 2))
    call(m2, name, 1)
    m2.unmapped.discard((0, 2))
    for _ in range(2):
        got = call(m2, name, 1)
        assert got["rows"] == {g: dict(measured=False, status=hm.ERR_STATE) for g in range(n)}
    assert m2.ar_area_down[name] == {(0, 2)} and getattr(m2, calls) == 3
    for other in LADDERS:
        if other != name:
            assert all(r["measured"] for r in call(m2, other, 1)["rows"].values()), other
    assert all(r["measured"] for r in m2.allreduce(1)["rows"].values())


def test_ll_and_ring_report_their_own_ladder_and_the_push_and_two_shot_the_bwcurve_one(oracle):
    m = hm.HandleModel(oracle, no_schedule, 1, 3 << 20, sm_count=132)
    assert m.ll(1)["sizes"] == [s for s in bwcurve_ref.ladder(3 << 20) if s <= 1 << 20]
    for name in ("ts", "ring", "push"):
        assert call(m, name, 1)["sizes"] == bwcurve_ref.ladder(3 << 20)
    # at N = 1 the ring pushes nothing and the push has no peer: their word faults are refused
    for name, v in (("ring", (1 << 32) | (1 << 24)), ("push", (3 << 48) | (1 << 32) | (1 << 24))):
        m.arm_measure(getattr(m, name + "_fault"), 0, v)
        assert call(m, name, 1) is None


def memcpy_direct(oracle, n, bpp, op, g, j, corrupt, fault=None, reps=1):
    """Per size of cell (g, j): ((S, X) of the last timed rep's destination, bad words, first bad offset, fails), from
    whole arrays: the source slice as it is at rest, and in timed rep 1 the fault (k, word, mode)."""
    c = memcpy_ref.cell(n, bpp, 1, op, g, j)
    src = sources(n, c["first_word"] + bpp // 8, corrupt)[c["src_rank"]][c["first_word"]:]
    out = []
    for k, s in enumerate(memcpy_ref.ladder(bpp)):
        nw = s // 8
        want = memcpy_ref.words(SEED, c, s)
        outs = [src[:nw].copy() for _ in range(reps + 1)]
        if fault is not None and fault[0] == k:
            if fault[2]:
                outs[1][:] = 0
            else:
                outs[1][fault[1]] = want[fault[1]] ^ np.uint64(1)
        bad = [np.flatnonzero(o != want) for o in outs]
        first = min((int(b[0]) for b in bad if len(b)), default=None)
        fails = any(len(b) for b in bad) or any(allreduce_ref.checksum(o) != allreduce_ref.checksum(want) for o in outs)
        out.append((allreduce_ref.checksum(outs[-1]), sum(len(b) for b in bad),
                    ref.U64_MAX if first is None else 8 * first, fails))
    return out


def memcpy_cells(got):
    return {key: [(sx, b, f, bool((c["bad_sizes"] >> k) & 1))
                  for k, (sx, b, f) in enumerate(zip(c["sx"], c["bad_words"], c["first_bad"]))]
            for key, c in got["cells"].items() if c["measured"]}


@pytest.mark.parametrize("op", [hm.OP_READ, hm.OP_WRITE], ids=["pull", "push"])
def test_memcpy_under_one_corruption_fails_exactly_the_cells_and_sizes_that_copy_it(oracle, op):
    n = 3
    m = edge_model(oracle, n)
    sizes = memcpy_ref.ladder(m.bpp)
    W = m.W
    for rank, word, mask in ((0, 0, 1), (2, W + 3 * G + 7, 1 << 63), (1, 2 * W - 1, 0xFFFF), (1, W - 1, 0xF0)):
        m.corrupt_word(rank, word, mask)
        got = m.memcpy(op, 2)
        assert got["sizes"] == sizes and set(got["cells"]) == {(g, j) for g in range(n) for j in range(n) if g != j}
        for (g, j), cell in got["cells"].items():
            c = memcpy_ref.cell(n, m.bpp, 1, op, g, j)
            at = word - c["first_word"]
            hit = c["src_rank"] == rank and 0 <= at < W
            bits = sum(1 << k for k, s in enumerate(sizes) if hit and s // 8 > at)
            assert cell["bad_sizes"] == bits and cell["status"] == (hm.ERR_INTEGRITY if bits else 0), (g, j, word)
            assert cell["bad_words"] == [3 * ((bits >> k) & 1) for k in range(len(sizes))]  # warm-up and two reps
            assert cell["first_bad"] == [8 * at if (bits >> k) & 1 else ref.U64_MAX for k in range(len(sizes))]
            words = memcpy_ref.words(SEED, c, m.bpp)
            if hit:
                words[at] ^= np.uint64(mask)
            assert cell["sx"] == [allreduce_ref.checksum(words[:s // 8]) for s in sizes], (g, j)
        m.corrupt_word(rank, word, mask)  # restore
    assert m.mc_calls == 4


@pytest.mark.parametrize("op", [hm.OP_READ, hm.OP_WRITE], ids=["pull", "push"])
def test_memcpy_under_corruptions_and_edge_faults_equals_a_direct_recomputation(oracle, op):
    n = 3
    m = edge_model(oracle, n)
    sizes = memcpy_ref.ladder(m.bpp)
    W, last = m.W, len(sizes) - 1
    corrupt = {(0, 5): 1 << 40, (1, W + 5): 0x3, (2, W - 1): 1 << 7, (0, 2 * W - 1): 0xFF, (1, 0): 1}
    for (r, k), mask in corrupt.items():
        m.corrupt_word(r, k, mask)
    got = memcpy_cells(m.memcpy(op, 1))
    for (g, j), cells in got.items():
        assert cells == memcpy_direct(oracle, n, m.bpp, op, g, j, corrupt), (g, j)
    # word 0 of size 0, the last word of the last, partial unit, and a word a corruption also changes; flip and drop
    for (g, j, k, w) in ((0, 1, 0, 0), (2, 1, last, W - 1), (1, 0, last, 5), (1, 2, 0, 0)):
        for mode in (0, 1):
            m.arm_measure(m.mc_fault, 0, (mode << 48) | ((g + 1) << 40) | ((j + 1) << 32) | ((k + 1) << 24) | w)
            for reps in (1, 2):
                got = memcpy_cells(m.memcpy(op, reps))
                for (gg, jj), cells in got.items():
                    f = (k, w, mode) if (gg, jj) == (g, j) else None
                    assert cells == memcpy_direct(oracle, n, m.bpp, op, gg, jj, corrupt, f, reps), (g, j, k, mode, reps)
    m.arm_measure(m.mc_fault, 0, 0)


def test_memcpy_refusals_counters_and_the_one_sided_skip_rule(oracle):
    n = 3
    m = hm.HandleModel(oracle, no_schedule, n, 1 << 20, sm_count=132)
    sizes = memcpy_ref.ladder(m.bpp)
    for op in (0, 3):
        assert m.memcpy(op, 1) is None
    for bad in ((2 << 48) | (1 << 40) | (2 << 32) | (1 << 24), (1 << 40) | (1 << 32) | (1 << 24),
                ((n + 1) << 40) | (1 << 32) | (1 << 24), (1 << 40) | (2 << 32) | ((len(sizes) + 1) << 24),
                (1 << 40) | (2 << 32) | (1 << 24) | sizes[0] // 8, (1 << 40) | (1 << 24)):
        m.arm_measure(m.mc_fault, 0, bad)
        assert m.memcpy(hm.OP_READ, 1) is None, hex(bad)
    assert m.mc_calls == 0 and m.area_down is None  # a refused call builds no exchange area
    m.arm_measure(m.mc_fault, 0, 0)
    m.memcpy(hm.OP_WRITE, 1)
    m.unmapped.add((2, 1))  # only the issuer's own direction stops, and only its cell
    got = m.memcpy(hm.OP_READ, 1)
    assert got["call_seq"] == 2 and got["cells"][(2, 1)] == dict(measured=False, status=hm.ERR_STATE)
    assert all(c["measured"] and c["status"] == 0 for key, c in got["cells"].items() if key != (2, 1))
    m.unmapped.discard((2, 1))
    assert all(c["measured"] for c in m.memcpy(hm.OP_READ, 1)["cells"].values())
    assert (m.a2a_calls, m.ar_calls, m.ts_calls, m.ll_calls, m.ring_calls, m.push_calls) == (0,) * 6


@pytest.mark.parametrize("first", ["memcpy", "alltoall", "ce_alltoall"])
def test_the_exchange_area_is_built_by_whichever_of_memcpy_and_alltoall_comes_first(oracle, first):
    n = 3
    m = hm.HandleModel(oracle, no_schedule, n, 1 << 20, sm_count=132)
    m.max_connections[0] = 32
    m.unmapped.add((0, 2))
    {"memcpy": lambda: m.memcpy(hm.OP_READ, 1), "alltoall": lambda: m.alltoall(1),
     "ce_alltoall": lambda: m.ce_alltoall(hm.OP_READ, 1)}[first]()
    assert m.area_down == {(0, 2)}
    m.unmapped.discard((0, 2))  # remap: the probe mapping is back, the exchange area's is not
    for op in (hm.OP_READ, hm.OP_WRITE):
        got = m.memcpy(op, 1)
        assert got["cells"][(0, 2)] == dict(measured=False, status=hm.ERR_STATE), op
        assert all(c["measured"] for key, c in got["cells"].items() if key != (0, 2))
    aa = m.alltoall(1)
    assert aa["cells"][(0, 2)] == dict(cell_measured=False, cell_status=hm.ERR_STATE)
    assert m.area_down == {(0, 2)}
    assert (m.mc_calls, m.a2a_calls, m.cea_calls) == {"memcpy": (3, 1, 0), "alltoall": (2, 2, 0),
                                                      "ce_alltoall": (2, 1, 1)}[first]
    # the copy-engine all-to-all needs every pair of the area: it stays off until close
    for op in (hm.OP_READ, hm.OP_WRITE):
        got = m.ce_alltoall(op, 1)
        assert got["ranks"] == {g: dict(measured=False, status=hm.ERR_STATE, blocks=0) for g in range(n)}
        assert got["cells"] == {(g, j): dict(cell_measured=False, cell_status=hm.ERR_STATE)
                                for g in range(n) for j in range(n) if g != j}
    # the all-reduces' areas are their own: built now, with every mapping up
    assert all(r["measured"] for r in m.twoshot(1)["rows"].values()) and m.ar_area_down["ts"] == frozenset()


# ---- the copy-engine all-to-all ------------------------------------------------------------------------------------
def ce_cells(got):
    """{cell: [((S, X), bad words, first bad, fails) per size]} of the cells the model says were checked."""
    return {key: [(sx, b, f, bool((c["bad_sizes"] >> k) & 1))
                  for k, (sx, b, f) in enumerate(zip(c["sx"], c["bad_words"], c["first_bad"]))]
            for key, c in got["cells"].items() if c["cell_measured"]}


def check_ce(oracle, m, op, reps, corrupt, faults=None):
    """One ce_alltoall call of the model against memcpy_direct for every block a local rank owns: the cell set, the
    rank rows, the verdicts, and per size the (S, X), bad words and first bad offset.  faults: {cell: (k, word, mode)}
    of modes 0 and 1."""
    n = m.n
    got = m.ce_alltoall(op, reps)
    cells = [c for c in ce_alltoall_ref.cells(n, m.diag) if ce_alltoall_ref.owner(op, *c) in m.local]
    assert sorted(got["cells"]) == sorted(cells)
    assert got["ranks"] == {g: dict(measured=True, status=0, blocks=n - 1 + m.diag) for g in m.local}
    assert got["area_min_bytes"] == n * m.bpp
    for (g, j), sizes in ce_cells(got).items():
        f = (faults or {}).get((g, j))
        want = memcpy_direct(oracle, n, m.bpp, op, g, j, corrupt, f, reps or 8)
        assert sizes == want, (g, j, f, reps)
        c = got["cells"][(g, j)]
        assert c["cell_status"] == (hm.ERR_INTEGRITY if c["bad_sizes"] else 0)
    return got


@pytest.mark.parametrize("op", [hm.OP_READ, hm.OP_WRITE], ids=["pull", "push"])
def test_ce_alltoall_under_one_several_and_cancelling_corruptions_equals_a_direct_recomputation(oracle, op):
    n = 3
    m = edge_model(oracle, n)
    m.max_connections[0] = 9
    sizes = memcpy_ref.ladder(m.bpp)
    W = m.W
    # one corruption: exactly the cells and sizes that copy it, (reps + 1) bad words each (the warm-up too)
    for reps in (1, 2, 0):
        for rank, word, mask in ((0, 0, 1), (2, W + 3 * G + 7, 1 << 63), (1, 2 * W - 1, 0xFFFF), (1, W - 1, 0xF0)):
            m.corrupt_word(rank, word, mask)
            got = check_ce(oracle, m, op, reps, {(rank, word): mask})
            for (g, j), cell in got["cells"].items():
                c = memcpy_ref.cell(n, m.bpp, 1, op, g, j)
                at = word - c["first_word"]
                hit = c["src_rank"] == rank and 0 <= at < W
                bits = sum(1 << k for k, s in enumerate(sizes) if hit and s // 8 > at)
                assert cell["bad_sizes"] == bits, (g, j, word)
                assert cell["bad_words"] == [((reps or 8) + 1) * ((bits >> k) & 1) for k in range(len(sizes))]
                assert cell["first_bad"] == [8 * at if (bits >> k) & 1 else ref.U64_MAX for k in range(len(sizes))]
            m.corrupt_word(rank, word, mask)  # restore
    assert m.corrupt == {} and m.cea_calls == 12
    # several at once, and two maskings of one word that cancel in part and then whole
    corrupt = {(0, 5): 1 << 40, (1, W + 5): 0x3, (2, W - 1): 1 << 7, (0, 2 * W - 1): 0xFF, (1, 0): 1}
    for (r, k), mask in corrupt.items():
        m.corrupt_word(r, k, mask)
    check_ce(oracle, m, op, 1, corrupt)
    m.corrupt_word(0, 5, (1 << 40) | 1)
    check_ce(oracle, m, op, 2, {**corrupt, (0, 5): 1})
    m.corrupt_word(0, 5, 1)
    check_ce(oracle, m, op, 2, {k: v for k, v in corrupt.items() if k != (0, 5)})
    assert (0, 5) not in m.corrupt


@pytest.mark.parametrize("op", [hm.OP_READ, hm.OP_WRITE], ids=["pull", "push"])
@pytest.mark.parametrize("n", [1, 3])
def test_ce_alltoall_edge_faults_of_every_mode_equal_a_direct_recomputation(oracle, n, op):
    """Modes 0 and 1 at word 0 of size 0, the last word of the last, partial unit and a word of that unit a corruption
    also changes (on the loop-back cell at N = 1), in timed rep 1 only; mode 2 changes no integrity field."""
    m = edge_model(oracle, n)
    m.max_connections[0] = 32
    sizes = memcpy_ref.ladder(m.bpp)
    W, last = m.W, len(sizes) - 1
    corrupt = {(n - 1, 5): 1 << 40, (0, W - 1): 0xFF}
    for (r, k), mask in corrupt.items():
        m.corrupt_word(r, k, mask)
    spots = [(0, 0, 0, 0), (0, 0, last, W - 1), (0, 0, last, W // 1024 * 1024 + 3), (0, 0, 0, 5)] if n == 1 else \
        [(0, 1, 0, 0), (2, 1, last, W - 1), (1, 0, last, 5), (1, 2, last, W // 1024 * 1024 + 3)]
    for g, j, k, w in spots:
        for mode in (0, 1):
            m.arm_measure(m.cea_fault, 0, (mode << 48) | ((g + 1) << 40) | ((j + 1) << 32) | ((k + 1) << 24) | w)
            for reps in (1, 2):
                got = check_ce(oracle, m, op, reps, corrupt, {(g, j): (k, w, mode)})
                assert got["cells"][(g, j)]["bad_sizes"] >> k & 1
        for reps in (1, 2):  # a hold of 3 ms: every block as if nothing were armed
            m.arm_measure(m.cea_fault, 0, (2 << 48) | ((g + 1) << 40) | ((j + 1) << 32) | ((k + 1) << 24) | 3000)
            check_ce(oracle, m, op, reps, corrupt)
    m.arm_measure(m.cea_fault, 0, 0)
    assert m.cea_calls == len(spots) * 6 and (m.mc_calls, m.a2a_calls) == (0, 0)


@pytest.mark.parametrize("op", [hm.OP_READ, hm.OP_WRITE], ids=["pull", "push"])
def test_ce_alltoall_fault_acts_only_in_the_process_that_hosts_its_issuer(oracle, op):
    """Process 0 of two (one rank each) checks the blocks it owns: a fault armed in process 1 on issuer 1 reaches cell
    (1, 0) when process 0 owns it (a push); the same fault armed in process 0 is validated but acts nowhere."""
    m = hm.HandleModel(oracle, no_schedule, 2, 1 << 20, sm_count=132, local=[0])
    sizes = memcpy_ref.ladder(m.bpp)
    v = (2 << 40) | (1 << 32) | (2 << 24) | 7  # issuer 1, target 0, size 1, word 7
    m.arm_measure(m.cea_fault, 1, v)
    got = m.ce_alltoall(op, 1)
    owned = {(0, 1)} if op == hm.OP_READ else {(1, 0)}
    assert set(got["cells"]) == owned and set(got["ranks"]) == {0}
    for key in owned:
        f = (1, 7, 0) if key == (1, 0) else None
        assert ce_cells(got)[key] == memcpy_direct(oracle, 2, m.bpp, op, *key, {}, f, 1)
        assert got["cells"][key]["bad_sizes"] == (0b10 if f else 0)
    m.arm_measure(m.cea_fault, 1, 0)
    m.arm_measure(m.cea_fault, 0, v)
    assert all(c["bad_sizes"] == 0 for c in m.ce_alltoall(op, 1)["cells"].values())
    m.arm_measure(m.cea_fault, 1, v + sizes[1] // 8)  # one word past its size, in the other process: refused here too
    assert m.ce_alltoall(op, 1) == hm.ERR_ARG and m.cea_calls == 2


def test_ce_alltoall_refusals_their_precedence_and_the_queue_limit_of_every_process(oracle):
    n = 3
    m = hm.HandleModel(oracle, no_schedule, n, 1 << 20, sm_count=132)
    sizes = memcpy_ref.ladder(m.bpp)
    m.max_connections[0] = 8  # 3 ranks on one device need 9 queues
    bad_fault = (3 << 48) | (1 << 40) | (2 << 32) | (1 << 24)
    m.arm_measure(m.cea_fault, 0, bad_fault)
    assert m.ce_alltoall(hm.OP_READ, 65) == hm.ERR_ARG    # reps first
    assert m.ce_alltoall(3, 2) == hm.ERR_ARG              # then the op
    assert m.ce_alltoall(hm.OP_READ, 2) == hm.ERR_ARG     # then the fault, before the queues
    for bad in ((1 << 40) | (1 << 32) | (1 << 24), ((n + 1) << 40) | (1 << 32) | (1 << 24),
                (1 << 40) | ((n + 1) << 32) | (1 << 24), (1 << 40) | (2 << 32) | ((len(sizes) + 1) << 24),
                (1 << 40) | (2 << 32) | (1 << 24) | sizes[0] // 8, (1 << 48) | (1 << 40) | (2 << 32) | (1 << 24)
                | sizes[0] // 8, (2 << 48) | (1 << 40) | (2 << 32) | (1 << 24) | 10_000_000, (1 << 40) | (2 << 32)):
        m.arm_measure(m.cea_fault, 0, bad)
        assert m.ce_alltoall(hm.OP_WRITE, 1) == hm.ERR_ARG, hex(bad)
    # a hold below timeout_ms / 2 names no word: accepted whatever its size
    m.arm_measure(m.cea_fault, 0, (2 << 48) | (1 << 40) | (2 << 32) | (1 << 24) | 9_999_999)
    assert m.ce_alltoall(hm.OP_WRITE, 1) == hm.ERR_UNSUPPORTED  # then the queues
    m.arm_measure(m.cea_fault, 0, 0)
    assert m.ce_alltoall(hm.OP_READ, 0) == hm.ERR_UNSUPPORTED
    assert m.cea_calls == 0 and m.area_down is None  # no refusal advances anything or builds the area
    m.max_connections[0] = 9  # need = limit runs
    got = m.ce_alltoall(hm.OP_READ, 0)
    assert got["call_seq"] == 1 and all(c["bad_words"] == [0] * len(sizes) for c in got["cells"].values())
    assert m.area_down == frozenset()
    # two processes of three ranks each: 18 queues; one process at 8 refuses both
    for limits, want in (({0: 32, 1: 8}, hm.ERR_UNSUPPORTED), ({0: 8, 1: 32}, hm.ERR_UNSUPPORTED),
                         ({0: 18, 1: 18}, None)):
        for me in (0, 1):
            mp = hm.HandleModel(oracle, no_schedule, 6, 5 << 20, sm_count=132, local=range(3 * me, 3 * me + 3))
            mp.max_connections.update(limits)
            got = mp.ce_alltoall(hm.OP_WRITE, 1)
            if want is None:
                assert got["call_seq"] == 1 and set(got["ranks"]) == set(mp.local)
                assert {ce_alltoall_ref.owner(hm.OP_WRITE, *c) for c in got["cells"]} == set(mp.local)
            else:
                assert got == want and mp.cea_calls == 0 and mp.area_down is None, (limits, me)
    # one rank per device, as a node of four GPUs opens them: 4 queues per device, which the default 8 allows
    m4 = hm.HandleModel(oracle, no_schedule, 4, 3 << 20, sm_count=132)
    m4.ordinal.update({g: g for g in range(4)})
    m4.max_connections[0] = 8
    assert m4.ce_alltoall(hm.OP_READ, 1)["call_seq"] == 1
    m4.ordinal.clear()  # all four on device 0: 16
    assert m4.ce_alltoall(hm.OP_READ, 1) == hm.ERR_UNSUPPORTED and m4.cea_calls == 1
    # two ranks on each of two devices need what one rank per device needs, twice
    m4 = hm.HandleModel(oracle, no_schedule, 4, 3 << 20, sm_count=132)
    m4.ordinal.update({0: 0, 1: 1, 2: 0, 3: 1})
    m4.max_connections[0] = 8
    assert m4.ce_alltoall(hm.OP_READ, 1)["call_seq"] == 1
    m4.ordinal[3] = 0
    assert m4.ce_alltoall(hm.OP_READ, 1) == hm.ERR_UNSUPPORTED and m4.cea_calls == 1


def test_max_connections_reads_the_variable_as_cdprobe_open_does():
    for value, want in ((None, 8), ("", 8), ("9", 9), ("32", 32), ("64", 32), ("0", 8), ("-4", 8), ("abc", 8),
                        ("12x", 12), (" 5", 5)):
        env = {} if value is None else {"CUDA_DEVICE_MAX_CONNECTIONS": value}
        assert hm.max_connections(env) == want, value


def test_ce_alltoall_down_rule_counters_and_the_sticky_area(oracle):
    """Any pair down stops every rank and reports every cell of a local rank, either way, as down; call_seq still
    advances and the area is built.  A pair down when the area was built keeps it off after the remap, while memcpy
    and the all-to-all skip only that cell.  Each measurement keeps its own counter."""
    n = 3
    m = hm.HandleModel(oracle, no_schedule, n, 1 << 20, sm_count=132)
    m.max_connections[0] = 32
    assert m.ce_alltoall(hm.OP_WRITE, 1)["call_seq"] == 1
    m.unmapped.add((2, 1))  # after the area: stops the call while down, not after the remap
    got = m.ce_alltoall(hm.OP_READ, 1)
    assert got["call_seq"] == 2 and got["ranks"] == {g: dict(measured=False, status=hm.ERR_STATE, blocks=0)
                                                     for g in range(n)}
    assert got["cells"] == {(g, j): dict(cell_measured=False, cell_status=hm.ERR_STATE)
                            for g in range(n) for j in range(n) if g != j}
    m.unmapped.discard((2, 1))
    assert all(r["measured"] for r in m.ce_alltoall(hm.OP_READ, 1)["ranks"].values())
    # only rank 0 local, two processes: its row, and the cells it issues or receives, are down
    m2 = hm.HandleModel(oracle, no_schedule, 2, 1 << 20, sm_count=132, local=[0])
    m2.unmapped.add((0, 1))
    got = m2.ce_alltoall(hm.OP_READ, 1)
    assert got["ranks"] == {0: dict(measured=False, status=hm.ERR_STATE, blocks=0)} and m2.area_down == {(0, 1)}
    assert set(got["cells"]) == {(0, 1), (1, 0)}
    m2.unmapped.clear()
    assert m2.ce_alltoall(hm.OP_WRITE, 1)["ranks"][0]["measured"] is False and m2.cea_calls == 2
    # counters: each its own
    m.alltoall(1)
    m.memcpy(hm.OP_READ, 1)
    m.memcpy(hm.OP_WRITE, 1)
    assert (m.cea_calls, m.a2a_calls, m.mc_calls) == (3, 1, 2)
    assert m.ce_alltoall(3, 1) == hm.ERR_ARG and m.ce_alltoall(hm.OP_READ, 2)["call_seq"] == 4
    assert (m.cea_calls, m.a2a_calls, m.mc_calls) == (4, 1, 2)


NVLS_TEXTS = {"reps": "reps must be at most 64",
              "mode": "the armed NVLS all-reduce fault has a mode above 1",
              "bits": "the armed NVLS all-reduce fault sets bits 32 to 47, which name nothing",
              "size": "the armed NVLS all-reduce fault names no size of this call",
              "word": "the armed NVLS all-reduce fault names no output word of its size",
              "other": "another process called cdprobe_allreduce_nvls with invalid arguments"}


def test_allreduce_nvls_refusals_in_their_order_with_their_texts(oracle):
    """Reps first, then the fault's mode, its unused bits, its size and its word; a refused call advances nothing."""
    m = hm.HandleModel(oracle, no_schedule, 3, 1 << 20, sm_count=132)
    sizes = bwcurve_ref.ladder(m.bpp)
    K = len(sizes)
    word_past = (K << 24) | sizes[-1] // 8
    for v, want in (((2 << 48) | (1 << 32) | ((K + 1) << 24) | word_past, "mode"),
                    ((1 << 63) | (1 << 24), "mode"),
                    ((1 << 48) | (1 << 32) | ((K + 1) << 24), "bits"),
                    ((1 << 47) | (1 << 24), "bits"),
                    (((K + 1) << 24) | 0xFFFFFF, "size"),
                    (5, "size"),
                    (word_past, "word"),
                    ((1 << 48) | (1 << 24) | sizes[0] // 8, "word")):
        m.arm_measure(m.nvls_fault, 0, v)
        assert m.allreduce_nvls(65) == NVLS_TEXTS["reps"], hex(v)
        assert m.allreduce_nvls(2) == NVLS_TEXTS[want], hex(v)
    assert m.nvls_calls == 0
    m.arm_measure(m.nvls_fault, 0, (1 << 48) | (K << 24) | (sizes[-1] // 8 - 1))  # the last word: accepted
    assert m.allreduce_nvls(2)["call_seq"] == 1
    m.arm_measure(m.nvls_fault, 0, 0)
    assert m.allreduce_nvls(0)["call_seq"] == 2 and m.allreduce_nvls(64)["call_seq"] == 3


def test_allreduce_nvls_a_bad_fault_in_another_process_refuses_with_its_own_text(oracle):
    sizes = bwcurve_ref.ladder(hm.HandleModel(oracle, no_schedule, 4, 3 << 20, sm_count=132).bpp)
    for me in (0, 1):
        m = hm.HandleModel(oracle, no_schedule, 4, 3 << 20, sm_count=132, local=range(2 * me, 2 * me + 2))
        m.arm_measure(m.nvls_fault, 1, (1 << 24) | sizes[0] // 8)  # process 1's: one word past size 0
        m.arm_measure(m.nvls_fault, 0, 1 << 24)                    # process 0's: word 0, valid
        assert m.allreduce_nvls(1, proc=me) == (NVLS_TEXTS["word"] if me == 1 else NVLS_TEXTS["other"])
        m.arm_measure(m.nvls_fault, 0, 2 << 48)                    # now both bad: each names its own
        assert m.allreduce_nvls(1, proc=me) == (NVLS_TEXTS["word"] if me == 1 else NVLS_TEXTS["mode"])
        m.arm_measure(m.nvls_fault, 1, 0)
        m.arm_measure(m.nvls_fault, 0, 0)
        got = m.allreduce_nvls(1, proc=me)
        assert got["call_seq"] == 1 and set(got["rows"]) == set(m.local)


def test_allreduce_nvls_runs_nothing_advances_only_its_own_counter_and_builds_nothing(oracle):
    """Every local row is unmeasured with CDPROBE_ERR_UNSUPPORTED, whether or not a pair is down, a word is corrupted
    or a valid fault is armed; no area is built and no other counter moves."""
    m = hm.HandleModel(oracle, no_schedule, 3, 1 << 20, sm_count=132)
    sizes = bwcurve_ref.ladder(m.bpp)
    want_rows = {g: dict(measured=False, status=hm.ERR_UNSUPPORTED) for g in range(3)}
    seq = 0
    for step in ("clean", "corrupt", "unmap", "fault", "remap"):
        if step == "corrupt":
            m.corrupt_word(1, 5, 1 << 9)
        elif step == "unmap":
            m.unmapped.add((2, 0))
        elif step == "fault":
            m.arm_measure(m.nvls_fault, 0, (1 << 48) | (len(sizes) << 24))
        elif step == "remap":
            m.unmapped.clear()
        seq += 1
        assert m.allreduce_nvls(1) == dict(call_seq=seq, sizes=sizes, rows=want_rows), step
    assert (m.ar_calls, m.ts_calls, m.ll_calls, m.ring_calls, m.push_calls, m.a2a_calls, m.mc_calls,
            m.cea_calls) == (0,) * 8
    assert m.area_down is None and all(v is None for v in m.ar_area_down.values())
    assert m.allreduce(1)["call_seq"] == 1 and m.nvls_calls == 5
    m1 = hm.HandleModel(oracle, no_schedule, 1, 1 << 20, sm_count=132)
    assert m1.allreduce_nvls(3)["rows"] == {0: dict(measured=False, status=hm.ERR_UNSUPPORTED)}


def test_allreduce_nvls_is_modelled_only_where_the_domain_cannot_form_a_multicast_object(oracle):
    """Ranks that share a device, or one rank whose one-device object the driver refuses: the call runs nothing.  One
    rank per device, or one rank the driver accepts, runs the kernel, which the model does not cover."""
    m = hm.HandleModel(oracle, no_schedule, 4, 3 << 20, sm_count=132)
    assert m.nvls_modelled()  # every rank on ordinal 0
    m.ordinal.update({0: 0, 1: 1, 2: 2, 3: 1})
    assert m.nvls_modelled()  # ranks 1 and 3 share a device
    m.ordinal[3] = 3
    assert not m.nvls_modelled()
    with pytest.raises(AssertionError):
        m.allreduce_nvls(1)
    assert m.nvls_calls == 0
    m1 = hm.HandleModel(oracle, no_schedule, 1, 1 << 20, sm_count=132)
    assert m1.nvls_modelled()
    m1.one_device_nvls_refused = False
    assert not m1.nvls_modelled()
