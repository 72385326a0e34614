"""Pins tests/handle_model.py against hand-built cases, without a GPU: the (S, X) of a slice with corrupted words, the
latency chase over overridden words, what a landing slot holds after a history of runs, unmaps and landing faults
(and so what cdprobe_diagnose must report on it), the counters and the unmapped-pair rule."""
import ctypes as C
import random

import numpy as np
import pytest

import handle_model as hm
import latency_ref
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
