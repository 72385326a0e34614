"""The word-level reference (tests/word_ref.py) against the C oracle and the diagnosis classifier, and the exact blind
spots of the probe's (S, X) checksum.  No GPU."""
import ctypes as C
import random

import numpy as np
import pytest

import word_ref as ref
from harness import c_tool

SEED = 0xCD5EED0000000001
INDICES = (0, 1, 2047, 2048, 1 << 32, (1 << 56) - 1)


# ---- the reference against the C oracle -------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [SEED, 0, (1 << 64) - 1, 0x0123456789ABCDEF])
def test_reference_words_equal_the_oracles(oracle, seed):
    L = oracle.lib()
    for rank in (0, 1, 7, 15):
        for k in INDICES:
            assert int(ref.src_words(seed, rank, k, 1)[0]) == L.cdoracle_src_word(seed, rank, k), (rank, k)
        run = ref.src_words(seed, rank, 2040, 16)  # a run across a granule boundary, vectorised
        assert [int(w) for w in run] == [L.cdoracle_src_word(seed, rank, 2040 + i) for i in range(16)]
    for src, dst, seq in ((0, 1, 1), (15, 0, 2), (3, 9, 20), (1, 1, (1 << 64) - 1)):
        salt = ref.write_salt(seed, src, dst, seq)
        assert salt == L.cdoracle_write_salt(seed, src, dst, seq)
        for k in INDICES:
            assert int(ref.write_words(salt, k, 1)[0]) == L.cdoracle_write_word(salt, k), (src, dst, seq, k)
    # wrap-around of salt + k
    salt = (1 << 64) - 3
    assert [int(w) for w in ref.write_words(salt, 0, 6)] == [L.cdoracle_write_word(salt, k) for k in range(6)]


def checksum(oracle, words):
    w = np.ascontiguousarray(words, dtype=np.uint64)
    s, x = C.c_uint64(), C.c_uint64()
    oracle.lib().cdoracle_checksum(w.ctypes.data_as(C.POINTER(C.c_uint64)), len(w), C.byref(s), C.byref(x))
    return s.value, x.value


@pytest.mark.parametrize("first,n", [(0, 2048), (4096, 5000), (12345, 3 * 2048 + 80)])
def test_reference_words_give_the_oracles_checksums(oracle, first, n):
    assert checksum(oracle, ref.src_words(SEED, 2, first, n)) == oracle.src_checksum(SEED, 2, first, n)
    salt = ref.write_salt(SEED, 1, 3, 17)
    if first == 0:
        assert checksum(oracle, ref.write_words(salt, 0, n)) == oracle.write_checksum(SEED, 1, 3, 17, n)


def test_inverses_recover_the_pattern_index():
    for rank in (0, 5, 15):
        x = ref.unsplitmix64(ref.src_words(SEED, rank, 0, 1 << 12)) ^ np.uint64(SEED)
        assert np.array_equal(x, np.arange(1 << 12, dtype=np.uint64) ^ np.uint64(rank << 56))
    for i, kk in enumerate(INDICES):
        w = ref.src_words(SEED, 3, kk, 1)
        assert int((ref.unsplitmix64(w) ^ np.uint64(SEED))[0]) == (3 << 56) ^ kk, i
    salt = ref.write_salt(SEED, 2, 0, 5)
    assert np.array_equal(ref.unwrite_word(ref.write_words(salt, 0, 4096)),
                          np.arange(4096, dtype=np.uint64) + np.uint64(salt))


# ---- the reference classifier against the C classifier the kernel compiles ------------------------------------
@pytest.fixture(scope="module")
def c_classify(tmp_path_factory):
    run = c_tool(tmp_path_factory, "diag_classify.cc", "-O1")
    return lambda cases: [tuple(r) for r in run(cases)]


def ref_answer(case):
    """(expected word k, kind, rank, word, run_seq) from the reference, for one line of diag_classify's input."""
    if case[0] == "read":
        _, seed, n_ranks, target, first, n_words, src_words, k, obs = case
        spec = ref.read_spec(seed, n_ranks, target, first, n_words, src_words)
    else:
        _, seed, n_ranks, issuer, target, run_seq, n_words, k, obs = case
        spec = ref.write_spec(seed, n_ranks, issuer, target, run_seq, n_words)
    kind, rank, word, seq = ref.classify(spec, [obs])
    return int(spec.expected(k, 1)[0]), int(kind[0]), int(rank[0]), int(word[0]), int(seq[0])


def random_read_cases(rng, count):
    cases, want = [], []
    for _ in range(count):
        seed = rng.getrandbits(64)
        n_ranks = rng.choice((1, 2, 3, 8, 16))
        target = rng.randrange(n_ranks)
        n_words = rng.choice((16, 2048, 6224, 1 << 17))
        n_slices = rng.choice((1, max(1, n_ranks - 1), n_ranks))
        src_words = n_slices * n_words
        first = rng.randrange(n_slices) * n_words
        k = rng.randrange(n_words)
        exp = int(ref.src_words(seed, target, first + k, 1)[0])
        pick = rng.randrange(8)
        if pick == 0:
            obs, w = 0, (ref.ZERO, -1, 0, 0)
        elif pick == 1:  # the target's word from elsewhere, the last index of the buffer included
            kp = rng.choice((0, src_words - 1, rng.randrange(src_words)))
            obs = int(ref.src_words(seed, target, kp, 1)[0])
            w = (ref.DISPLACED, target, kp, 0) if kp != first + k else None
        elif pick == 2:  # another rank's word; rank 15 when the domain has one
            r = n_ranks - 1 if rng.random() < 0.5 else rng.randrange(n_ranks)
            kp = rng.choice((0, src_words - 1, rng.randrange(src_words)))
            obs = int(ref.src_words(seed, r, kp, 1)[0])
            w = (ref.FOREIGN if r != target else ref.DISPLACED, r, kp, 0) if (r, kp) != (target, first + k) else None
        elif pick == 3:  # one past the source buffer
            obs, w = int(ref.src_words(seed, rng.randrange(n_ranks), src_words, 1)[0]), (ref.FLIP, -1, 0, 0)
        elif pick == 4:  # a rank outside the domain
            obs, w = int(ref.src_words(seed, rng.randrange(n_ranks, 256), rng.randrange(src_words), 1)[0]), \
                (ref.FLIP, -1, 0, 0)
        elif pick == 5:  # flipped bits, bit 63 included
            obs, w = exp ^ (rng.getrandbits(64) | 1 << 63), (ref.FLIP, -1, 0, 0)
        elif pick == 6:
            obs, w = exp ^ (1 << rng.randrange(64)), (ref.FLIP, -1, 0, 0)
        else:
            obs, w = rng.getrandbits(64), None
        cases.append(("read", seed, n_ranks, target, first, n_words, src_words, k, obs))
        want.append(w)
    return cases, want


def random_write_cases(rng, count):
    cases, want = [], []
    for _ in range(count):
        seed = rng.getrandbits(64)
        n_ranks = rng.choice((1, 2, 3, 8, 16))
        issuer, target = rng.randrange(n_ranks), rng.randrange(n_ranks)
        run_seq = rng.choice((1, 2, 5, 9, 10, 1000, rng.getrandbits(40) + 10))
        n_words = rng.choice((16, 2048, 6224, 1 << 17))
        k = rng.randrange(n_words)
        salt = ref.write_salt(seed, issuer, target, run_seq)
        exp = int(ref.write_words(salt, k, 1)[0])

        def ww(src, seq, kp):
            return int(ref.write_words(ref.write_salt(seed, src, target, seq), kp, 1)[0])

        kp = rng.choice((0, n_words - 1, rng.randrange(n_words)))
        pick = rng.randrange(9)
        if pick == 0:
            obs, w = 0, (ref.ZERO, -1, 0, 0)
        elif pick == 1:
            obs, w = ww(issuer, run_seq, kp), (ref.DISPLACED, issuer, kp, 0) if kp != k else None
        elif pick == 2:  # up to 8 runs back is STALE, 9 back is not traced
            d = rng.randrange(1, 10)
            if d < run_seq:
                obs = ww(issuer, run_seq - d, kp)
                w = (ref.STALE, issuer, kp, run_seq - d) if d <= 8 else (ref.FLIP, -1, 0, 0)
            else:
                obs, w = exp ^ 2, (ref.FLIP, -1, 0, 0)
        elif pick == 3:
            r = n_ranks - 1 if rng.random() < 0.5 else rng.randrange(n_ranks)
            obs = ww(r, run_seq, kp)
            w = (ref.FOREIGN, r, kp, 0) if r != issuer else (ref.DISPLACED, r, kp, 0) if kp != k else None
        elif pick == 4:  # one past the slot, from the current or a stale salt
            obs, w = ww(issuer, run_seq - rng.randrange(min(run_seq, 9)), n_words), (ref.FLIP, -1, 0, 0)
        elif pick == 5:
            obs, w = ww(issuer, run_seq - 9, kp) if run_seq > 9 else exp ^ 1, (ref.FLIP, -1, 0, 0)
        elif pick == 6:
            obs, w = exp ^ (rng.getrandbits(64) or 1), (ref.FLIP, -1, 0, 0)
        elif pick == 7:
            obs, w = exp ^ (1 << rng.randrange(64)), (ref.FLIP, -1, 0, 0)
        else:
            obs, w = rng.getrandbits(64), None
        cases.append(("write", seed, n_ranks, issuer, target, run_seq, n_words, k, obs))
        want.append(w)
    return cases, want


@pytest.mark.parametrize("op", ["read", "write"])
def test_reference_classifier_equals_the_c_classifier(c_classify, op):
    rng = random.Random(0xC1A55 + (op == "write"))
    cases, want = (random_read_cases if op == "read" else random_write_cases)(rng, 4000)
    got = c_classify(cases)
    seen = set()
    for c, g, w in zip(cases, got, want):
        r = ref_answer(c)
        assert r == g, (c, r, g)
        if w is not None:
            assert r[1:] == w, (c, r, w)
            seen.add(w[0])
    assert seen == {ref.FLIP, ref.ZERO, ref.DISPLACED, ref.FOREIGN} | ({ref.STALE} if op == "write" else set())


def test_classifier_boundaries(c_classify):
    """The edges named in the spec, each against both classifiers: rank 15, 8 runs back against 9, the last index
    of the region against one past it."""
    n_words, src_words = 4096, 15 * 4096
    cases = []
    for kp in (src_words - 1, src_words):
        cases.append(("read", SEED, 16, 5, 2 * n_words, n_words, src_words, 3, int(ref.src_words(SEED, 15, kp, 1)[0])))
    cases.append(("read", SEED, 15, 5, 0, n_words, src_words, 3, int(ref.src_words(SEED, 15, 0, 1)[0])))
    for d in (8, 9):
        for kp in (n_words - 1, n_words):
            salt = ref.write_salt(SEED, 3, 9, 20 - d)
            cases.append(("write", SEED, 16, 3, 9, 20, n_words, 5, int(ref.write_words(salt, kp, 1)[0])))
    salt = ref.write_salt(SEED, 15, 9, 20)
    cases.append(("write", SEED, 16, 3, 9, 20, n_words, 5, int(ref.write_words(salt, n_words - 1, 1)[0])))
    got = c_classify(cases)
    want = [(ref.FOREIGN, 15, src_words - 1, 0), (ref.FLIP, -1, 0, 0), (ref.FLIP, -1, 0, 0),
            (ref.STALE, 3, n_words - 1, 12), (ref.FLIP, -1, 0, 0), (ref.FLIP, -1, 0, 0), (ref.FLIP, -1, 0, 0),
            (ref.FOREIGN, 15, n_words - 1, 0)]
    for c, g, w in zip(cases, got, want):
        assert ref_answer(c) == g and g[1:] == w, (c, g, w)


def test_expected_report_of_a_handmade_region():
    spec = ref.read_spec(SEED, 2, 1, 0, 3 * 2048, 3 * 2048)
    obs = spec.expected().copy()
    obs[5] = 0
    obs[2048] ^= np.uint64(1 << 63 | 1)
    obs[3 * 2048 - 1] = ref.src_words(SEED, 0, 7, 1)[0]
    rep = ref.expected_report(spec, obs)
    assert (rep["bad_words"], rep["bad_granules"], rep["first_bad"], rep["last_bad"]) == (3, 3, 40, 8 * (3 * 2048 - 1))
    assert rep["kind_count"] == [1, 1, 0, 0, 1] and rep["zero_words"] == 1
    assert rep["bit_flips"] == [1] + [0] * 62 + [1]
    assert [(s["offset"], s["kind"], s["rank"], s["word"]) for s in rep["sample"]] == [
        (40, ref.ZERO, -1, 0), (8 * 2048, ref.FLIP, -1, 0), (8 * (3 * 2048 - 1), ref.FOREIGN, 0, 7)]
    clean = ref.expected_report(spec, spec.expected())
    assert (clean["bad_words"], clean["first_bad"], clean["last_bad"], clean["sample"]) == (0, ref.U64_MAX, 0, [])


# ---- what (S, X) cannot see ----------------------------------------------------------------------------------------
G = ref.GRANULE_WORDS


def swapped(words, a, b, n):
    w = words.copy()
    w[a:a + n], w[b:b + n] = words[b:b + n], words[a:a + n]
    return w


def test_checksum_blind_spots_are_exactly_the_fold6_classes(oracle):
    """S is order-free; X is order-free inside a 16 KiB granule and only tells granules apart by fold6(g), which has
    64 values.  So a placement bug that keeps words inside their granule, or swaps two granules of one fold6 class,
    leaves (S, X) as it was.  Only a word-for-word diff (cdprobe_diagnose) sees it."""
    words = ref.src_words(SEED, 0, 0, 70 * G)
    clean = checksum(oracle, words)
    assert clean == oracle.src_checksum(SEED, 0, 0, 70 * G)
    # unchanged: two words of one granule, the two 8 KiB units of a granule, granules of one fold6 class
    assert ref.fold6(1) == ref.fold6(64) == 1
    for w in (swapped(words, 3 * G + 5, 3 * G + 2000, 1), swapped(words, 7 * G, 7 * G + G // 2, G // 2),
              swapped(words, 1 * G, 64 * G, G)):
        assert not np.array_equal(w, words) and checksum(oracle, w) == clean
    # X changes, S does not: granules of different fold6 classes
    for a, b in ((0, 1), (1, 2)):
        assert ref.fold6(a) != ref.fold6(b)
        s, x = checksum(oracle, swapped(words, a * G, b * G, G))
        assert s == clean[0] and x != clean[1], (a, b)
    # a word replaced by a copy of another changes S
    w = words.copy()
    w[10] = w[11]
    assert checksum(oracle, w)[0] != clean[0]
    # a 1 GiB slice: 65536 granules in 64 fold6 classes of 1024 each
    classes = np.bincount([ref.fold6(g) for g in range((1 << 30) // (8 * G))], minlength=64)
    assert len(classes) == 64 and (classes == 1024).all()
