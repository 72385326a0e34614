"""The rep-record fold of measure.cc (summarize, ladder_times, bw_times, bw_summarize), copied verbatim and compiled for
the host (tests/rep_times.py), against a plain restatement of each, on records built by hand at the places a fold goes
wrong: a slow warm-up rep, releases that differ from rep to rep, every rep count's median, the all-to-all's block scale,
ties in the half-rate size, an aborted kernel, a timed-out rep, nanosecond counts past float32's 24 bits, and a bad
checksum in the warm-up only.  Every published ns_min / ns_median / ns_max, peak_gbps and half_bytes of bwcurve, the
all-reduces, the all-to-all, memcpy and the CE all-to-all passes through these functions.

Each deliberate error of rep_times.MUTATIONS must make the cases CAUGHT names fail."""
import random

import pytest

import rep_times as rt
from harness import header_values

SIZES = [4096 << k for k in range(6)]


@pytest.fixture(scope="module")
def fold(tmp_path_factory):
    return rt.Fold(rt.build(tmp_path_factory.mktemp("rep_times")))


def records(sizes, reps, rel, dur, sums=None):
    """A BwScratch record dict: rep r of size k released at rel(k, r) and lasting dur(k, r) ns; (S, X) from sums(k, r)
    or (0, 0)."""
    b = {"t_rel": [[rel(k, r) for r in range(reps + 1)] for k in range(len(sizes))]}
    b["t_end"] = [[b["t_rel"][k][r] + dur(k, r) for r in range(reps + 1)] for k in range(len(sizes))]
    if sums is not None:
        b["sum"] = [[sums(k, r)[0] for r in range(reps + 1)] for k in range(len(sizes))]
        b["xr"] = [[sums(k, r)[1] for r in range(reps + 1)] for k in range(len(sizes))]
    return b


def pairs_bw_times(fold, b, sizes, reps, scale):
    return [(fold.bw_times(b, sizes, reps, scale), rt.bw_times(b, sizes, reps, scale))]


# ---- the cases: each returns [(what the copy gave, what the restatement says)] --------------------------------------
def case_warmup(fold):
    """Rep 0 takes 1000 times as long as any timed rep: it reaches no min, median or max."""
    out = []
    for reps in (1, 2, 3, 8):
        b = records(SIZES, reps, lambda k, r: 10**9 + 10**6 * (k * 70 + r),
                    lambda k, r: 1000 * (2000 + 31 * k + 7 * r) if r == 0 else 2000 + 31 * k + 7 * r)
        got = fold.bw_times(b, SIZES, reps, 1.0)
        assert max(got[1]["ns_max"]) < 10**5, got  # the warm-up never shows
        out += [(got, rt.bw_times(b, SIZES, reps, 1.0))]
        ns = [2_000_000] + [1000 + 13 * r for r in range(1, reps + 1)]
        got = fold.summarize(ns, [0] * (reps + 1), [0] * (reps + 1), reps, 1, 0)
        assert got["ns_max"] < 10**4, got
        out += [(got, rt.summarize(ns, [0] * (reps + 1), [0] * (reps + 1), reps, 1, 0))]
    return out


def case_own_release(fold):
    """Every rep is released at its own time, far from the rep before's, and lasts a distinct time: a window opened at
    another rep's release shows."""
    out = []
    for reps in (1, 2, 5, 64):
        b = records(SIZES, reps, lambda k, r: 5 * 10**9 + 10**6 * (k * 70 + r) + 977 * r * r,
                    lambda k, r: 3000 + 101 * k + 37 * ((r * 7) % 11))
        out += pairs_bw_times(fold, b, SIZES, reps, 1.0)
    return out


def case_median_every_reps(fold):
    """For every reps in 1 .. 64, the median is element reps // 2 of the sorted timed reps, through bw_times, ladder_times
    and summarize; the reps come in a scrambled order so that a sort that is missing shows too."""
    out = []
    for reps in range(1, 65):
        perm = random.Random(reps).sample(range(reps), reps)
        b = records(SIZES[:2], reps, lambda k, r: 10**7 * (r + 1), lambda k, r: 1000 + 64 * perm[r - 1] + k if r else 9)
        out += pairs_bw_times(fold, b, SIZES[:2], reps, 1.0)
        ns = [[2000.0 + 32 * perm[r] + 8 * k for r in range(reps)] for k in range(len(SIZES))]
        out += [(fold.ladder_times(ns, SIZES, reps, 1.0), rt.ladder_times(ns, SIZES, reps, 1.0))]
        t = [5] + [700 + 3 * perm[r] for r in range(reps)]
        out += [(fold.summarize(t, [0] * (reps + 1), [0] * (reps + 1), reps, 1, 0),
                 rt.summarize(t, [0] * (reps + 1), [0] * (reps + 1), reps, 1, 0))]
    return out


def case_block_scale(fold):
    """The all-to-all's rate is blocks x size / median: peak_gbps and half_bytes follow the scale, and the times do
    not."""
    out = []
    # a ladder whose rate keeps rising: half_bytes moves with the medians, not the scale, but peak scales by blocks
    b = records(SIZES, 3, lambda k, r: 10**8 * (k + 1) + 10**5 * r, lambda k, r: 4000 + 500 * k + r)
    for blocks in (1, 2, 3, 7, 15):
        got = fold.bw_times(b, SIZES, 3, float(blocks))
        want = rt.bw_times(b, SIZES, 3, float(blocks))
        assert got[1]["peak_gbps"] == rt.f32(blocks * SIZES[-1] / got[1]["ns_median"][-1]), got
        out += [(got, want)]
    return out


def case_half_ties(fold):
    """half_bytes is the first size whose rate reaches half the peak: a rate exactly at peak / 2, and equal rates at
    two sizes, take the smaller size."""
    out = []
    for meds, half in (([1000, 1000, 1000], 8192), ([1000, 2000, 2000], 4096), ([4000, 1000, 1000], 8192),
                       ([1000, 1000, 4000], 4096)):
        ns = [[float(m)] for m in meds]
        got = fold.ladder_times(ns, SIZES[:3], 1, 1.0)
        assert got["half_bytes"] == half, (meds, got)
        out += [(got, rt.ladder_times(ns, SIZES[:3], 1, 1.0))]
    return out


def case_abort(fold):
    """An aborted kernel: TIMEOUT, measured, and no times at all, whatever its records hold; bw_summarize adds no
    checks."""
    b = records(SIZES, 4, lambda k, r: 10**6 * (k * 5 + r), lambda k, r: 100 + k + r, lambda k, r: (1, 2))
    b["abort"] = 1
    got = fold.bw_times(b, SIZES, 4, 2.0)
    assert got == (False, dict(got[1], status=rt.ERR_TIMEOUT, measured=1)) and not any(got[1]["ns_max"])
    return [(got, rt.bw_times(b, SIZES, 4, 2.0)),
            (fold.bw_summarize(b, [(1, 2)] * len(SIZES), SIZES, 4), rt.bw_summarize(b, [(1, 2)] * len(SIZES), SIZES, 4))]


def case_timeout_rep(fold):
    """A TIMEOUT rep ends the digest with its own word and leaves no times; a rep after it counts for nothing; another
    non-zero status is kept, and a digest other than want is INTEGRITY."""
    out = []
    T = rt.ERR_TIMEOUT
    for status, want in (([0, 0, T, 0, 0], 0x1 ^ 0x2 ^ 0x4), ([T, 0, 0, 0, 0], 0x1), ([0, 0, 0, 0, T], 0x1F),
                         ([0, -4, 0, 0, 0], 0x1F), ([0, -4, 0, 0, 0], 0), ([0, 0, 0, 0, 0], 0x1F)):
        args = ([10, 20, 30, 40, 50], [1, 2, 4, 8, 16], status, 4, 1, want)
        got = fold.summarize(*args)
        out += [(got, rt.summarize(*args))]
    assert out[0][0]["digest"] == 0x7 and out[0][0]["status"] == T and out[0][0]["ns_max"] == 0.0
    return out


def case_float_past_2_24(fold):
    """Nanosecond counts at and past 2^24 round to float32 once, to nearest-even, in bw_times and in summarize."""
    big = [1 << 24, (1 << 24) + 1, (1 << 24) + 3, (1 << 30) + 65, (1 << 40) + (1 << 16), (1 << 40) + (1 << 16) + 1,
           (1 << 24) - 1]
    b = {"t_rel": [[7 * 10**9 + 10**12 * r for r in range(len(big) + 1)]]}
    b["t_end"] = [[t + ([5] + big)[r] for r, t in enumerate(b["t_rel"][0])]]
    got = fold.bw_times(b, SIZES[:1], len(big), 1.0)
    assert got[1]["ns_max"] == [float((1 << 40) + (1 << 17))] and got[1]["ns_min"] == [float((1 << 24) - 1)], got
    out = [(got, rt.bw_times(b, SIZES[:1], len(big), 1.0))]
    for per_rep in (1, 3, 1024):
        args = ([5] + big, [0] * (len(big) + 1), [0] * (len(big) + 1), len(big), per_rep, 0)
        out += [(fold.summarize(*args), rt.summarize(*args))]
    return out


def case_bad_warmup(fold):
    """A size whose warm-up rep alone read a wrong (S, X) is bad; a wrong (S, X) in a timed rep is too; the last timed
    rep's (S, X) is the one reported."""
    out = []
    want = [(1000 + k, 2000 + k) for k in range(len(SIZES))]
    for bad in ({(1, 0)}, {(0, 0), (3, 2)}, {(5, 3)}, set()):
        b = records(SIZES, 3, lambda k, r: 10**6 * (k * 5 + r), lambda k, r: 500 + k + r,
                    lambda k, r: (want[k][0] + ((k, r) in bad), want[k][1]))
        got = fold.bw_summarize(b, want, SIZES, 3)
        assert got["bad_sizes"] == sum(1 << k for k in {k for k, _ in bad}), (bad, got)
        out += [(got, rt.bw_summarize(b, want, SIZES, 3))]
    return out


def case_random(fold):
    """Seeded random records of every shape: ladder lengths 1 .. 24, reps 1 .. 64, windows of 1 ns to 10 ms, the
    all-to-all's scales, (S, X) that are mostly right."""
    rng = random.Random(0xF01D)
    out = []
    for _ in range(150):
        n, reps, scale = rng.randint(1, 24), rng.randint(1, 64), float(rng.choice([1, 1, 2, 3, 15]))
        sizes = [4096 << k for k in range(n)]
        want = [(rng.getrandbits(64), rng.getrandbits(64)) for _ in range(n)]
        b = records(sizes, reps, lambda k, r: rng.getrandbits(50), lambda k, r: rng.randint(1, 10**7),
                    lambda k, r: want[k] if rng.random() < 0.97 else (rng.getrandbits(64), want[k][1]))
        out += pairs_bw_times(fold, b, sizes, reps, scale)
        out += [(fold.bw_summarize(b, want, sizes, reps), rt.bw_summarize(b, want, sizes, reps))]
        ns = [rng.getrandbits(34) for _ in range(reps + 1)]
        dig = [rng.getrandbits(64) for _ in range(reps + 1)]
        st = [rng.choice([0] * 20 + [rt.ERR_TIMEOUT, -4]) for _ in range(reps + 1)]
        w = 0
        for d in dig:
            w ^= d
        per = rng.choice([1, 2, 1024, 65536])
        out += [(fold.summarize(ns, dig, st, reps, per, w), rt.summarize(ns, dig, st, reps, per, w))]
    return out


CASES = {name[5:]: fn for name, fn in dict(globals()).items() if name.startswith("case_")}
# the cases each deliberate error must fail
CAUGHT = {"bw_times_previous_rel": ["own_release", "random"],
          "warmup_in_stats": ["warmup", "median_every_reps"],
          "median_low": ["median_every_reps"]}


def test_error_codes_are_the_headers(tmp_path):
    assert header_values(tmp_path, "CDPROBE_ERR_TIMEOUT", "CDPROBE_ERR_INTEGRITY") == [rt.ERR_TIMEOUT & (2**64 - 1),
                                                                                       rt.ERR_INTEGRITY & (2**64 - 1)]


def test_each_function_is_copied_whole():
    """Each template is found once and reaches the copy unchanged; a second definition would fail the extraction."""
    funcs = rt.extract()
    text = rt.generate()
    for name in rt.FUNCTIONS:
        assert funcs[name] in text and funcs[name].rstrip().endswith("}")
    with pytest.raises(AssertionError):
        rt.extract(open(rt.MEASURE).read() + funcs["bw_times"])


@pytest.mark.parametrize("case", sorted(CASES))
def test_fold_equals_restatement(fold, case):
    for i, (got, want) in enumerate(CASES[case](fold)):
        assert got == want, (case, i)


@pytest.mark.parametrize("mutation", sorted(rt.MUTATIONS))
def test_each_mutation_is_seen(tmp_path, mutation):
    """A case sees a mutation when some pair differs, or when one of its own bounds fails first."""
    bad = rt.Fold(rt.build(tmp_path, mutation))
    for case in CAUGHT[mutation]:
        try:
            seen = any(got != want for got, want in CASES[case](bad))
        except AssertionError:
            seen = True
        assert seen, (mutation, case)
