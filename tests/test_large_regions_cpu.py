"""The streaming references of tests/large_ref.py pinned to the dense ones, and the plan at the byte offsets where
32-bit arithmetic breaks: 2^31, 2^32 and the plan's ceiling of 16 GiB per pair.

The plan's placement (src_off, land_off, alloc_bytes, every cell_offset and memcpy_cell) and the size ladders are read
from plan.cc and probe_types.h compiled on the host, next to cdprobe_plan, and compared with a restatement from the
oracle's plan and the allocation rules (DESIGN §5: a 2 MiB control granule, then the source buffer and the landing
slots, each rounded up to the 2 MiB VMM granule)."""
import random
import subprocess

import numpy as np
import pytest

import allreduce_ref
import bwcurve_ref
import large_ref
import memcpy_ref
import word_ref as ref
from kernel_tools import CSRC

SEED = 0xCD5EED0000000001
GIB = 1 << 30
VMM = 2 << 20
MODE_SLICED, MODE_FULL = 1, 2
LOCAL_DIAG = 0x04
ERR_ARG = -2
OP_READ, OP_WRITE = 1, 2
MAX_BPP = 16 * GIB
EDGE_BPPS = [(1 << 31) - 128, 1 << 31, (1 << 31) + 128, (1 << 32) - 128, 1 << 32, (1 << 32) + 8192 + 128, MAX_BPP]
G = ref.GRANULE_WORDS


# ---- prefix_sums against the oracle ------------------------------------------------------------------------------
def ladder_with_tails(nbytes):
    """The ladder of nbytes, with 4096 and 8192 even where the region is shorter than the ladder's first size."""
    return sorted({s for s in bwcurve_ref.ladder(nbytes) + [4096, 8192] if s <= nbytes})


@pytest.mark.parametrize("nbytes", [128, 4096 - 128, 16384 + 640, (3 << 20) + 8192 + 128])
@pytest.mark.parametrize("first_word", [0, 2049, 5 * G + 777])
def test_prefix_sums_equal_the_oracle(oracle, nbytes, first_word, monkeypatch):
    # chunks of 3 granules and a bit, so that the 3 MiB region crosses many chunk edges inside granules and sizes
    monkeypatch.setattr(large_ref, "CHUNK_WORDS", 3 * G + 640)
    sizes = ladder_with_tails(nbytes)
    for rank in (0, 5):
        got = large_ref.prefix_sums(large_ref.src_fn(SEED, rank, first_word), nbytes // 8, sizes)
        assert got == [oracle.src_checksum(SEED, rank, first_word, s // 8) for s in sizes], rank
    got = large_ref.prefix_sums(large_ref.write_fn(SEED, 3, 1, 9), nbytes // 8, sizes)
    assert got == [oracle.write_checksum(SEED, 3, 1, 9, s // 8) for s in sizes]


def test_prefix_sums_at_the_default_chunk_cross_a_chunk_edge(oracle):
    nbytes = 8 * large_ref.CHUNK_WORDS + 8192 + 128
    sizes = bwcurve_ref.ladder(nbytes)
    assert sizes[-2] == 8 * large_ref.CHUNK_WORDS
    got = large_ref.prefix_sums(large_ref.src_fn(SEED, 2, 3), nbytes // 8, sizes)
    assert got[-2:] == [oracle.src_checksum(SEED, 2, 3, s // 8) for s in sizes[-2:]]
    assert got[:3] == [oracle.src_checksum(SEED, 2, 3, s // 8) for s in sizes[:3]]


def test_prefix_sums_refuse_a_size_past_the_region():
    with pytest.raises(AssertionError):
        large_ref.prefix_sums(large_ref.src_fn(SEED, 0), 16, [136])


# ---- allreduce_sums against allreduce_ref ------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3, 16])
def test_allreduce_sums_equal_the_dense_reference(n, monkeypatch):
    monkeypatch.setattr(large_ref, "CHUNK_WORDS", 5 * G + 8)
    bpp = (1 << 20) + 5 * 1024 + 128
    sizes = tuple(allreduce_ref.ladder(bpp))
    got = large_ref.allreduce_sums(SEED, n, sizes)
    assert [(g.sum, g.xr) for g in got] == list(allreduce_ref.expected(SEED, n, sizes))
    assert all(g.bad_words == 0 and g.first_bad == large_ref.U64_MAX for g in got)
    clean = allreduce_ref.output_words(SEED, n, bpp // 8)
    for rank, word, mask in ((n - 1, 5, 1 << 17), (0, 40000, 1 << 63), (n // 2, bpp // 8 - 1, 0xFF00)):
        got = large_ref.allreduce_sums(SEED, n, sizes, corrupt=(rank, word, mask))
        assert [(g.sum, g.xr) for g in got] == allreduce_ref.expected_corrupted(SEED, n, sizes, rank, word, mask)
        bad = allreduce_ref.output_words(SEED, n, bpp // 8)
        orig = int(ref.src_words(SEED, rank, word, 1)[0])
        bad[word] = np.uint64((int(bad[word]) - orig + (orig ^ mask)) % (1 << 64))
        for g, s in zip(got, sizes):
            diff = np.flatnonzero(bad[:s // 8] != clean[:s // 8])
            assert (g.bad_words, g.first_bad) == (len(diff), 8 * int(diff[0]) if len(diff) else large_ref.U64_MAX), s


# ---- sparse_report against word_ref.expected_report --------------------------------------------------------------
def fault_words(spec, rng, idx, kinds, other_ranks):
    """(k, observed) for every k of idx, cycling through `kinds`."""
    exp = spec.expected()
    out = []
    for m, k in enumerate(idx):
        kind, e = kinds[m % len(kinds)], int(exp[k])
        if kind == "flip":
            v = e ^ rng.choice((1 << rng.randrange(64), rng.getrandbits(64) | 1))
        elif kind == "zero":
            v = 0
        elif kind == "same":  # written back as it was: not a bad word
            v = e
        elif spec.is_write:
            seq, w = {"displaced": (spec.run_seq, spec.issuer), "stale": (spec.run_seq - rng.randint(1, 8), spec.issuer),
                      "foreign": (spec.run_seq, rng.choice(other_ranks))}[kind]
            kp = rng.randrange(spec.n_words)
            kp = kp if (kind != "displaced" or kp != k) else (k + 1) % spec.n_words
            v = int(ref.write_words(ref.write_salt(SEED, w, spec.target, seq), kp, 1)[0])
        elif kind == "displaced":
            kp = rng.randrange(spec.src_words)
            kp = kp if kp != spec.first_word + k else (kp + 1) % spec.src_words
            v = int(ref.src_words(SEED, spec.target, kp, 1)[0])
        else:  # foreign
            v = int(ref.src_words(SEED, rng.choice(other_ranks), rng.randrange(spec.src_words), 1)[0])
        out.append((k, v))
    return out


def observed(spec, faults):
    w = spec.expected().copy()
    for k, v in faults:
        w[k] = np.uint64(v)
    return w


READ_KINDS = ["flip", "zero", "displaced", "foreign", "same"]
WRITE_KINDS = ["flip", "zero", "displaced", "stale", "foreign", "same"]


@pytest.mark.parametrize("trial", range(6))
@pytest.mark.parametrize("op", ["read", "write"])
def test_sparse_report_equals_the_dense_report(op, trial):
    rng = random.Random(f"{op}{trial}")
    n_words = rng.choice([16, 3 * G + 80, 5 * G])
    if op == "read":
        spec = ref.read_spec(SEED, 4, 2, rng.choice([0, n_words]), n_words, 3 * n_words)
        kinds = list(READ_KINDS)
    else:
        spec = ref.write_spec(SEED, 4, 1, 3, 12, n_words)
        kinds = list(WRITE_KINDS)
    rng.shuffle(kinds)
    count = rng.choice([12, 17, 40]) if n_words > 16 else rng.choice([12, 16])
    idx = sorted(set(rng.sample(range(n_words), min(count, n_words) - 1)) | {n_words - 1})
    faults = fault_words(spec, rng, idx, kinds, (0, 1, 3) if op == "read" else (0, 2))
    if n_words >= 2 * G:  # a whole granule, every word flipped, on top
        faults += [(k, int(spec.expected(k, 1)[0]) ^ 1 << (k % 64)) for k in range(G, 2 * G)]
    rng.shuffle(faults)
    want = ref.expected_report(spec, observed(spec, faults))
    got = large_ref.sparse_report(spec, faults)
    assert got == want
    present = {c for c in range(5) if want["kind_count"][c]}
    assert present == set(range(5)) - ({ref.STALE} if op == "read" else set()) or n_words == 16


def test_sparse_report_of_a_clean_region_and_of_a_later_pair_for_the_same_word():
    spec = ref.read_spec(SEED, 1, 0, 0, 1 << 29, 1 << 29)  # 4 GiB, never built
    e = int(large_ref._expected_at(spec, np.array([(1 << 29) - 1], dtype=np.uint64))[0])
    assert e == int(ref.src_words(SEED, 0, (1 << 29) - 1, 1)[0])
    clean = large_ref.sparse_report(spec, [((1 << 29) - 1, e)])
    assert clean["bad_words"] == 0 and clean["first_bad"] == large_ref.U64_MAX and clean["sample"] == []
    rep = large_ref.sparse_report(spec, [((1 << 29) - 1, 0), ((1 << 29) - 1, e ^ 4), (1 << 28, 0)])
    assert rep["bad_words"] == 2 and rep["first_bad"] == 1 << 31 and rep["last_bad"] == (1 << 32) - 8
    assert rep["kind_count"] == [1, 1, 0, 0, 0] and rep["bit_flips"][2] == 1 and rep["bad_granules"] == 2
    with pytest.raises(AssertionError):
        large_ref.sparse_report(spec, [(1 << 29, 0)])


# ---- the plan past 2^31 and 2^32, and its ceiling -----------------------------------------------------------------
HARNESS = r"""
#include <stdio.h>
#include "plan.h"
using namespace cdp;
int main() {
  unsigned n, mode, flags;
  unsigned long long bytes;
  while (scanf("%u %llu %u %u", &n, &bytes, &mode, &flags) == 4) {
    Plan p;
    const int rc = make_plan(n, bytes, mode, flags, &p);
    printf("%d", rc);
    if (rc == CDPROBE_OK) {
      printf(" %u %u %u %u %u %llu %llu %llu %llu %llu %llu", p.n, p.rounds, p.n_slots, p.n_slices, p.diag_slot,
             (unsigned long long)p.bpp, (unsigned long long)p.src_bytes, (unsigned long long)p.land_bytes,
             (unsigned long long)p.src_off, (unsigned long long)p.land_off, (unsigned long long)p.alloc_bytes);
      for (unsigned op = 1; op <= 2; ++op)
        for (unsigned i = 0; i < n; ++i)
          for (unsigned j = 0; j < n; ++j) {
            printf(" %llu", (unsigned long long)cell_offset(p, op, i, j));
            const MemcpyCell c = memcpy_cell(p, op, i, j);
            printf(" %u %llu %llu %u %llu", c.src_rank, (unsigned long long)c.src_off,
                   (unsigned long long)c.first_word, c.dst_rank, (unsigned long long)c.dst_off);
          }
      uint64_t size[kBwMaxSizes];
      const uint32_t k = bwcurve_ladder(p.bpp, size);
      printf(" %u %u", k, ll_ladder(p.bpp, size));
      for (uint32_t q = 0; q < k; ++q) printf(" %llu", (unsigned long long)size[q]);
    }
    printf("\n");
  }
}
"""


@pytest.fixture(scope="module")
def host_plan(tmp_path_factory):
    """plan(n, bytes, mode, flags) -> the Plan of plan.cc compiled for the host, with every cell's offsets and memcpy
    cell and the ladders of its bytes_per_pair, or the error code."""
    d = tmp_path_factory.mktemp("plan")
    exe = d / "plan"
    (d / "main.cc").write_text(HARNESS)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", CSRC, str(d / "main.cc"), f"{CSRC}/plan.cc", "-o", str(exe)],
                   check=True)

    def plan(queries):
        inp = "".join(f"{n} {b} {m} {f}\n" for n, b, m, f in queries)
        lines = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout.splitlines()
        out = []
        for (n, _, _, _), line in zip(queries, lines):
            v = [int(x) for x in line.split()]
            if v[0] != 0:
                out.append(v[0])
                continue
            keys = "n rounds n_slots n_slices diag_slot bpp src_bytes land_bytes src_off land_off alloc_bytes".split()
            p = dict(zip(keys, v[1:12]))
            it = iter(v[12:])
            p["cells"] = {(op, i, j): (next(it), tuple(next(it) for _ in range(5)))
                          for op in (1, 2) for i in range(n) for j in range(n)}
            k, p["ll_sizes"] = next(it), next(it)
            p["ladder"] = [next(it) for _ in range(k)]
            out.append(p)
        assert len(out) == len(queries)
        return out

    return plan


def round_up(v, a):
    return -(-v // a) * a


def config_bytes(n, bpp, mode):
    """The config bytes whose plan has this bytes_per_pair: bpp per peer in sliced mode, with a remainder the plan
    rounds away."""
    peers = max(n - 1, 1)
    return bpp * peers + 127 * peers if mode == MODE_SLICED else bpp + 127


CASES = [(n, bpp, mode, flags) for bpp in EDGE_BPPS for mode in (MODE_SLICED, MODE_FULL) for n in (1, 2, 3, 16)
         for flags in (0, LOCAL_DIAG)]


def test_the_plan_agrees_with_the_oracle_past_2_31_and_2_32_up_to_16_gib(pkg, oracle, host_plan):
    queries = [(n, config_bytes(n, bpp, mode), mode, flags) for n, bpp, mode, flags in CASES]
    for (n, bpp, mode, flags), q, hp in zip(CASES, queries, host_plan(queries)):
        ctx = (n, bpp, mode, flags)
        diag = bool(flags & LOCAL_DIAG) or n == 1
        op_ = oracle.plan(n, q[1], mode, diag)
        lp = pkg.plan(n, q[1], mode, flags)
        for f in ("n", "rounds", "n_slots", "n_slices", "bytes_per_pair", "src_bytes", "land_bytes"):
            assert getattr(lp, f) == getattr(op_, f), (ctx, f)
        assert lp.bytes_per_pair == bpp and lp.abi == 2, ctx
        assert [list(r) for r in lp.partner] == [list(r) for r in op_.partner], ctx
        # the host build of the same plan, and where everything lies in a rank's allocation
        assert (hp["n"], hp["rounds"], hp["n_slots"], hp["n_slices"], hp["bpp"], hp["src_bytes"], hp["land_bytes"]) == \
            (lp.n, lp.rounds, lp.n_slots, lp.n_slices, bpp, lp.src_bytes, lp.land_bytes), ctx
        land_off = VMM + round_up(op_.src_bytes, VMM)
        assert (hp["src_off"], hp["land_off"], hp["alloc_bytes"], hp["diag_slot"]) == \
            (VMM, land_off, land_off + round_up(op_.land_bytes, VMM), n - 1), ctx
        for i in range(n):
            for j in range(n):
                if i == j and not diag:
                    continue
                slot = n - 1 if i == j else oracle.lib().cdoracle_slot(i, j)
                assert hp["cells"][(OP_READ, i, j)][0] == VMM + (0 if mode == MODE_FULL else slot) * bpp, (ctx, i, j)
                assert hp["cells"][(OP_WRITE, i, j)][0] == land_off + slot * bpp, (ctx, i, j)
                for op in (OP_READ, OP_WRITE):
                    c = memcpy_ref.cell(n, bpp, mode, op, i, j)
                    assert hp["cells"][(op, i, j)][1] == (c["src_rank"], VMM + c["src_off"], c["first_word"],
                                                          c["dst_rank"], c["dst_off"]), (ctx, op, i, j)
        assert hp["ladder"] == bwcurve_ref.ladder(bpp), ctx
        assert hp["ll_sizes"] == len([s for s in bwcurve_ref.ladder(bpp) if s <= 1 << 20]) == 9, ctx


def test_the_plan_refuses_more_than_16_gib_per_pair(pkg, host_plan):
    """The product's own rule: the oracle's plan has no ceiling."""
    lib = pkg.abi.load_library()
    over = MAX_BPP + 128
    cases = [(b, n, mode, flags) for b in (MAX_BPP, over) for mode in (MODE_SLICED, MODE_FULL) for n in (1, 2, 3, 16)
             for flags in (0, LOCAL_DIAG)]
    queries = [(n, config_bytes(n, b, mode), mode, flags) for b, n, mode, flags in cases]
    for (bpp, *_), q, hp in zip(cases, queries, host_plan(queries)):
        if bpp == over:
            assert hp == ERR_ARG, q
            assert lib.cdprobe_plan(*q, pkg.abi.PlanT()) == ERR_ARG, q
        else:
            assert hp["bpp"] == MAX_BPP and pkg.plan(*q).bytes_per_pair == MAX_BPP, q


def test_the_ladder_at_16_gib_has_23_sizes_ending_at_the_ceiling(host_plan):
    sizes = bwcurve_ref.ladder(MAX_BPP)
    assert len(sizes) == 23 and sizes[-1] == MAX_BPP and sizes[-2] == MAX_BPP // 2
    assert host_plan([(1, MAX_BPP, MODE_SLICED, 0)])[0]["ladder"] == sizes
    # the ladder's own 24-size limit lies past what a plan can reach
    assert len(bwcurve_ref.ladder(32 * GIB)) == 24 == bwcurve_ref.MAX_SIZES
