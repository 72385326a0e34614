"""cdprobe_allreduce_push without a GPU: the declared and exported symbol, its fault option and encoder, the argument
errors, the wrapper, the owner of a unit (twoshot_owner) against the two-shot's chunks, the Python restatement of a rep
and of every fault mode, the barrier lines, the compiled kernel's reductions and spills, and the Go mirror."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import allreduce_push_ref as ref
import allreduce_ref
import bwcurve_ref
import word_ref
from conftest import ROOT
from harness import FakeLib, c_tool, declared_symbols, exported_symbols, fake_probe, header_values
from kernel_tools import kernel_sass, ptxas_report

HEADER = os.path.join(ROOT, "include", "cdprobe.h")
U64_MAX = (1 << 64) - 1
SEED = 0xCD5EED0000000001


def test_option_and_symbol_match_the_header(pkg, tmp_path):
    a = pkg.abi
    assert header_values(tmp_path, "CDPROBE_OPT_ALLREDUCE_PUSH_FAULT") == [a.OPT_ALLREDUCE_PUSH_FAULT] == [24]
    assert a.SYMBOLS["cdprobe_allreduce_push"] == a.SYMBOLS["cdprobe_allreduce"]


def test_the_symbol_is_declared_and_exported_and_the_abi_set_still_matches(pkg):
    exported = exported_symbols(pkg.abi.LIB_PATH)
    declared = declared_symbols()
    assert "cdprobe_allreduce_push" in declared and "cdprobe_allreduce_push" in exported
    assert declared == set(pkg.abi.SYMBOLS)


def test_the_fault_encoder_and_its_refusals(pkg):
    a = pkg.abi
    assert a.allreduce_push_fault(2, 5, 77) == (3 << 32) | (6 << 24) | 77
    assert a.allreduce_push_fault(0, 0, 9, mode=1) == (1 << 48) | (1 << 32) | (1 << 24) | 9
    assert a.allreduce_push_fault(1, 2, 2000, mode=2) == (2 << 48) | (2 << 32) | (3 << 24) | 2000
    assert a.allreduce_push_fault(15, 23, (1 << 24) - 1, 3) == (3 << 48) | (16 << 32) | (24 << 24) | ((1 << 24) - 1)
    assert a.allreduce_push_fault(15, 23, (1 << 24) - 1, 3) >> 50 == 0
    for bad in (dict(mode=4), dict(mode=-1), dict(word=1 << 24), dict(word=-1), dict(rank=0xffff), dict(rank=-1),
                dict(k=255), dict(k=-1)):
        args = dict(rank=0, k=0, word=0, mode=0)
        args.update(bad)
        with pytest.raises(ValueError):
            a.allreduce_push_fault(**args)


# ---- errors without a GPU -------------------------------------------------------------------------------------------
def test_a_null_handle_and_bad_reps_are_refused_and_fill_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.AllReduceT()
    t.n, t.call_seq, t.n_sizes, t.measured[0], t.bad_words[0][0] = 77, 5, 3, 1, 9
    assert lib.cdprobe_allreduce_push(None, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.reps, t.call_seq, t.n_sizes, t.row_mask) == (2, 0, a.ALLREDUCE_DEFAULT_REPS, 0, 0, 0)
    assert sum(t.measured) == 0 and t.bad_words[0][0] == 0
    assert lib.cdprobe_allreduce_push(None, 0, None) == a.ERR_ARG
    for reps in (1, a.ALLREDUCE_MAX_REPS + 1, 2 ** 32 - 1):
        t = a.AllReduceT()
        assert lib.cdprobe_allreduce_push(None, reps, C.byref(t)) == a.ERR_ARG
        assert (t.abi, t.reps) == (2, reps) and sum(t.measured) == 0
    assert lib.cdprobe_set_option(None, a.OPT_ALLREDUCE_PUSH_FAULT, 1) == a.ERR_ARG


def test_open_without_a_gpu_still_fails_loudly(pkg):
    """No device here: opening a handle is an error, never a silent fall-back."""
    if os.path.exists("/dev/nvidia0"):
        pytest.skip("a GPU is present")
    with pytest.raises(pkg.ProbeError):
        pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 20))


def test_wrapper_passes_its_arguments(pkg):
    a = pkg.abi
    calls = []

    class Lib(FakeLib):
        def cdprobe_allreduce_push(self, h, reps, out):
            calls.append((h.value, reps))
            t = out._obj
            t.abi, t.n, t.row_mask, t.reps, t.call_seq, t.n_sizes, t.path = 2, 3, 2, reps or 8, 4, 2, 1
            t.size[0], t.size[1] = 4096, 8192
            t.measured[1], t.measured[2] = 1, 1
            t.status[0], t.status[1], t.status[2] = a.ERR_STATE, a.ERR_INTEGRITY, a.ERR_TIMEOUT
            t.ns_min[1][0], t.ns_median[1][0], t.ns_max[1][0] = 1.0, 2.0, 3.0
            t.ns_median[1][1], t.sum[1][1], t.xr[1][1] = 4.0, 7, 9
            t.bad_words[1][1], t.first_bad[1][0], t.first_bad[1][1] = 1, U64_MAX, 8
            t.t0_ns[1], t.peak_gbps[1], t.half_bytes[1], t.bad_sizes[1] = 2.0, 2048.0, 4096, 2
            return a.ERR_ARG if reps > 64 else a.OK

    with fake_probe(pkg, Lib()) as p:
        ar = p.AllReducePush()
        assert calls[-1] == (0x1234, 0)
        assert type(ar) is pkg.AllReduce
        assert (ar.n, ar.row_mask, ar.reps, ar.call_seq, ar.path, ar.sizes) == (3, 2, 8, 4, 1, [4096, 8192])
        assert ar.measured == [False, True, True]
        assert ar.status == [a.ERR_STATE, a.ERR_INTEGRITY, a.ERR_TIMEOUT]
        assert ar.ns_median[1] == [2.0, 4.0] and ar.ns_min[1] == [1.0, 0.0]
        assert ar.ns_median[0] is None and ar.sum[2] is None
        assert ar.sum[1] == [0, 7] and ar.xr[1] == [0, 9]
        assert ar.bad_words[1] == [0, 1] and ar.first_bad[1] == [U64_MAX, 8]
        p.AllReducePush(reps=3)
        assert calls[-1] == (0x1234, 3)
        with pytest.raises(pkg.ProbeError) as e:
            p.AllReducePush(65)
        assert e.value.code == a.ERR_ARG


# ---- the owner of a unit ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def helper(tmp_path_factory):
    return c_tool(tmp_path_factory, "push_owner.cc")


def test_the_owner_is_the_inverse_of_the_two_shot_chunks(helper):
    """For n = 1 ... 16 and unit counts from 0 up to the 32 GiB ladder's largest (4 Mi units), every U < n included:
    every unit's owner holds it in its chunk."""
    top = ref.units(bwcurve_ref.ladder(32 << 30)[-1])
    assert top == 4 << 20
    counts = sorted(set(range(0, 40)) | {57, 63, 64, 65, 127, 128, 129, 1000, 4095, 4096, 4097, 131071, 131072,
                                         (1 << 20) + 3, top - 1, top})
    cases = [(U, n) for n in range(1, 17) for U in counts]
    for (U, n), (got_u, bad) in zip(cases, helper([f"C {U} {n}" for U, n in cases])):
        assert (got_u, bad) == (U, -1), (U, n, bad)


def test_the_owner_matches_the_restatement(helper):
    cases = [(U, n, u) for n in (1, 2, 3, 5, 7, 8, 16) for U in (1, 2, 3, 7, 16, 17, 1000, 4 << 20)
             for u in sorted({0, U // 3, U // 2, U - 1})]
    got = helper([f"W {U} {n} {u}" for U, n, u in cases])
    for (U, n, u), (o,) in zip(cases, got):
        lo, hi = U * o // n, U * (o + 1) // n
        assert o == ref.owner(U, n, u) and lo <= u < hi, (U, n, u, o)


def test_the_barrier_lines_fit_the_ctrl_granule_and_the_barrier_count_fits_16_bits(helper):
    (off,), = helper(["G"])
    assert off == 78 << 10 and off % 128 == 0 and off + 16 * 128 <= 2 << 20
    assert 3 * (64 + 1) * 24 < 1 << 16  # three domain barriers per rep, 64 timed reps and a warm-up, 24 sizes


# ---- the restatement ------------------------------------------------------------------------------------------------
def sources(n, W, zero_every=0):
    out = []
    for j in range(n):
        w = word_ref.src_words(SEED, j, 0, W).copy()
        if zero_every:
            w[j::zero_every] = 0  # some source words are 0: a skipped or doubled reduction leaves them right
        out.append(w)
    return out


SIZES = [4096, 8192, 24704, 57 * 8192 + 384, 16 * 8192]


@pytest.mark.parametrize("n", [1, 2, 3, 5, 8, 16])
@pytest.mark.parametrize("size", SIZES)
def test_a_clean_rep_leaves_the_all_reduce_in_every_row(n, size):
    W = size // 8
    srcs = sources(n, W)
    want = allreduce_ref.output_words(SEED, n, W)
    for row in ref.rep(srcs, size):
        assert (row == want).all()


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
@pytest.mark.parametrize("n", [1, 2, 3, 8])
def test_each_fault_fails_exactly_the_rows_and_words_the_table_names(n, mode):
    if mode == 3 and n == 1:
        pytest.skip("mode 3 needs a peer")
    for size in SIZES:
        W = size // 8
        srcs = sources(n, W, zero_every=5)
        want = sum(srcs[1:], srcs[0].copy())
        for rank in range(n):
            for word in sorted({0, W // 2 + 1, W - 1}):
                if mode == 3 and ref.word_owner(size, n, word) == rank:
                    continue
                f = (mode, rank, word)
                got = {r: [int(w) for w in np.flatnonzero(row != want)] for r, row in enumerate(ref.rep(srcs, size, f))}
                got = {r: ws for r, ws in got.items() if ws}
                assert got == ref.failing(srcs, size, f), (size, f)
                assert got, (size, f)  # the sources hold non-zero words in every unit


def test_bus_bandwidth_is_the_algorithm_bandwidth_times_2_n_minus_1_over_n():
    assert ref.busbw(100.0, 1) == 0.0 and ref.busbw(100.0, 2) == 100.0 and ref.busbw(100.0, 8) == 175.0


# ---- the compiled kernel ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kernel(pkg):
    return kernel_sass(pkg.abi.LIB_PATH, r"^_ZN3cdp21allreduce_push_kernelE")[1]


def test_the_tma_path_reduces_in_bulk_and_the_ld_st_paths_with_system_scope_reds(kernel):
    """cp.reduce.async.bulk.global.shared::cta.bulk_group.add.u64 compiles to UBLKRED.G.S.ADD.U64, and
    red.relaxed.sys.global.add.u64 to REDG.E.ADD.64.STRONG.SYS; the stage is filled by a bulk copy."""
    assert any(re.match(r"(@!?U?P\w+ )?UBLKRED\.G\.S\.ADD\.U64 ", t) for t in kernel)
    assert any(re.match(r"(@!?U?P\w+ )?REDG\.E\.ADD\.64\.STRONG\.SYS ", t) for t in kernel)
    assert any(re.match(r"(@!?U?P\w+ )?UBLKCP\.S\.G ", t) for t in kernel)


def test_ptxas_reports_no_spills_in_the_push_unit():
    props = ptxas_report("allreduce_push_kernels.cu")
    push = [k for k in props if "allreduce_push_kernelE" in k]
    assert len(push) == 1, props
    assert props[push[0]][1:] == (0, 0), props



# ---- Go mirror ----------------------------------------------------------------------------------------------------
def test_go_push_is_consistent_across_shim_stub_and_header():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()
    assert "func (p *Probe) AllReducePush(reps int) (AllReduce, error)" in shim
    assert "func (*Probe) AllReducePush(int) (AllReduce, error)" in stub
    # optional binding: a missing symbol does not fail cdp_load, and AllReducePush reports ErrUnsupported
    assert 'dlsym(cdp_dl, "cdprobe_allreduce_push")' in shim and "cdp_has_allreduce_push() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_arpush" not in required
    # the push converts its result through the same function, without adding to the strings other tests count
    assert "push := allReduceOf(res)" in shim
    assert shim.count(" allReduceOf(ar)") == 3 and shim.count("return allReduceOf(ar), nil") == 2
    hdr = open(HEADER).read()
    assert "CDPROBE_API int cdprobe_allreduce_push(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out);" in hdr
    assert re.search(r"#define CDPROBE_OPT_ALLREDUCE_PUSH_FAULT 24u", hdr)
