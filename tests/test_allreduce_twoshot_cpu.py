"""cdprobe_allreduce_twoshot without a GPU: the declared and exported symbol and its fault option, the argument errors,
the wrapper, the chunk partition of probe_types.h against the Python restatement, the compiled kernel's stores, fences
and register use, and the Go mirror."""
import ctypes as C
import os
import re

import pytest

import allreduce_twoshot_ref as ref
from conftest import ROOT
from harness import FakeLib, c_tool, declared_symbols, exported_symbols, fake_probe, header_values
from kernel_tools import kernel_sass, ptxas_report

HEADER = os.path.join(ROOT, "include", "cdprobe.h")
U64_MAX = (1 << 64) - 1


def test_option_and_symbol_match_the_header(pkg, tmp_path):
    a = pkg.abi
    assert header_values(tmp_path, "CDPROBE_OPT_ALLREDUCE_TWOSHOT_FAULT") == [a.OPT_ALLREDUCE_TWOSHOT_FAULT] == [21]
    assert a.SYMBOLS["cdprobe_allreduce_twoshot"] == a.SYMBOLS["cdprobe_allreduce"]
    assert a.allreduce_twoshot_fault(2, 5, 77) == (3 << 32) | (6 << 24) | 77
    assert a.allreduce_twoshot_fault(0, 0, 0, drop=True) == (1 << 48) | (1 << 32) | (1 << 24)
    assert a.allreduce_twoshot_fault(15, 23, (1 << 24) - 1, True) >> 49 == 0


def test_the_symbol_is_declared_and_exported(pkg):
    exported = exported_symbols(pkg.abi.LIB_PATH)
    declared = declared_symbols()
    assert "cdprobe_allreduce_twoshot" in declared and "cdprobe_allreduce_twoshot" in exported


# ---- errors without a GPU -------------------------------------------------------------------------------------------
def test_a_null_handle_and_bad_reps_are_refused_and_fill_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.AllReduceT()
    t.n, t.call_seq, t.n_sizes, t.measured[0], t.bad_words[0][0] = 77, 5, 3, 1, 9
    assert lib.cdprobe_allreduce_twoshot(None, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.reps, t.call_seq, t.n_sizes, t.row_mask) == (2, 0, a.ALLREDUCE_DEFAULT_REPS, 0, 0, 0)
    assert sum(t.measured) == 0 and t.bad_words[0][0] == 0
    assert lib.cdprobe_allreduce_twoshot(None, 0, None) == a.ERR_ARG
    for reps in (1, a.ALLREDUCE_MAX_REPS + 1, 2 ** 32 - 1):
        t = a.AllReduceT()
        assert lib.cdprobe_allreduce_twoshot(None, reps, C.byref(t)) == a.ERR_ARG
        assert (t.abi, t.reps) == (2, reps) and sum(t.measured) == 0
    assert lib.cdprobe_set_option(None, a.OPT_ALLREDUCE_TWOSHOT_FAULT, 1) == a.ERR_ARG


def test_wrapper_passes_its_arguments(pkg):
    a = pkg.abi
    calls = []

    class Lib(FakeLib):
        def cdprobe_allreduce_twoshot(self, h, reps, out):
            calls.append((h.value, reps))
            t = out._obj
            t.abi, t.n, t.row_mask, t.reps, t.call_seq, t.n_sizes, t.path = 2, 3, 2, reps or 8, 4, 2, 1
            t.size[0], t.size[1] = 4096, 8192
            t.measured[1], t.measured[2] = 1, 1
            t.status[0], t.status[1], t.status[2] = a.ERR_STATE, a.ERR_INTEGRITY, a.ERR_TIMEOUT
            t.ns_min[1][0], t.ns_median[1][0], t.ns_max[1][0] = 1.0, 2.0, 3.0
            t.ns_median[1][1], t.sum[1][1], t.xr[1][1] = 4.0, 7, 9
            t.bad_words[1][1], t.first_bad[1][0], t.first_bad[1][1] = 1024, U64_MAX, 8192
            t.t0_ns[1], t.peak_gbps[1], t.half_bytes[1], t.bad_sizes[1] = 2.0, 2048.0, 4096, 2
            return a.ERR_ARG if reps > 64 else a.OK

    with fake_probe(pkg, Lib()) as p:
        ar = p.AllReduceTwoShot()
        assert calls[-1] == (0x1234, 0)
        assert type(ar) is pkg.AllReduce
        assert (ar.n, ar.row_mask, ar.reps, ar.call_seq, ar.path, ar.sizes) == (3, 2, 8, 4, 1, [4096, 8192])
        assert ar.measured == [False, True, True]
        assert ar.status == [a.ERR_STATE, a.ERR_INTEGRITY, a.ERR_TIMEOUT]
        assert ar.ns_median[1] == [2.0, 4.0] and ar.ns_min[1] == [1.0, 0.0]
        assert ar.ns_median[0] is None and ar.sum[2] is None
        assert ar.sum[1] == [0, 7] and ar.xr[1] == [0, 9]
        assert ar.bad_words[1] == [0, 1024] and ar.first_bad[1] == [U64_MAX, 8192]
        assert (ar.t0_ns[1], ar.peak_gbps[1], ar.half_bytes[1], ar.bad_sizes[1]) == (2.0, 2048.0, 4096, 2)
        p.AllReduceTwoShot(reps=3)
        assert calls[-1] == (0x1234, 3)
        with pytest.raises(pkg.ProbeError) as e:
            p.AllReduceTwoShot(65)
        assert e.value.code == a.ERR_ARG


# ---- the chunk partition -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def chunks(tmp_path_factory):
    run = c_tool(tmp_path_factory, "twoshot_chunks.cc")
    return lambda cases: [[tuple(v[2 * r:2 * r + 2]) for r in range(len(v) // 2)] for v in run(cases)]


def test_chunks_are_a_disjoint_cover_and_match_the_restatement(chunks):
    """For n from 1 to 16: fewer units than ranks, exactly n, one more, sizes with a partial last unit (128 bytes, one
    vector past a unit, 1 GiB plus one vector) and large ladders."""
    sizes = [128, 4096, 8192, 8192 + 128, 3 * 8192, 57 * 8192 + 384, 1 << 20, (1 << 30) + 128, 32 << 30]
    cases = []
    for n in range(1, 17):
        cases += [(ref.units(s), n) for s in sizes] + [(u, n) for u in (0, 1, n - 1, n, n + 1, 2 * n + 3)]
    got = chunks(cases)
    for (U, n), row in zip(cases, got):
        assert row == [ref.chunk(U, n, r) for r in range(n)], (U, n)
        covered = [u for lo, hi in row for u in range(lo, hi)] if U < 100000 else None
        if covered is not None:
            assert covered == list(range(U)), (U, n)  # in rank order, each unit once
        assert row[0][0] == 0 and row[-1][1] == U and all(row[r][1] == row[r + 1][0] for r in range(n - 1))
        assert all(lo <= hi for lo, hi in row)
        if U < n:
            assert sum(1 for lo, hi in row if lo == hi) == n - U  # some ranks own nothing
        assert max(hi - lo for lo, hi in row) - min(hi - lo for lo, hi in row) <= 1


def test_the_fault_owner_and_unit_of_a_partial_last_unit():
    size = 57 * 8192 + 384
    last = size // 8 - 1
    assert ref.owner(size, 3, last) == 2 and ref.unit_words(size, last) == 48
    assert ref.owner(size, 3, 0) == 0 and ref.unit_words(size, 0) == 1024
    assert [ref.owner(128, n, 0) for n in (1, 2, 5)] == [0, 1, 4]  # one unit: the last rank owns it
    assert ref.busbw(100.0, 4) == pytest.approx(150.0) and ref.busbw(100.0, 1) == 0.0


# ---- the compiled kernel ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kernel(pkg):
    return kernel_sass(pkg.abi.LIB_PATH, r"^_ZN3cdp24allreduce_twoshot_kernel")[1]


def test_every_read_path_the_pushes_and_the_fences_are_compiled_in(kernel):
    """The one-shot's read side (TMA bulk loads completed on mbarriers, 128-bit ld/st loads), the pushes and the
    clearing stores (128-bit global stores), the check's L2 loads and the fence.sys before the closing barrier."""
    assert any(t.startswith("UBLKCP.S.G") for t in kernel)
    assert any(t.startswith("SYNCS.PHASECHK.TRANS64.TRYWAIT") for t in kernel)
    assert sum(t.startswith("LDG.E.NA.128") for t in kernel) >= 32
    assert sum(t.startswith("STG.E.NA.128") for t in kernel) >= 3 * 16 + 1
    assert any(t.startswith("LDG.E.128.STRONG.GPU") for t in kernel)  # ld.global.cg: the check reads at L2
    assert any(re.match(r"MEMBAR\.(SC|ALL)\.SYS", t) for t in kernel)
    assert not any(t.startswith("UBLKCP.G.S") for t in kernel)  # the sums do not leave through TMA


def test_ptxas_reports_no_spills_in_the_twoshot_unit():
    props = ptxas_report("allreduce_twoshot_kernels.cu")
    ts = [k for k in props if "allreduce_twoshot_kernelE" in k]
    assert len(ts) == 1, props
    assert props[ts[0]][1:] == (0, 0), props


# ---- Go mirror ----------------------------------------------------------------------------------------------------
def test_go_twoshot_is_consistent_across_shim_stub_and_header():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()
    assert "func (p *Probe) AllReduceTwoShot(reps int) (AllReduce, error)" in shim
    assert "func (*Probe) AllReduceTwoShot(int) (AllReduce, error)" in stub
    # optional binding: a missing symbol does not fail cdp_load, and AllReduceTwoShot reports ErrUnsupported
    assert 'dlsym(cdp_dl, "cdprobe_allreduce_twoshot")' in shim and "cdp_has_allreduce_twoshot() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_ar2" not in required
    # both all-reduces fill their result through the one conversion, which reads only fields the header declares
    assert shim.count("return allReduceOf(ar), nil") == 2
    hdr = open(HEADER).read()
    assert "CDPROBE_API int cdprobe_allreduce_twoshot(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out);" in hdr
    assert re.search(r"#define CDPROBE_OPT_ALLREDUCE_TWOSHOT_FAULT 21u", hdr)
    hdr_struct = hdr[hdr.index("typedef struct {", hdr.index("One-shot all-reduce across the domain")):
                     hdr.index("} cdprobe_allreduce_t;")]
    for fld in set(re.findall(r"\bar\.(\w+)", shim)):
        assert re.search(rf"\b{fld}\b", hdr_struct), fld
