"""cdprobe_allreduce_nvls without a GPU: the declared and exported symbol, its fault option, path constant and encoder,
the ABI version and struct sizes, the argument errors, the wrapper, the Python restatement of a rep and of both fault
modes, the barrier lines, the compiled kernel's multicast instructions and spills, and the Go mirror."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import allreduce_nvls_ref as ref
import allreduce_ref
import word_ref
from conftest import ROOT
from harness import FakeLib, declared_symbols, exported_symbols, fake_probe, header_values
from kernel_tools import kernel_sass, ptxas_report

HEADER = os.path.join(ROOT, "include", "cdprobe.h")
CSRC = os.path.join(ROOT, "k8s-dra-driver-gpu_b200", "csrc")
U64_MAX = (1 << 64) - 1
SEED = 0xCD5EED0000000001


def test_option_path_and_symbol_match_the_header(pkg, tmp_path):
    a = pkg.abi
    got = header_values(tmp_path, "CDPROBE_OPT_ALLREDUCE_NVLS_FAULT", "CDPROBE_ALLREDUCE_PATH_NVLS")
    assert got == [a.OPT_ALLREDUCE_NVLS_FAULT, a.ALLREDUCE_PATH_NVLS] == [25, 5]
    assert a.SYMBOLS["cdprobe_allreduce_nvls"] == a.SYMBOLS["cdprobe_allreduce"]


PARENT_SIZES = {"cdprobe_config_t": 192, "cdprobe_result_t": 12376, "cdprobe_info_t": 5184, "cdprobe_plan_t": 304,
                "cdprobe_trace_t": 2632, "cdprobe_schedule_t": 1488, "cdprobe_topology_t": 2424,
                "cdprobe_diag_sample_t": 48, "cdprobe_diag_t": 1416, "cdprobe_latency_t": 6440,
                "cdprobe_pingpong_t": 6440, "cdprobe_atomics_t": 6704, "cdprobe_bwcurve_t": 178664,
                "cdprobe_allreduce_t": 17528, "cdprobe_alltoall_t": 204160}  # x86-64, from the parent commit's header


def test_the_abi_version_and_every_struct_size_are_unchanged(pkg, tmp_path):
    a = pkg.abi
    got = header_values(tmp_path, "CDPROBE_ABI_VERSION", *(f"sizeof({t})" for t in PARENT_SIZES))
    assert got[0] == a.ABI_VERSION == 2
    assert dict(zip(PARENT_SIZES, got[1:])) == PARENT_SIZES
    py = [a.ConfigT, a.ResultT, a.InfoT, a.PlanT, a.TraceT, a.ScheduleT, a.TopologyT, a.DiagSampleT, a.DiagT,
          a.LatencyT, a.PingPongT, a.AtomicsT, a.BwCurveT, a.AllReduceT, a.AllToAllT]
    assert [C.sizeof(t) for t in py] == list(PARENT_SIZES.values())


def test_the_symbol_is_declared_and_exported_and_the_abi_set_still_matches(pkg):
    exported = exported_symbols(pkg.abi.LIB_PATH)
    declared = declared_symbols()
    assert "cdprobe_allreduce_nvls" in declared and "cdprobe_allreduce_nvls" in exported
    assert declared == set(pkg.abi.SYMBOLS)


def test_the_fault_encoder_and_its_refusals(pkg):
    a = pkg.abi
    assert a.allreduce_nvls_fault(5, 77) == (6 << 24) | 77
    assert a.allreduce_nvls_fault(0, 9, mode=1) == (1 << 48) | (1 << 24) | 9
    assert a.allreduce_nvls_fault(254, (1 << 24) - 1, 1) == (1 << 48) | (255 << 24) | ((1 << 24) - 1)
    assert (a.allreduce_nvls_fault(254, (1 << 24) - 1, 1) >> 32) & 0xffff == 0
    for bad in (dict(mode=2), dict(mode=-1), dict(word=1 << 24), dict(word=-1), dict(k=255), dict(k=-1)):
        args = dict(k=0, word=0, mode=0)
        args.update(bad)
        with pytest.raises(ValueError):
            a.allreduce_nvls_fault(**args)


# ---- errors without a GPU -------------------------------------------------------------------------------------------
def test_a_null_handle_and_bad_reps_are_refused_and_fill_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.AllReduceT()
    t.n, t.call_seq, t.n_sizes, t.measured[0], t.bad_words[0][0] = 77, 5, 3, 1, 9
    assert lib.cdprobe_allreduce_nvls(None, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.reps, t.call_seq, t.n_sizes, t.row_mask) == (2, 0, a.ALLREDUCE_DEFAULT_REPS, 0, 0, 0)
    assert sum(t.measured) == 0 and t.bad_words[0][0] == 0
    assert lib.cdprobe_allreduce_nvls(None, 0, None) == a.ERR_ARG
    for reps in (1, a.ALLREDUCE_MAX_REPS + 1, 2 ** 32 - 1):
        t = a.AllReduceT()
        assert lib.cdprobe_allreduce_nvls(None, reps, C.byref(t)) == a.ERR_ARG
        assert (t.abi, t.reps) == (2, reps) and sum(t.measured) == 0
    assert lib.cdprobe_set_option(None, a.OPT_ALLREDUCE_NVLS_FAULT, 1) == a.ERR_ARG


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
        def cdprobe_allreduce_nvls(self, h, reps, out):
            calls.append((h.value, reps))
            t = out._obj
            t.abi, t.n, t.row_mask, t.reps, t.call_seq, t.n_sizes, t.path = 2, 2, 3, reps or 8, 4, 2, 5
            t.size[0], t.size[1] = 4096, 8192
            t.measured[0] = 1
            t.status[0], t.status[1] = a.ERR_INTEGRITY, a.ERR_UNSUPPORTED
            t.ns_min[0][0], t.ns_median[0][0], t.ns_max[0][0] = 1.0, 2.0, 3.0
            t.ns_median[0][1], t.sum[0][1], t.xr[0][1] = 4.0, 7, 9
            t.bad_words[0][1], t.first_bad[0][0], t.first_bad[0][1] = 1, U64_MAX, 8
            return a.ERR_ARG if reps > 64 else a.OK

    with fake_probe(pkg, Lib()) as p:
        ar = p.AllReduceNVLS()
        assert calls[-1] == (0x1234, 0)
        assert type(ar) is pkg.AllReduce
        assert (ar.n, ar.row_mask, ar.reps, ar.call_seq, ar.path, ar.sizes) == (2, 3, 8, 4, 5, [4096, 8192])
        assert ar.measured == [True, False]
        assert ar.status == [a.ERR_INTEGRITY, a.ERR_UNSUPPORTED]
        assert ar.ns_median[0] == [2.0, 4.0] and ar.ns_median[1] is None
        assert ar.sum[0] == [0, 7] and ar.bad_words[0] == [0, 1] and ar.first_bad[0] == [U64_MAX, 8]
        p.AllReduceNVLS(reps=3)
        assert calls[-1] == (0x1234, 3)
        with pytest.raises(pkg.ProbeError) as e:
            p.AllReduceNVLS(65)
        assert e.value.code == a.ERR_ARG


# ---- the restatement ------------------------------------------------------------------------------------------------
def sources(n, W, zero_unit=None):
    out = []
    for j in range(n):
        w = word_ref.src_words(SEED, j, 0, W).copy()
        if zero_unit is not None:
            lo, hi = ref.unit_span(8 * W, zero_unit)
            w[lo:hi:3] = 0  # some words of the unit sum to 0 in every rank: a skipped store leaves them right
        out.append(w)
    return out


SIZES = [4096, 8192, 24704, 57 * 8192 + 384, 16 * 8192]


@pytest.mark.parametrize("n", range(1, 17))
@pytest.mark.parametrize("size", SIZES)
def test_a_clean_rep_leaves_the_all_reduce_in_every_row(n, size):
    W = size // 8
    want = allreduce_ref.output_words(SEED, n, W)
    rows = ref.rep(sources(n, W), size)
    assert len(rows) == n and all((row == want).all() for row in rows)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("n", range(1, 17))
def test_each_fault_fails_exactly_the_rows_and_words_the_table_names(n, mode):
    for size in SIZES:
        W = size // 8
        for word in sorted({0, W // 2 + 1, W - 1}):
            srcs = sources(n, W, zero_unit=word // ref.UNIT_WORDS)
            want = sum(srcs[1:], srcs[0].copy())
            f = (mode, word)
            got = {r: [int(w) for w in np.flatnonzero(row != want)] for r, row in enumerate(ref.rep(srcs, size, f))}
            got = {r: ws for r, ws in got.items() if ws}
            assert got == ref.failing(srcs, size, f), (size, f)
            assert sorted(got) == list(range(n)), (size, f)  # every row, whoever owns the word
            if mode == 1:
                lo, hi = ref.unit_span(size, word // ref.UNIT_WORDS)
                assert all(lo <= w < hi for w in got[0]) and len(got[0]) < hi - lo


def test_the_owner_of_a_word_holds_it_in_the_two_shot_chunk():
    for n in range(1, 17):
        for size in SIZES:
            U = ref.units(size)
            for word in (0, size // 16, size // 8 - 1):
                o = ref.word_owner(size, n, word)
                assert U * o // n <= word // ref.UNIT_WORDS < U * (o + 1) // n


def test_bus_bandwidth_is_the_algorithm_bandwidth_times_2_n_minus_1_over_n():
    assert ref.busbw(100.0, 1) == 0.0 and ref.busbw(100.0, 2) == 100.0 and ref.busbw(100.0, 8) == 175.0


def test_the_barrier_lines_fit_the_ctrl_granule(tmp_path):
    src = tmp_path / "lines.cc"
    src.write_text('#include <stdio.h>\n#include "probe_types.h"\n'
                   'int main() { printf("%llu %llu %llu %zu\\n", (unsigned long long)cdp::kNvlsOff, '
                   '(unsigned long long)cdp::kPushOff, (unsigned long long)cdp::kCtrlBytes, sizeof(cdp::FlagLine)); }\n')
    exe = tmp_path / "lines"
    subprocess.run(["g++", "-std=c++17", "-I", CSRC, str(src), "-o", str(exe)], check=True)
    off, push, ctrl, line = map(int, subprocess.run([str(exe)], capture_output=True, text=True,
                                                    check=True).stdout.split())
    assert line == 128 and off == 80 << 10 and off == push + 16 * line
    assert off % 128 == 0 and off + 16 * line <= ctrl == 2 << 20
    assert 2 * (64 + 1) * 24 < 1 << 16  # two domain barriers per rep, 64 timed reps and a warm-up, 24 sizes


# ---- the compiled kernel ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kernel(pkg):
    return kernel_sass(pkg.abi.LIB_PATH, r"^_ZN3cdp21allreduce_nvls_kernelE")[1]


def test_the_kernel_reduces_with_multimem_ld_reduce_and_stores_16_bytes(kernel):
    """multimem.ld_reduce.relaxed.sys.global.add.u64 compiles to LDGMC.E.ADD.64.STRONG.SYS, and
    multimem.st.relaxed.sys.global.v4.f32 to STG.E.128.STRONG.SYS: two reductions per 16-byte store."""
    red = [t for t in kernel if re.match(r"(@!?U?P\w+ )?LDGMC\.E\.ADD\.64\.STRONG\.SYS ", t)]
    st = [t for t in kernel if re.match(r"(@!?U?P\w+ )?STG\.E\.128\.STRONG\.SYS ", t)]
    assert len(red) == 32 and len(st) >= 16


def test_no_other_kernel_issues_a_multimem_reduction(pkg):
    lib = pkg.abi.LIB_PATH
    for name in ["cdprobe_kernel", "bwcurve_kernel", "alltoall_kernel", "allreduce_kernel", "allreduce_twoshot_kernel",
                 "allreduce_ll_kernel", "allreduce_ring_kernel", "allreduce_push_kernel"]:
        ins = kernel_sass(lib, rf"^_ZN3cdp{len(name)}{name}E")[1]
        assert not any("LDGMC" in t for t in ins), name


def test_ptxas_reports_no_spills_in_the_nvls_unit():
    props = ptxas_report("allreduce_nvls_kernels.cu")
    nvls = [k for k in props if "allreduce_nvls_kernelE" in k]
    assert len(nvls) == 1, props
    assert props[nvls[0]][1:] == (0, 0), props



# ---- Go mirror ----------------------------------------------------------------------------------------------------
def test_go_nvls_is_consistent_across_shim_stub_and_header():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()
    assert "func (p *Probe) AllReduceNVLS(reps int) (AllReduce, error)" in shim
    assert "func (*Probe) AllReduceNVLS(int) (AllReduce, error)" in stub
    # optional binding: a missing symbol does not fail cdp_load, and AllReduceNVLS reports ErrUnsupported
    assert 'dlsym(cdp_dl, "cdprobe_allreduce_nvls")' in shim and "cdp_has_allreduce_nvls() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_arnvls" not in required
    assert "nvls := allReduceOf(res)" in shim
    hdr = open(HEADER).read()
    assert "CDPROBE_API int cdprobe_allreduce_nvls(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out);" in hdr
    assert re.search(r"#define CDPROBE_OPT_ALLREDUCE_NVLS_FAULT 25u", hdr)
    assert re.search(r"#define CDPROBE_ALLREDUCE_PATH_NVLS 5u", hdr)
