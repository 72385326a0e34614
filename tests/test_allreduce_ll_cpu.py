"""cdprobe_allreduce_ll without a GPU: the declared and exported symbol, its fault option, path constant and encoder, the
argument errors, the wrapper, the ladder, flags, salts and slot layout of probe_types.h against the Python
restatement, the compiled kernel's packet stores and loads and its spills, and the Go mirror."""
import ctypes as C
import os
import re

import pytest

import allreduce_ll_ref as ref
from conftest import ROOT
from harness import FakeLib, c_tool, declared_symbols, exported_symbols, fake_probe, header_values
from kernel_tools import kernel_sass, ptxas_report

HEADER = os.path.join(ROOT, "include", "cdprobe.h")
U64_MAX = (1 << 64) - 1


def test_option_path_and_symbol_match_the_header(pkg, tmp_path):
    a = pkg.abi
    out = header_values(tmp_path, "CDPROBE_OPT_ALLREDUCE_LL_FAULT", "CDPROBE_ALLREDUCE_PATH_LL")
    assert out == [a.OPT_ALLREDUCE_LL_FAULT, a.ALLREDUCE_PATH_LL] == [22, 3]
    assert a.SYMBOLS["cdprobe_allreduce_ll"] == a.SYMBOLS["cdprobe_allreduce"]


def test_the_fault_encoder_and_its_refusals(pkg):
    a = pkg.abi
    assert a.allreduce_ll_fault(2, 0, 5, 77) == (3 << 40) | (1 << 32) | (6 << 24) | 77
    assert a.allreduce_ll_fault(0, 1, 0, 2000, mode=1) == (1 << 48) | (1 << 40) | (2 << 32) | (1 << 24) | 2000
    assert a.allreduce_ll_fault(15, 14, 23, (1 << 24) - 1, 1) >> 49 == 0
    assert a.allreduce_ll_fault(1, 1, 3, 500, mode=2) == (2 << 48) | (2 << 40) | (2 << 32) | (4 << 24) | 500
    assert a.allreduce_ll_fault(254, 254, 254, (1 << 24) - 1, 2) >> 50 == 0
    for bad in (dict(mode=3), dict(mode=-1), dict(arg=1 << 24), dict(arg=-1), dict(sender=255), dict(receiver=-1),
                dict(k=255)):
        args = dict(sender=0, receiver=1, k=0, arg=0, mode=0)
        args.update(bad)
        with pytest.raises(ValueError):
            a.allreduce_ll_fault(**args)


def test_the_symbol_is_declared_and_exported(pkg):
    exported = exported_symbols(pkg.abi.LIB_PATH)
    declared = declared_symbols()
    assert "cdprobe_allreduce_ll" in declared and "cdprobe_allreduce_ll" in exported


# ---- errors without a GPU -------------------------------------------------------------------------------------------
def test_a_null_handle_and_bad_reps_are_refused_and_fill_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.AllReduceT()
    t.n, t.call_seq, t.n_sizes, t.measured[0], t.bad_words[0][0] = 77, 5, 3, 1, 9
    assert lib.cdprobe_allreduce_ll(None, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.reps, t.call_seq, t.n_sizes, t.row_mask) == (2, 0, a.ALLREDUCE_DEFAULT_REPS, 0, 0, 0)
    assert sum(t.measured) == 0 and t.bad_words[0][0] == 0
    assert lib.cdprobe_allreduce_ll(None, 0, None) == a.ERR_ARG
    for reps in (1, a.ALLREDUCE_MAX_REPS + 1, 2 ** 32 - 1):
        t = a.AllReduceT()
        assert lib.cdprobe_allreduce_ll(None, reps, C.byref(t)) == a.ERR_ARG
        assert (t.abi, t.reps) == (2, reps) and sum(t.measured) == 0
    assert lib.cdprobe_set_option(None, a.OPT_ALLREDUCE_LL_FAULT, 1) == a.ERR_ARG


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
        def cdprobe_allreduce_ll(self, h, reps, out):
            calls.append((h.value, reps))
            t = out._obj
            t.abi, t.n, t.row_mask, t.reps, t.call_seq, t.n_sizes, t.path = 2, 3, 2, reps or 8, 4, 2, 3
            t.size[0], t.size[1] = 4096, 8192
            t.measured[1], t.measured[2] = 1, 1
            t.status[0], t.status[1], t.status[2] = a.ERR_STATE, a.ERR_INTEGRITY, a.ERR_TIMEOUT
            t.ns_min[1][0], t.ns_median[1][0], t.ns_max[1][0] = 1.0, 2.0, 3.0
            t.ns_median[1][1], t.sum[1][1], t.xr[1][1] = 4.0, 7, 9
            t.bad_words[1][1], t.first_bad[1][0], t.first_bad[1][1] = 1, U64_MAX, 8
            t.t0_ns[1], t.peak_gbps[1], t.half_bytes[1], t.bad_sizes[1] = 2.0, 2048.0, 4096, 2
            return a.ERR_ARG if reps > 64 else a.OK

    with fake_probe(pkg, Lib()) as p:
        ar = p.AllReduceLL()
        assert calls[-1] == (0x1234, 0)
        assert type(ar) is pkg.AllReduce
        assert (ar.n, ar.row_mask, ar.reps, ar.call_seq, ar.path, ar.sizes) == (3, 2, 8, 4, a.ALLREDUCE_PATH_LL,
                                                                                 [4096, 8192])
        assert ar.measured == [False, True, True]
        assert ar.status == [a.ERR_STATE, a.ERR_INTEGRITY, a.ERR_TIMEOUT]
        assert ar.ns_median[1] == [2.0, 4.0] and ar.ns_min[1] == [1.0, 0.0]
        assert ar.ns_median[0] is None and ar.sum[2] is None
        assert ar.sum[1] == [0, 7] and ar.xr[1] == [0, 9]
        assert ar.bad_words[1] == [0, 1] and ar.first_bad[1] == [U64_MAX, 8]
        p.AllReduceLL(reps=3)
        assert calls[-1] == (0x1234, 3)
        with pytest.raises(pkg.ProbeError) as e:
            p.AllReduceLL(65)
        assert e.value.code == a.ERR_ARG


# ---- ladder, flags, salts and slots ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def helper(tmp_path_factory):
    return c_tool(tmp_path_factory, "ll_flags.cc")


def test_the_ladder_matches_the_restatement_from_128_bytes_to_32_gib(helper):
    bpps = sorted({128, 256, 4096 - 128, 4096, 4096 + 128, 57 * 8192 + 384, (1 << 20) - 128, 1 << 20,
                   (1 << 20) + 128, 3 << 20, 1 << 30, 32 << 30} | {1 << e for e in range(7, 36)})
    got = helper([f"L {b}" for b in bpps])
    for bpp, row in zip(bpps, got):
        want = ref.ladder(bpp)
        assert row == [len(want)] + want, bpp
        assert want[-1] == min(bpp, ref.MAX_BYTES) and all(s <= ref.MAX_BYTES for s in want)
    assert helper(["L 34359738496"]) == [[0]]  # above 32 GiB: no ladder, as for the bwcurve


def test_flags_are_never_zero_and_distinct_within_a_call_and_from_the_call_before(helper):
    """Every (k < 24, r <= 64) of one call and of the next, for call numbers across the 2^16 wrap."""
    calls = [1, 2, 255, 256, 65534, 65535, 65536, 65537, 131071, 131072, (1 << 40) + 65535]
    cases = [(c, k, r) for c in calls for k in range(24) for r in range(65)]
    got = [v[0] for v in helper([f"F {c} {k} {r}" for c, k, r in cases])]
    flags = {}
    for (c, k, r), f in zip(cases, got):
        assert f == ref.flag(c, k, r) and f != 0 and f < 1 << 32
        flags.setdefault(c, set()).add(f)
    for c in calls:
        assert len(flags[c]) == 24 * 65, c
        if c + 1 in flags:
            assert not flags[c] & flags[c + 1], c


def test_salts_match_the_restatement(helper):
    cases = [(0xCD5EED0000000001, j, ref.flag(c, k, r)) for j in (0, 1, 15) for c in (1, 65536) for k in (0, 23)
             for r in (0, 1, 64)]
    got = [v[0] for v in helper([f"S {s} {j} {f}" for s, j, f in cases])]
    assert got == [ref.salt(s, j, f) for s, j, f in cases]
    assert len(set(got)) == len(got)


def test_slots_tile_the_area_for_every_domain_size(helper):
    lines, want = [], []
    for n in range(1, 17):
        for s_max in (128, 4096, 57 * 8192 + 384, 1 << 20):
            W = s_max // 8
            for p in (0, 1):
                for s in sorted({0, n // 2, n - 1}):
                    for w in sorted({0, 1, W // 2, W - 1}):
                        lines.append(f"O {p} {n} {s} {s_max} {w}")
                        want.append((p, n, s, s_max, w))
    got = helper(lines)
    for (p, n, s, s_max, w), (off, area) in zip(want, got):
        assert off == ref.slot(p, n, s, s_max, w) and area == ref.area_bytes(n, s_max)
        assert off % 16 == 0 and off + 16 <= area
    assert ref.area_bytes(16, 1 << 20) == 64 << 20
    # the last packet of the last sender in parity 1 ends the area
    assert ref.slot(1, 16, 15, 1 << 20, (1 << 17) - 1) + 16 == 64 << 20


# ---- the compiled kernel ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kernel(pkg):
    return kernel_sass(pkg.abi.LIB_PATH, r"^_ZN3cdp19allreduce_ll_kernel")[1]


def test_the_packets_are_single_128_bit_system_scope_accesses(kernel):
    """st.relaxed.sys.global.v2.u64 and ld.relaxed.sys.global.v2.u64 compile to one STG.E.128.STRONG.SYS and one
    LDG.E.128.STRONG.SYS; the kernel has no TMA copy and no fence.sys."""
    assert any(t.startswith("STG.E.128.STRONG.SYS") for t in kernel)
    assert any(t.startswith("LDG.E.128.STRONG.SYS") for t in kernel)
    assert not any(t.startswith(("UBLKCP", "SYNCS.PHASECHK")) for t in kernel)
    assert not any(re.match(r"MEMBAR\.(SC|ALL)\.SYS", t) for t in kernel)
    assert any(t.startswith("LDG.E.64.STRONG.GPU") for t in kernel)  # the word check's ld.global.cg


def test_the_word_check_clears_every_word_it_reads(kernel):
    """After its ld.global.cg of an output word, the word check stores 0 over it, so the next size or call finds 0s
    wherever it makes no store; then a fence, before the next size's opening barrier."""
    loads = [k for k, t in enumerate(kernel) if t.startswith("LDG.E.64.STRONG.GPU")]
    clears = [k for k, t in enumerate(kernel) if re.match(r"STG\.E\.64 .*, RZ$", t)]
    assert loads and clears and any(k > min(loads) for k in clears)
    assert any(t.startswith("MEMBAR.SC.GPU") for t in kernel[min(clears):])


def test_ptxas_reports_no_spills_in_the_ll_unit():
    props = ptxas_report("allreduce_ll_kernels.cu")
    ll = [k for k in props if "allreduce_ll_kernelE" in k]
    assert len(ll) == 1, props
    assert props[ll[0]][1:] == (0, 0), props



# ---- Go mirror ----------------------------------------------------------------------------------------------------
def test_go_ll_is_consistent_across_shim_stub_and_header():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()
    assert "func (p *Probe) AllReduceLL(reps int) (AllReduce, error)" in shim
    assert "func (*Probe) AllReduceLL(int) (AllReduce, error)" in stub
    # optional binding: a missing symbol does not fail cdp_load, and AllReduceLL reports ErrUnsupported
    assert 'dlsym(cdp_dl, "cdprobe_allreduce_ll")' in shim and "cdp_has_allreduce_ll() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_arll" not in required
    # the three all-reduces fill their result through the one conversion
    assert shim.count(" allReduceOf(ar)") == 3 and "ll := allReduceOf(ar)" in shim
    hdr = open(HEADER).read()
    assert "CDPROBE_API int cdprobe_allreduce_ll(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out);" in hdr
    assert re.search(r"#define CDPROBE_OPT_ALLREDUCE_LL_FAULT 22u", hdr)
    assert re.search(r"#define CDPROBE_ALLREDUCE_PATH_LL 3u", hdr)
