"""cdprobe_alltoall without a GPU: the ABI layout, the salt sequence and block words of the reference against the
oracle, the per-rank summary on hand-built medians, the argument errors, the wrapper, the compiled kernel's store paths
and register use, and the Go mirror."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import alltoall_ref as ref
import word_ref
from conftest import ROOT
from harness import FakeLib, assert_layout, declared_symbols, exported_symbols, fake_probe, header_values
from kernel_tools import kernel_sass, ptxas_report

HEADER = os.path.join(ROOT, "include", "cdprobe.h")
U64_MAX = (1 << 64) - 1


def test_alltoall_struct_layout_matches_c(pkg, tmp_path):
    a = pkg.abi
    assert_layout(tmp_path, {"cdprobe_alltoall_t": a.AllToAllT})
    assert header_values(tmp_path, "CDPROBE_OPT_ALLTOALL_FAULT") == [a.OPT_ALLTOALL_FAULT] == [20]
    assert "cdprobe_alltoall" in a.SYMBOLS
    assert a.alltoall_fault(2, 0, 5, 77) == (3 << 40) | (1 << 32) | (6 << 24) | 77


def test_every_declared_symbol_is_exported(pkg):
    exported = exported_symbols(pkg.abi.LIB_PATH)
    declared = declared_symbols()
    assert "cdprobe_alltoall" in declared
    assert declared <= exported, declared - exported


# ---- the salt sequence and the block words -------------------------------------------------------------------------
def test_sequence_values_never_equal_a_run_seq_and_never_repeat():
    seen = set()
    for call in (1, 2, 3, (1 << 51) - 1):
        for k in range(24):
            for r in range(65):
                v = ref.alltoall_seq(call, k, r)
                assert v >> 63 == 1  # a run_seq counts runs from 1 and never reaches 2^63
                seen.add(v)
    assert len(seen) == 4 * 24 * 65


def test_block_words_restate_the_write_pattern():
    seed, i, j, call, k, r = 0x1234, 3, 5, 7, 2, 4
    w = ref.block_words(seed, i, j, call, k, r, 10)
    salt = word_ref.write_salt(seed, i, j, ref.alltoall_seq(call, k, r))
    for q in range(10):
        z = ((salt + q) * word_ref.GOLDEN) % (1 << 64)
        assert int(w[q]) == z ^ (z >> 32), q
    # a new salt every rep: a block that did not arrive is the previous rep's words, which do not pass the check
    assert not np.array_equal(w, ref.block_words(seed, i, j, call, k, r - 1, 10))


@pytest.mark.parametrize("words", [1, 2047, 2048, 2049, 70 * 2048 + 37])
def test_block_checksums_equal_the_oracle(oracle, words):
    for seed, i, j, call, k, r in ((0xCD5EED0000000001, 0, 1, 1, 0, 8), (0xABCDEF, 15, 15, 9, 23, 64),
                                   (7, 3, 0, (1 << 51) + 5, 11, 0)):
        seq = ref.alltoall_seq(call, k, r)
        got = ref.checksum(ref.block_words(seed, i, j, call, k, r, words))
        assert got == oracle.write_checksum(seed, i, j, seq, words), (seed, i, j, call, k, r)


def test_expected_is_the_last_timed_rep():
    sizes = [4096, 8192]
    got = ref.expected(1, 0, 1, 3, 2, sizes)
    assert got == [ref.checksum(ref.block_words(1, 0, 1, 3, k, 2, s // 8)) for k, s in enumerate(sizes)]


def test_block_order_interleaves_from_the_next_rank():
    every = lambda s, d: s != d  # noqa: E731
    assert ref.block_order(2, 5, every) == [3, 4, 0, 1]
    assert ref.block_order(2, 5, lambda s, d: True) == [3, 4, 0, 1, 2]
    assert ref.block_order(0, 1, lambda s, d: True) == [0]
    assert ref.block_order(1, 4, lambda s, d: s != d and d != 3) == [2, 0]


def test_rank_summary_on_hand_built_medians():
    """t0_ns is the smallest size's median; peak_gbps is the largest blocks x size / median; half_bytes the smallest
    size whose egress reaches half of it."""
    sizes = [4096, 8192, 16384, 32768]
    t0, peak, half = ref.summary(sizes, [1000.0, 2000.0, 4000.0, 8000.0], 1)  # egress 4.096 at every size
    assert (t0, half) == (1000.0, 4096) and peak == pytest.approx(4.096)
    t0, peak, half = ref.summary(sizes, [2048.0, 2048.0, 2048.0, 4096.0], 3)  # egress 6, 12, 24, 24
    assert (t0, peak, half) == (2048.0, 24.0, 8192)
    assert ref.summary(sizes, [0.0, 1024.0, 1024.0, 1024.0], 2) == (0.0, 64.0, 16384)


# ---- errors without a GPU -------------------------------------------------------------------------------------------
def test_alltoall_rejects_a_null_handle_and_fills_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.AllToAllT()
    t.n, t.call_seq, t.n_sizes, t.measured[0], t.cell_measured[3] = 77, 5, 3, 1, 1
    assert lib.cdprobe_alltoall(None, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.reps, t.call_seq, t.n_sizes, t.row_mask) == (2, 0, a.ALLTOALL_DEFAULT_REPS, 0, 0, 0)
    assert sum(t.measured) == 0 and sum(t.cell_measured) == 0
    assert lib.cdprobe_alltoall(None, 0, None) == a.ERR_ARG
    for reps in (1, a.ALLTOALL_MAX_REPS + 1, 2 ** 32 - 1):
        t = a.AllToAllT()
        assert lib.cdprobe_alltoall(None, reps, C.byref(t)) == a.ERR_ARG
        assert (t.abi, t.reps) == (2, reps) and sum(t.measured) == 0
    assert lib.cdprobe_set_option(None, a.OPT_ALLTOALL_FAULT, 1) == a.ERR_ARG


def test_wrapper_passes_its_arguments(pkg):
    a = pkg.abi
    calls = []

    class Lib(FakeLib):
        def cdprobe_alltoall(self, h, reps, out):
            calls.append((h.value, reps))
            t = out._obj
            t.abi, t.n, t.row_mask, t.reps, t.call_seq, t.n_sizes, t.path = 2, 3, 2, reps or 8, 4, 2, 1
            t.area_bytes = 6 << 20
            t.size[0], t.size[1] = 4096, 8192
            t.measured[1], t.measured[2] = 1, 1
            t.status[1], t.status[2] = 0, a.ERR_TIMEOUT
            t.blocks[1] = 2
            t.ns_min[1][0], t.ns_median[1][0], t.ns_max[1][0] = 1.0, 2.0, 3.0
            t.t0_ns[1], t.peak_gbps[1], t.half_bytes[1] = 2.0, 8.0, 4096
            c = 0 * 16 + 1
            t.cell_measured[c], t.cell_status[c], t.bad_sizes[c] = 1, a.ERR_INTEGRITY, 2
            t.bad_words[c][1], t.first_bad[c][0], t.first_bad[c][1], t.sum[c][1], t.xr[c][1] = 1, U64_MAX, 24, 7, 9
            t.cell_status[2 * 16 + 1] = a.ERR_STATE
            return a.ERR_ARG if reps > 64 else a.OK

    with fake_probe(pkg, Lib()) as p:
        aa = p.AllToAll()
        assert calls[-1] == (0x1234, 0)
        assert (aa.n, aa.row_mask, aa.reps, aa.call_seq, aa.path, aa.sizes, aa.area_bytes) == \
            (3, 2, 8, 4, 1, [4096, 8192], 6 << 20)
        assert aa.measured == [False, True, True] and aa.status == [0, 0, a.ERR_TIMEOUT]
        assert aa.blocks == [None, 2, 0]
        assert aa.ns_median[1] == [2.0, 0.0] and aa.ns_min[1] == [1.0, 0.0]
        assert aa.ns_median[0] is None and aa.ns_median[2] is None
        assert (aa.t0_ns[1], aa.peak_gbps[1], aa.half_bytes[1]) == (2.0, 8.0, 4096)
        assert aa.cell_measured[0][1] and aa.cell_status[0][1] == a.ERR_INTEGRITY and aa.bad_sizes[0][1] == 2
        assert aa.bad_words[0][1] == [0, 1] and aa.first_bad[0][1] == [U64_MAX, 24]
        assert aa.sum[0][1] == [0, 7] and aa.xr[0][1] == [0, 9]
        assert not aa.cell_measured[2][1] and aa.cell_status[2][1] == a.ERR_STATE and aa.sum[2][1] is None
        p.AllToAll(reps=3)
        assert calls[-1] == (0x1234, 3)
        with pytest.raises(pkg.ProbeError) as e:
            p.AllToAll(65)
        assert e.value.code == a.ERR_ARG
        assert pkg.AllToAll is type(aa)


# ---- the compiled kernel ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kernel(pkg):
    return kernel_sass(pkg.abi.LIB_PATH, r"^_ZN3cdp15alltoall_kernel")[1]


def test_every_write_path_is_compiled_in(kernel):
    """The TMA bulk stores from shared memory (UBLKCP global <- shared), and the st.global.v4 stores of the two ld/st
    paths, all through the probe's write jobs; the fence.sys before the completion stamp."""
    assert any(t.startswith("UBLKCP.G.S") for t in kernel)
    assert sum(t.startswith("STG.E.NA.128") for t in kernel) >= 2
    assert any(t.startswith("MEMBAR.SC.SYS") or t.startswith("MEMBAR.ALL.SYS") for t in kernel)
    assert any(t.startswith("LDG.E.NA.128") for t in kernel)  # the word check


def test_ptxas_reports_no_spills_in_the_alltoall_unit():
    props = ptxas_report("alltoall_kernels.cu")
    a2a = [k for k in props if "alltoall_kernelE" in k]
    assert len(a2a) == 1, props
    assert props[a2a[0]][1:] == (0, 0), props


# ---- Go mirror ----------------------------------------------------------------------------------------------------
def test_go_alltoall_is_consistent_across_shim_and_stub():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()

    def struct(src, name):
        body = src[src.index(f"type {name} struct {{"):]
        return body[:body.index("\n}")]

    assert "func (p *Probe) AllToAll(reps int) (AllToAll, error)" in shim
    assert "func (*Probe) AllToAll(int) (AllToAll, error)" in stub
    decls = re.findall(r"^\t([A-Z]\w*(?:, [A-Z]\w*)*) ", struct(shim, "AllToAll"), re.M)
    names = {n.strip() for d in decls for n in d.split(",")}
    assert {"Sizes", "Measured", "Status", "Blocks", "T0Ns", "PeakGBps", "HalfBytes", "NsMin", "NsMedian", "NsMax",
            "CellMeasured", "CellStatus", "BadSizes", "BadWords", "FirstBad", "Sum", "Xr", "RowMask", "CallSeq",
            "Path", "Reps", "AreaBytes"} <= names
    for n in names:
        assert re.search(rf"\b{n}\b", struct(stub, "AllToAll")), n
    assert 'dlsym(cdp_dl, "cdprobe_alltoall")' in shim and "cdp_has_alltoall() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_a2a" not in required
    hdr = open(HEADER).read()
    hdr_struct = hdr[hdr.index("typedef struct {", hdr.index("One-shot all-to-all across the domain")):
                     hdr.index("} cdprobe_alltoall_t;")]
    for fld in set(re.findall(r"\baa\.(\w+)", shim)):
        assert re.search(rf"\b{fld}\b", hdr_struct), fld
