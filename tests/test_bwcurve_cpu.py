"""cdprobe_bwcurve without a GPU: the ABI layout, the size ladder and summary against tests/bwcurve_ref.py, the
expected-checksum fold of probe_types.h against the oracle, the argument errors, the wrapper, the compiled kernel's
data paths, barrier and timer order, its register use, and the Go mirror."""
import ctypes as C
import os
import random
import re

import pytest

import bwcurve_ref as ref
from conftest import ROOT
from harness import FakeLib, assert_layout, c_tool, fake_probe, header_values
from kernel_tools import kernel_sass, ptxas_report

HEADER = os.path.join(ROOT, "include", "cdprobe.h")
GIB = 1 << 30
G = 2048  # words per 16 KiB granule


def test_bwcurve_struct_layout_matches_c(pkg, tmp_path):
    a = pkg.abi
    assert_layout(tmp_path, {"cdprobe_bwcurve_t": a.BwCurveT})
    assert header_values(tmp_path, "CDPROBE_BWCURVE_MAX_SIZES") == [a.BWCURVE_MAX_SIZES] == [ref.MAX_SIZES] == [24]
    assert "cdprobe_bwcurve" in a.SYMBOLS


# ---- the ladder and the summary ---------------------------------------------------------------------------------
def test_ladder_restatement_by_hand():
    assert ref.ladder(128) == [128]
    assert ref.ladder(4096) == [4096]
    assert ref.ladder(4096 + 128) == [4096, 4096 + 128]
    assert ref.ladder(8192) == [4096, 8192]
    g = ref.ladder(GIB)
    assert g == [4096 << k for k in range(18)] + [GIB] and len(g) == 19
    assert len(ref.ladder(32 * GIB)) == 24
    with pytest.raises(ValueError):
        ref.ladder(32 * GIB + 128)


def test_summary_restatement_by_hand():
    sizes = [4096, 8192, 16384, 32768]
    flat = [1000.0, 2000.0, 4000.0, 8000.0]  # 4.096 bytes/ns at every size
    t0, peak, half = ref.summary(sizes, flat)
    assert (t0, half) == (1000.0, 4096) and abs(peak - 4.096) < 1e-6
    mid = [4096.0, 1024.0, 8192.0, 32768.0]  # rates 1, 8, 2, 1: the peak is the second size
    t0, peak, half = ref.summary(sizes, mid)
    assert (t0, peak, half) == (4096.0, 8.0, 8192)
    rising = [4096.0, 4096.0, 4096.0, 4096.0]  # rates 1, 2, 4, 8: half the peak first reached at 16 KiB
    assert ref.summary(sizes, rising) == (4096.0, 8.0, 16384)
    assert ref.summary([128], [50.0]) == (50.0, ref.summary([128], [50.0])[1], 128)


@pytest.fixture(scope="module")
def fold(tmp_path_factory):
    return c_tool(tmp_path_factory, "bwcurve_fold.cc")


def test_library_ladder_matches_the_restatement(fold):
    cases = [128, 256, 4096 - 128, 4096, 4096 + 128, 8192, 8192 + 128, 1 << 20, (1 << 20) + 5 * 1024 + 128,
             GIB // 7 // 128 * 128, GIB, 16 * GIB, 32 * GIB - 128, 32 * GIB]
    for bpp, got in zip(cases, fold([("L", b) for b in cases])):
        assert got[0] == len(got) - 1 and got[1:] == ref.ladder(bpp), bpp
    # the library refuses what the restatement refuses: host-only arithmetic, so no 32 GiB allocation is needed
    for bpp in (32 * GIB + 128, 64 * GIB, 1 << 62):
        with pytest.raises(ValueError):
            ref.ladder(bpp)
        assert fold([("L", bpp)]) == [[0]]


def test_prefix_fold_matches_the_oracle(fold, oracle):
    """Every prefix of the ladder, and prefixes that end inside a granule, for random (seed, rank, slice): the fold of
    per-granule sums plus the generated tail equals cdoracle_src_checksum of that prefix."""
    rng = random.Random(20261015)
    lines, want = [], []
    for _ in range(12):
        seed, rank = rng.getrandbits(64), rng.randrange(16)
        bpp = rng.choice([128, 4096, 4096 + 128, 70 * G * 8 + 300 * 8 // 16 * 16, (1 << 20) + 5 * 1024 + 128,
                          rng.randrange(1, 200) * 128])
        first = rng.randrange(8) * (bpp // 8)  # slice s of the source
        words = bpp // 8
        prefixes = sorted({s // 8 for s in ref.ladder(bpp)} | {rng.randrange(1, words + 1) for _ in range(3)} |
                          {min(words, G - 1), min(words, G + 1)})
        lines.append(("F", seed, rank, first, words, len(prefixes), *prefixes))
        want.append([v for n in prefixes for v in oracle.src_checksum(seed, rank, first, n)])
    assert fold(lines) == want


# ---- errors without a GPU -------------------------------------------------------------------------------------------
def test_bwcurve_rejects_a_null_handle_and_fills_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.BwCurveT()
    t.n, t.call_seq, t.n_sizes = 77, 5, 3
    assert lib.cdprobe_bwcurve(None, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.reps, t.call_seq, t.n_sizes, t.row_mask) == (2, 0, a.BWCURVE_DEFAULT_REPS, 0, 0, 0)
    assert lib.cdprobe_bwcurve(None, 0, None) == a.ERR_ARG
    for reps in (1, a.BWCURVE_MAX_REPS + 1, 2 ** 32 - 1):
        t = a.BwCurveT()
        assert lib.cdprobe_bwcurve(None, reps, C.byref(t)) == a.ERR_ARG
        assert (t.abi, t.reps) == (2, reps) and sum(t.measured) == 0


def test_wrapper_passes_its_arguments(pkg):
    a = pkg.abi
    calls = []

    class Lib(FakeLib):
        def cdprobe_bwcurve(self, h, reps, out):
            calls.append((h.value, reps))
            t = out._obj
            t.abi, t.n, t.row_mask, t.reps, t.call_seq, t.n_sizes, t.path = 2, 2, 1, reps or 8, 3, 2, 1
            t.size[0], t.size[1] = 4096, 8192
            t.measured[1] = 1
            t.ns_min[1][0], t.ns_median[1][0], t.ns_max[1][0] = 1.0, 2.0, 3.0
            t.ns_median[1][1], t.sum[1][1], t.xr[1][1] = 4.0, 7, 9
            t.t0_ns[1], t.peak_gbps[1], t.half_bytes[1], t.bad_sizes[1] = 2.0, 2048.0, 4096, 2
            t.status[0], t.status[1] = a.ERR_STATE, a.ERR_INTEGRITY
            return a.ERR_ARG if reps > 64 else a.OK

    with fake_probe(pkg, Lib()) as p:
        bw = p.BwCurve()
        assert calls[-1] == (0x1234, 0)
        assert (bw.n, bw.reps, bw.call_seq, bw.path, bw.sizes) == (2, 8, 3, 1, [4096, 8192])
        assert bw.measured == [[False, True], [False, False]]
        assert bw.status == [[a.ERR_STATE, a.ERR_INTEGRITY], [0, 0]]
        assert bw.ns_median[0][1] == [2.0, 4.0] and bw.ns_min[0][1] == [1.0, 0.0] and bw.ns_median[0][0] is None
        assert bw.sum[0][1] == [0, 7] and bw.xr[0][1] == [0, 9]
        assert (bw.t0_ns[0][1], bw.peak_gbps[0][1], bw.half_bytes[0][1], bw.bad_sizes[0][1]) == (2.0, 2048.0, 4096, 2)
        p.BwCurve(reps=3)
        assert calls[-1] == (0x1234, 3)
        with pytest.raises(pkg.ProbeError) as e:
            p.BwCurve(65)
        assert e.value.code == a.ERR_ARG
        assert pkg.BwCurve is type(bw)


# ---- the compiled kernel ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kernel(pkg):
    return kernel_sass(pkg.abi.LIB_PATH, r"^_ZN3cdp14bwcurve_kernel")[1]


def body(text):
    """The kernel up to the EXIT that ends its rep loop (out-of-line slow paths, such as mbar_drain, follow it)."""
    end = next(k for k, t in enumerate(text) if t.startswith("REDG.E.MAX.64"))
    return text[:next(k for k in range(end, len(text)) if text[k] == "EXIT") + 1]


def test_every_read_path_is_compiled_in(kernel):
    """The TMA bulk path (UBLKCP into shared memory, completed on an mbarrier: SYNCS) and the two ld/st paths
    (128-bit global loads that bypass L1) are all in the kernel, and none of the write path's stores is."""
    b = body(kernel)
    assert any(t.startswith("UBLKCP.S.G") for t in b)
    assert any(t.startswith("SYNCS.ARRIVE.TRANS64") for t in b)
    assert any(t.startswith("SYNCS.PHASECHK.TRANS64.TRYWAIT") for t in b)
    assert sum(t.startswith("LDG.E.NA.128") for t in b) >= 32  # 16 vectors in flight per lane, on each ld/st path
    assert not any(t.startswith(("STG.E.128", "UBLKCP.G.S")) for t in kernel)


def test_the_closing_timer_read_follows_the_reps_loads_and_fold(kernel):
    """The completion stamp is a %globaltimer read made after the CTA barrier that follows every warp's last load
    and fold, and after the CTA's (S, X) reductions; it is the value the REDG.MAX stores."""
    b = body(kernel)
    mx = next(k for k, t in enumerate(b) if t.startswith("REDG.E.MAX.64"))
    timer = max(k for k in range(mx) if "SR_GLOBALTIMER" in b[k])
    assert re.match(r"CS2R (R\d+), SR_GLOBALTIMERLO", b[timer])
    reg = re.match(r"CS2R (R\d+)", b[timer]).group(1)
    assert b[mx].endswith(reg)
    bar = max(k for k in range(timer) if b[k].startswith("BAR.SYNC"))
    loads = [k for k, t in enumerate(b) if t.startswith(("LDG.E.NA.128", "SYNCS.PHASECHK"))]
    assert loads and max(loads) < bar < timer
    reds = [k for k, t in enumerate(b) if re.match(r"REDG\.E\.(ADD|XOR)\.64", t)]
    assert len(reds) == 2 and bar < min(reds) and max(reds) < timer


def test_ptxas_reports_no_spills_in_the_bwcurve_unit():
    props = ptxas_report("bwcurve_kernels.cu")
    bw = [k for k in props if "bwcurve_kernelE" in k or "granules_kernelINS_13SrcRegionWord" in k]
    assert len(bw) == 2, props
    assert all(v[1:] == (0, 0) for v in props.values()), props


# ---- Go mirror ----------------------------------------------------------------------------------------------------
def test_go_bwcurve_is_consistent_across_shim_and_stub():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()

    def struct(src, name):
        body = src[src.index(f"type {name} struct {{"):]
        return body[:body.index("\n}")]

    assert "func (p *Probe) BwCurve(reps int) (BwCurve, error)" in shim
    assert "func (*Probe) BwCurve(int) (BwCurve, error)" in stub
    decls = re.findall(r"^\t([A-Z]\w*(?:, [A-Z]\w*)*) ", struct(shim, "BwCurve"), re.M)
    names = {n.strip() for d in decls for n in d.split(",")}
    assert {"Sizes", "Measured", "Status", "BadSizes", "T0Ns", "PeakGBps", "HalfBytes", "NsMin", "NsMedian", "NsMax",
            "Sum", "Xr", "RowMask", "CallSeq", "Path", "Reps"} <= names
    for n in names:
        assert re.search(rf"\b{n}\b", struct(stub, "BwCurve")), n
    # optional binding: a missing symbol does not fail cdp_load, and BwCurve reports ErrUnsupported
    assert 'dlsym(cdp_dl, "cdprobe_bwcurve")' in shim and "cdp_has_bwcurve() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_bw" not in required
    # the shim reads only fields the header declares
    hdr = open(HEADER).read()
    hdr_struct = hdr[hdr.index("typedef struct {", hdr.index("Bandwidth versus transfer size")):hdr.index("} cdprobe_bwcurve_t;")]
    for fld in set(re.findall(r"\bbw\.(\w+)", shim)):
        assert re.search(rf"\b{fld}\b", hdr_struct), fld
