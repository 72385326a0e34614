"""cdprobe_allreduce without a GPU: the ABI layout, the expected-checksum fold of probe_types.h and the numpy reference
against the oracle, the per-row summary on hand-built medians, the argument errors, the wrapper, the compiled kernel's
data paths and timer order, its register use, and the Go mirror."""
import ctypes as C
import os
import random
import re
import shutil
import subprocess

import numpy as np
import pytest

import allreduce_ref as ref
from conftest import ROOT

HEADER = os.path.join(ROOT, "include", "cdprobe.h")
CSRC = os.path.join(ROOT, "k8s-dra-driver-gpu_b200", "csrc")
G = 2048  # words per 16 KiB granule
U64_MAX = (1 << 64) - 1


def test_allreduce_struct_layout_matches_c(pkg, tmp_path):
    a = pkg.abi
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{HEADER}"', "int main(void){",
             'printf("sizeof %zu\\n", sizeof(cdprobe_allreduce_t));',
             'printf("opt %u\\n", CDPROBE_OPT_ALLREDUCE_FAULT);']
    for fname, _ in a.AllReduceT._fields_:
        lines.append(f'printf("{fname} %zu\\n", offsetof(cdprobe_allreduce_t, {fname}));')
    lines.append("return 0;}")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-o", str(exe), str(src)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["sizeof"]) == C.sizeof(a.AllReduceT)
    for fname, _ in a.AllReduceT._fields_:
        assert int(got[fname]) == getattr(a.AllReduceT, fname).offset, fname
    assert int(got["opt"]) == a.OPT_ALLREDUCE_FAULT == 19
    assert "cdprobe_allreduce" in a.SYMBOLS
    assert a.allreduce_fault(2, 5, 77) == (3 << 32) | (6 << 24) | 77


def test_every_declared_symbol_is_exported(pkg):
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not found")
    out = subprocess.run([nm, "-D", "--defined-only", pkg.abi.LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if l.strip()}
    declared = set(re.findall(r"CDPROBE_API\s+[\w\s\*]+?\b(cdprobe_\w+)\s*\(", open(HEADER).read()))
    assert "cdprobe_allreduce" in declared
    assert declared <= exported, declared - exported


# ---- the expected checksums ----------------------------------------------------------------------------------------
def oracle_checksum(oracle, words):
    w = np.ascontiguousarray(words, dtype=np.uint64)
    s, x = C.c_uint64(), C.c_uint64()
    oracle.lib().cdoracle_checksum(w.ctypes.data_as(C.POINTER(C.c_uint64)), len(w), C.byref(s), C.byref(x))
    return s.value, x.value


def test_output_words_restatement_by_hand():
    seed = 0x1234
    for n in (1, 2, 5):
        w = ref.output_words(seed, n, 3)
        for k in range(3):
            want = sum(int(ref.word_ref.src_words(seed, j, k, 1)[0]) for j in range(n)) % (1 << 64)
            assert int(w[k]) == want, (n, k)
    # at n = 1 the output is the rank's own pattern
    assert (ref.output_words(seed, 1, 5000) == ref.word_ref.src_words(seed, 0, 0, 5000)).all()


@pytest.fixture(scope="module")
def fold(tmp_path_factory):
    exe = tmp_path_factory.mktemp("ar") / "allreduce_fold"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-I", CSRC, os.path.join(ROOT, "tests", "c", "allreduce_fold.cc"),
                    "-o", str(exe)], check=True)

    def run(lines):
        text = "".join(" ".join(str(x) for x in l) + "\n" for l in lines)
        out = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
        assert len(out) == len(lines)
        return [[int(x) for x in l.split()] for l in out]

    return run


@pytest.mark.parametrize("n", [1, 2, 3, 8, 16])
def test_prefix_fold_and_reference_match_the_oracle(fold, oracle, n):
    """For several seeds, every prefix of the ladder and prefixes that end inside a granule: the library's fold of
    per-granule sums plus the generated tail, and the numpy reference, both equal cdoracle_checksum over the numpy sum
    of the ranks' pattern words."""
    rng = random.Random(20261015 + n)
    lines, want, refs = [], [], []
    for seed in (0xCD5EED0000000001, rng.getrandbits(64), rng.getrandbits(64)):
        words = rng.choice([70 * G + 37, 3 * G, (1 << 20) // 8 + 5 * 128 + 16])
        prefixes = sorted({s // 8 for s in ref.ladder(words * 8) if s // 8 <= words} |
                          {rng.randrange(1, words + 1) for _ in range(3)} | {G - 1, G, G + 1, words})
        out = ref.output_words(seed, n, words)
        lines.append(("F", seed, n, words, len(prefixes), *prefixes))
        want.append([v for p in prefixes for v in oracle_checksum(oracle, out[:p])])
        refs.append([v for p in prefixes for v in ref.checksum(out[:p])])
    assert fold(lines) == want
    assert refs == want


def test_corrupted_reference_moves_exactly_one_word(oracle):
    seed, n, w, mask = 0xCD5EED0000000001, 3, 4097, 1 << 17
    sizes = (4096, 32768, 65536)
    got = ref.expected_corrupted(seed, n, sizes, 2, w, mask)
    out = ref.output_words(seed, n, max(sizes) // 8)
    orig = int(ref.word_ref.src_words(seed, 2, w, 1)[0])
    out[w] = np.uint64((int(out[w]) - orig + (orig ^ mask)) % (1 << 64))
    assert got == [oracle_checksum(oracle, out[:s // 8]) for s in sizes]
    assert got[0] == ref.expected(seed, n, sizes)[0]  # the smallest prefix does not reach the word


def test_row_summary_on_hand_built_medians():
    """A row's t0_ns, peak_gbps and half_bytes are bwcurve's summary of its medians (algorithm bandwidth)."""
    sizes = [4096, 8192, 16384, 32768]
    assert ref.summary(sizes, [1000.0, 2000.0, 4000.0, 8000.0])[2] == 4096
    t0, peak, half = ref.summary(sizes, [2048.0, 2048.0, 2048.0, 4096.0])  # rates 2, 4, 8, 8
    assert (t0, peak, half) == (2048.0, 8.0, 8192)
    assert ref.summary(sizes, [0.0, 1024.0, 1024.0, 1024.0]) == (0.0, 32.0, 16384)  # a 0 median counts as rate 0


# ---- errors without a GPU -------------------------------------------------------------------------------------------
def test_allreduce_rejects_a_null_handle_and_fills_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.AllReduceT()
    t.n, t.call_seq, t.n_sizes, t.measured[0] = 77, 5, 3, 1
    assert lib.cdprobe_allreduce(None, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.reps, t.call_seq, t.n_sizes, t.row_mask) == (2, 0, a.ALLREDUCE_DEFAULT_REPS, 0, 0, 0)
    assert sum(t.measured) == 0
    assert lib.cdprobe_allreduce(None, 0, None) == a.ERR_ARG
    for reps in (1, a.ALLREDUCE_MAX_REPS + 1, 2 ** 32 - 1):
        t = a.AllReduceT()
        assert lib.cdprobe_allreduce(None, reps, C.byref(t)) == a.ERR_ARG
        assert (t.abi, t.reps) == (2, reps) and sum(t.measured) == 0
    assert lib.cdprobe_set_option(None, a.OPT_ALLREDUCE_FAULT, 1) == a.ERR_ARG


def test_wrapper_passes_its_arguments(pkg):
    a = pkg.abi
    calls = []

    class FakeLib:
        def cdprobe_allreduce(self, h, reps, out):
            calls.append((h.value, reps))
            t = out._obj
            t.abi, t.n, t.row_mask, t.reps, t.call_seq, t.n_sizes, t.path = 2, 3, 2, reps or 8, 4, 2, 2
            t.size[0], t.size[1] = 4096, 8192
            t.measured[1], t.measured[2] = 1, 1
            t.status[0], t.status[1], t.status[2] = a.ERR_STATE, a.ERR_INTEGRITY, a.ERR_TIMEOUT
            t.ns_min[1][0], t.ns_median[1][0], t.ns_max[1][0] = 1.0, 2.0, 3.0
            t.ns_median[1][1], t.sum[1][1], t.xr[1][1] = 4.0, 7, 9
            t.bad_words[1][1], t.first_bad[1][0], t.first_bad[1][1] = 1, U64_MAX, 24
            t.t0_ns[1], t.peak_gbps[1], t.half_bytes[1], t.bad_sizes[1] = 2.0, 2048.0, 4096, 2
            return a.ERR_ARG if reps > 64 else a.OK

        def cdprobe_strerror(self, rc):
            return b"invalid argument"

        def cdprobe_last_error(self):
            return b""

    p = object.__new__(pkg.Probe)
    p._lib, p._h = FakeLib(), C.c_void_p(0x1234)
    try:
        ar = p.AllReduce()
        assert calls[-1] == (0x1234, 0)
        assert (ar.n, ar.row_mask, ar.reps, ar.call_seq, ar.path, ar.sizes) == (3, 2, 8, 4, 2, [4096, 8192])
        assert ar.measured == [False, True, True]
        assert ar.status == [a.ERR_STATE, a.ERR_INTEGRITY, a.ERR_TIMEOUT]
        assert ar.ns_median[1] == [2.0, 4.0] and ar.ns_min[1] == [1.0, 0.0]
        assert ar.ns_median[0] is None and ar.ns_median[2] is None and ar.sum[2] is None  # not run; timed out
        assert ar.sum[1] == [0, 7] and ar.xr[1] == [0, 9]
        assert ar.bad_words[1] == [0, 1] and ar.first_bad[1] == [U64_MAX, 24]
        assert (ar.t0_ns[1], ar.peak_gbps[1], ar.half_bytes[1], ar.bad_sizes[1]) == (2.0, 2048.0, 4096, 2)
        p.AllReduce(reps=3)
        assert calls[-1] == (0x1234, 3)
        with pytest.raises(pkg.ProbeError) as e:
            p.AllReduce(65)
        assert e.value.code == a.ERR_ARG
        assert pkg.AllReduce is type(ar)
    finally:
        p._h = C.c_void_p()


# ---- the compiled kernel ------------------------------------------------------------------------------------------
def cuobjdump():
    return shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)


@pytest.fixture(scope="module")
def kernel(pkg):
    exe = cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([exe, "-sass", pkg.abi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for f in re.split(r"\n\s*Function : ", sass):
        if f.split("\n", 1)[0].strip().startswith("_ZN3cdp16allreduce_kernel"):
            return [t.strip() for t in re.findall(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", f)]
    pytest.fail("allreduce_kernel not in the library")


def stamp(text):
    """Index of the rep's completion stamp: the 64-bit atomic max whose value is a %globaltimer read."""
    for k, t in enumerate(text):
        m = re.match(r"(?:REDG|ATOMG)\.E\.MAX\.64\S*\s.*,\s*(R\d+)$", t)
        if m and k > 0 and re.match(rf"CS2R {m.group(1)}, SR_GLOBALTIMERLO", text[k - 1]):
            return k
    pytest.fail("no completion stamp in allreduce_kernel")


def test_every_read_path_and_the_vector_stores_are_compiled_in(kernel):
    """The TMA bulk path (UBLKCP into shared memory, completed on an mbarrier: SYNCS), the two ld/st paths (128-bit
    global loads that bypass L1), and the sum's 128-bit global stores on every path."""
    b = kernel[:stamp(kernel)]
    assert any(t.startswith("UBLKCP.S.G") for t in b)
    assert any(t.startswith("SYNCS.ARRIVE.TRANS64") for t in b)
    assert any(t.startswith("SYNCS.PHASECHK.TRANS64.TRYWAIT") for t in b)
    assert sum(t.startswith("LDG.E.NA.128") for t in b) >= 32  # 16 vectors in flight per lane, on each ld/st path
    assert sum(t.startswith("STG.E.NA.128") for t in b) >= 3 * 16  # 16 vectors per lane and unit, on each path
    assert not any(t.startswith("UBLKCP.G.S") for t in kernel)  # the sum does not leave through TMA


def test_the_closing_timer_read_follows_the_last_store(kernel):
    """The completion stamp is a %globaltimer read made after every store of the rep, the fence that waits for them,
    the CTA barrier and the CTA's (S, X) reductions; it is the value the atomic max stores."""
    mx = stamp(kernel)
    timer = mx - 1
    stores = [k for k, t in enumerate(kernel[:mx]) if t.startswith("STG.E.NA.128")]
    fence = max(k for k in range(timer) if kernel[k].startswith("MEMBAR.SC.GPU"))
    bar = max(k for k in range(timer) if kernel[k].startswith("BAR.SYNC"))
    loads = [k for k, t in enumerate(kernel[:mx]) if t.startswith(("LDG.E.NA.128", "SYNCS.PHASECHK"))]
    assert stores and loads and max(loads) < max(stores) < fence < bar < timer
    reds = [k for k in range(bar, timer) if re.match(r"(REDG|ATOMG)\.E\.(ADD|XOR)\.64", kernel[k])]
    assert len(reds) == 2


def test_ptxas_reports_no_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    proc = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                           "-c", os.path.join(CSRC, "probe_kernels.cu"), "-o", str(tmp_path / "p.o")],
                          capture_output=True, text=True, check=True)
    props = dict(re.findall(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+ bytes spill stores, "
                            r"\d+ bytes spill loads)", proc.stderr))
    ar = [k for k in props if "allreduce" in k]
    assert len(ar) == 2, proc.stderr
    assert all(props[k] == "0 bytes spill stores, 0 bytes spill loads" for k in ar), props


# ---- Go mirror ----------------------------------------------------------------------------------------------------
def test_go_allreduce_is_consistent_across_shim_and_stub():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()

    def struct(src, name):
        body = src[src.index(f"type {name} struct {{"):]
        return body[:body.index("\n}")]

    assert "func (p *Probe) AllReduce(reps int) (AllReduce, error)" in shim
    assert "func (*Probe) AllReduce(int) (AllReduce, error)" in stub
    decls = re.findall(r"^\t([A-Z]\w*(?:, [A-Z]\w*)*) ", struct(shim, "AllReduce"), re.M)
    names = {n.strip() for d in decls for n in d.split(",")}
    assert {"Sizes", "Measured", "Status", "BadSizes", "T0Ns", "PeakGBps", "HalfBytes", "NsMin", "NsMedian", "NsMax",
            "Sum", "Xr", "BadWords", "FirstBad", "RowMask", "CallSeq", "Path", "Reps"} <= names
    for n in names:
        assert re.search(rf"\b{n}\b", struct(stub, "AllReduce")), n
    # optional binding: a missing symbol does not fail cdp_load, and AllReduce reports ErrUnsupported
    assert 'dlsym(cdp_dl, "cdprobe_allreduce")' in shim and "cdp_has_allreduce() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_ar" not in required
    # the shim reads only fields the header declares
    hdr = open(HEADER).read()
    hdr_struct = hdr[hdr.index("typedef struct {", hdr.index("One-shot all-reduce across the domain")):
                     hdr.index("} cdprobe_allreduce_t;")]
    for fld in set(re.findall(r"\bar\.(\w+)", shim)):
        assert re.search(rf"\b{fld}\b", hdr_struct), fld
