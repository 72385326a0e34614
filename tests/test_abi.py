"""C-ABI checks that need no GPU: the library loads, exports every symbol include/cdprobe.h
declares, the ctypes mirror has the C layout, host-only entry points agree with the oracle,
and the product path fails loudly (no CPU fallback) when there is no CUDA device."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest

from conftest import ROOT, gpu_count
from harness import FakeLib, assert_layout, declared_symbols, fake_probe


def test_exports_every_declared_symbol(pkg):
    declared = declared_symbols()
    assert declared == set(pkg.abi.SYMBOLS), declared ^ set(pkg.abi.SYMBOLS)
    lib = pkg.abi.load_library()
    for name in declared:
        assert getattr(lib, name) is not None
    out = subprocess.run(["nm", "-D", "--defined-only", pkg.abi.LIB_PATH], capture_output=True, text=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    assert declared <= exported
    # nothing but the ABI leaks out of the library
    assert {e for e in exported if not e.startswith("cdprobe_")} == set()


def test_abi_version_and_strerror(pkg):
    lib = pkg.abi.load_library()
    assert lib.cdprobe_abi_version() == pkg.abi.ABI_VERSION == 2
    assert lib.cdprobe_strerror(0) == b"ok"
    for code in range(-10, 0):
        assert lib.cdprobe_strerror(code) not in (b"", b"unknown cdprobe error")
    assert lib.cdprobe_strerror(-99) == b"unknown cdprobe error"


def test_struct_layout_matches_c(pkg, tmp_path):
    """sizeof/offsetof of every ABI struct, taken from the header by gcc, equal the ctypes mirror."""
    a = pkg.abi
    structs = {"cdprobe_config_t": a.ConfigT, "cdprobe_result_t": a.ResultT, "cdprobe_info_t": a.InfoT,
               "cdprobe_plan_t": a.PlanT, "cdprobe_trace_t": a.TraceT,
               "cdprobe_topology_t": a.TopologyT, "cdprobe_schedule_t": a.ScheduleT}
    assert_layout(tmp_path, structs)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("n", list(range(1, 17)))
def test_plan_matches_oracle(pkg, oracle, n, mode):
    for nbytes in (1 << 30, 64 << 20, 1000003 * 128 + 77):
        for flags in (0, pkg.abi.FLAG_LOCAL_DIAG):
            p = pkg.plan(n, nbytes, mode, flags)
            o = oracle.plan(n, nbytes, mode, bool(flags))
            assert p.bytes_per_pair == o.bytes_per_pair
            assert (p.rounds, p.n_slots, p.n_slices) == (o.rounds, o.n_slots, o.n_slices)
            assert (p.src_bytes, p.land_bytes) == (o.src_bytes, o.land_bytes)
            assert [list(r) for r in p.partner] == [list(r) for r in o.partner]


def test_plan_matches_golden(pkg, golden):
    for g in golden["plans"]:
        p = pkg.plan(g["n"], g["bytes"], g["mode"], pkg.abi.FLAG_LOCAL_DIAG if (g["diag"] and g["n"] > 1) else 0)
        assert p.bytes_per_pair == g["bytes_per_pair"]
        assert [[p.partner[r][i] for i in range(g["n"])] for r in range(g["rounds"])] == g["partner"]


def test_plan_rejects_bad_arguments(pkg):
    lib = pkg.abi.load_library()
    p = pkg.abi.PlanT()
    assert lib.cdprobe_plan(0, 1 << 30, 1, 0, C.byref(p)) == pkg.abi.ERR_ARG
    assert lib.cdprobe_plan(17, 1 << 30, 1, 0, C.byref(p)) == pkg.abi.ERR_ARG
    assert lib.cdprobe_plan(8, 1 << 30, 3, 0, C.byref(p)) == pkg.abi.ERR_ARG
    assert lib.cdprobe_plan(8, 100, 1, 0, C.byref(p)) == pkg.abi.ERR_ARG  # < 128 B per pair
    assert lib.cdprobe_plan(8, 1 << 30, 1, 0, None) == pkg.abi.ERR_ARG


def test_open_rejects_bad_abi_and_null(pkg):
    lib = pkg.abi.load_library()
    h = C.c_void_p()
    c = pkg.Config(bytes=1 << 20).to_c()
    c.abi = 99
    assert lib.cdprobe_open(C.byref(c), C.byref(h)) == pkg.abi.ERR_ABI
    assert lib.cdprobe_open(None, C.byref(h)) == pkg.abi.ERR_ARG
    assert lib.cdprobe_run(None, None) == pkg.abi.ERR_ARG
    lib.cdprobe_close(None)  # must be a no-op


def test_corrupt_landing_null_handle_and_wrapper_packing(pkg):
    """cdprobe_corrupt_landing refuses a null handle; Probe.CorruptLanding hands the library the local rank, the
    target, the count and the (word, mask) pairs as two uint64 arrays, [] as n = 0, and raises on an error code."""
    a = pkg.abi
    lib = a.load_library()
    assert a.SYMBOLS["cdprobe_corrupt_landing"] == (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                                              C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)])
    w, m = (C.c_uint64 * 1)(3), (C.c_uint64 * 1)(1)
    assert lib.cdprobe_corrupt_landing(None, 0, 1, 1, w, m) == a.ERR_ARG
    assert lib.cdprobe_corrupt_landing(None, 0, 1, 0, None, None) == a.ERR_ARG

    calls = []

    class Lib(FakeLib):
        def cdprobe_corrupt_landing(self, h, local, target, n, word, mask):
            calls.append((h.value, local, target, n, [word[e] for e in range(n)], [mask[e] for e in range(n)]))
            return a.ERR_ARG if n > 8 else a.OK

    with fake_probe(pkg, Lib()) as p:
        p.CorruptLanding(1, 3, [(0, 1), (1 << 40, (1 << 63) | 5)])
        p.CorruptLanding(0, 0, [])
        assert calls == [(0x1234, 1, 3, 2, [0, 1 << 40], [1, (1 << 63) | 5]), (0x1234, 0, 0, 0, [], [])]
        with pytest.raises(pkg.ProbeError) as e:
            p.CorruptLanding(0, 1, [(k, 1) for k in range(9)])
        assert e.value.code == a.ERR_ARG and calls[-1][3] == 9


@pytest.mark.skipif(gpu_count() > 0, reason="this box has a GPU; the loud-failure path needs a CPU-only box")
def test_open_fails_loudly_without_a_gpu(pkg):
    """No CUDA driver => CDPROBE_ERR_NO_DEVICE with a reason; there is no CPU fallback to fall into."""
    with pytest.raises(pkg.ErrUnsupported) as e:
        pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 20))
    assert e.value.code == pkg.abi.ERR_NO_DEVICE
    assert e.value.detail  # says which CUDA call refused


def test_product_does_not_reference_the_oracle():
    """The product tree must not import, link or mention the oracle (it is test infrastructure)."""
    pkgdir = os.path.join(ROOT, "k8s-dra-driver-gpu_b200")
    for dirpath, _, files in os.walk(pkgdir):
        for f in files:
            if f.endswith((".py", ".cc", ".cu", ".h", ".cuh")):
                text = open(os.path.join(dirpath, f), errors="replace").read()
                assert "cdoracle" not in text and "libcdoracle" not in text, f
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, re.M), f
    out = subprocess.run(["ldd", os.path.join(pkgdir, "libcdprobe.so")], capture_output=True, text=True).stdout
    assert "cdoracle" not in out and "libcuda" not in out and "nvidia-ml" not in out  # NVML/driver are dlopen'ed lazily


def test_gate_arithmetic_without_a_gpu(pkg):
    """cdprobe_gate: the verdict's bandwidth threshold as host arithmetic (include/cdprobe.h: link_peak_gbps).
    Default reference = nominal NVLink 4 rate (450 GB/s per direction) de-rated for the 6 us of a phase's ramp and drain."""
    import pytest

    GIB = 1 << 30
    r, w = pkg.gate(pkg.Config(bytes=GIB), 8)                      # the headline config: defaults
    bpp = GIB // 7 // 128 * 128
    assert r == pytest.approx(0.65 * bpp / (bpp / 450.0 + 6000.0), rel=1e-5)
    assert w == pytest.approx(0.65 * bpp / (bpp / 450.0 + 6000.0), rel=1e-5)
    assert 285 < r < 290 and 285 < w < 290
    r1, w1 = pkg.gate(pkg.Config(bytes=GIB, flags=pkg.abi.FLAG_UNIDIRECTIONAL), 8)
    assert r1 == pytest.approx(0.65 * bpp / (bpp / 450.0 + 6000.0), rel=1e-5) and w1 == pytest.approx(r1, rel=1e-6)
    assert pkg.gate(pkg.Config(bytes=GIB, min_fraction=0.85, link_peak_gbps=900.0), 8) == (pytest.approx(765.0), pytest.approx(765.0))
    assert pkg.gate(pkg.Config(bytes=GIB, link_peak_gbps=900.0), 8) == (pytest.approx(585.0), pytest.approx(585.0))  # absolute rule
    assert pkg.gate(pkg.Config(bytes=GIB), 1) == (0.0, 0.0)        # loop-back: HBM speed is not a fabric property
    assert pkg.gate(pkg.Config(bytes=GIB, mode=pkg.abi.MODE_REACH_ONLY), 8) == (0.0, 0.0)
    small = pkg.gate(pkg.Config(bytes=16 << 20), 8)[0]             # small slices: the fixed overhead dominates, the gate follows
    assert small < 0.75 * r
    with pytest.raises(pkg.ProbeError):
        pkg.gate(pkg.Config(bytes=GIB, min_fraction=-1.0), 8)
