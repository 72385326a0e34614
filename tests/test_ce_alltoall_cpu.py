"""cdprobe_ce_alltoall without a GPU: the ABI layout and option, where its flag lines sit in the Ctrl granule, the flag
values, the hardware-queue arithmetic against the reference for every small domain, the fault encoder, the argument
errors, the wrapper on hand-built results, and the Go mirror."""
import ctypes as C
import os
import re
import subprocess

import pytest

import ce_alltoall_ref as ref
from conftest import ROOT
from harness import FakeLib, assert_layout, c_tool_exe, fake_probe, header_values

HEADER = os.path.join(ROOT, "include", "cdprobe.h")
U64_MAX = (1 << 64) - 1


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    """run(lines) over tests/c/ce_a2a_host.cc, linked with plan.cc: one line of integers per input line."""
    exe = c_tool_exe(tmp_path_factory, "ce_a2a_host.cc", csrc=["plan.cc"])

    def run(lines):
        text = "".join(" ".join(str(x) for x in l) + "\n" for l in lines)
        out = subprocess.run([exe], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
        assert len(out) == len(lines)
        return [[int(x) for x in l.split()] for l in out]

    return run


def test_struct_layout_matches_c(pkg, tmp_path):
    a = pkg.abi
    assert_layout(tmp_path, {"cdprobe_ce_alltoall_t": a.CeAllToAllT})
    assert header_values(tmp_path, "CDPROBE_OPT_CE_ALLTOALL_FAULT", "CDPROBE_ABI_VERSION") == \
        [a.OPT_CE_ALLTOALL_FAULT, a.ABI_VERSION] == [28, 2]
    assert a.SYMBOLS["cdprobe_ce_alltoall"] == \
        (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(a.CeAllToAllT)])


def test_flag_lines_sit_after_the_nvls_lines_inside_the_ctrl_granule(host):
    [[off, nvls, lines, ctrl]] = host(["O"])
    assert off == 82 << 10 and off == nvls + lines and lines == 16 * 128
    assert off % 128 == 0 and off + lines <= ctrl


def test_flag_values_rise_along_call_size_and_rep(host):
    for reps in (1, 8, 64):
        seq = [(c, k, r) for c in (1, 2, 3) for k in range(24) for r in range(reps + 1)]
        got = [v for [v] in host([("V", c, k, r, reps) for c, k, r in seq])]
        assert got == [ref.value(c, k, r, reps) for c, k, r in seq]
        assert all(a < b for a, b in zip(got, got[1:])), reps
        # every value of a call lies below every value of the next, so no GEQ wait of the next is satisfied early
        for c in (1, 2):
            assert max(v for v, (cc, _, _) in zip(got, seq) if cc == c) < \
                min(v for v, (cc, _, _) in zip(got, seq) if cc == c + 1)
    # the largest ladder and rep count fit the low 16 bits
    assert ref.value(1, 23, 64, 64) < (2 << 16)


def test_queue_count_matches_the_reference(host):
    cases = []
    for n in range(1, 17):
        for diag in (False, True):
            if n == 1 and not diag:
                continue  # a one-rank domain always has its loop-back slice
            for devices in range(1, 5):
                for procs in (1, 2):
                    if n % procs:
                        continue
                    n_local = n // procs
                    cases.append((n, diag, [(i * 7 + 3) % devices for i in range(n_local)]))
    got = host([("Q", n, int(d), len(o), *o) for n, d, o in cases])
    for (n, diag, ords), (need, worst) in zip(cases, got):
        assert (need, worst) == ref.queues(n, diag, ords), (n, diag, ords)
    # the shapes the GPU suite and the tool rely on: one rank fits the default 8, eight ranks on one device do not
    assert ref.queues(1, True, [0]) == (2, 0) and ref.queues(2, False, [0, 0]) == (4, 0)
    assert ref.queues(8, False, [0] * 8) == (64, 0) and ref.queues(8, True, [0, 0]) == (18, 0)


def test_fault_encoder_and_its_refusals(pkg):
    a = pkg.abi
    assert a.ce_alltoall_fault(2, 0, 5, 77) == (3 << 40) | (1 << 32) | (6 << 24) | 77
    assert a.ce_alltoall_fault(0, 15, 0, 9, mode=2) == (2 << 48) | (1 << 40) | (16 << 32) | (1 << 24) | 9
    v = a.ce_alltoall_fault(254, 254, 254, (1 << 24) - 1, 1)
    assert (v >> 48, (v >> 40) & 0xff, (v >> 32) & 0xff, (v >> 24) & 0xff, v & 0xffffff) == \
        (1, 255, 255, 255, (1 << 24) - 1)
    for bad in (dict(mode=3), dict(arg=1 << 24), dict(issuer=255), dict(k=-1), dict(target=-1)):
        with pytest.raises(ValueError):
            a.ce_alltoall_fault(**(dict(issuer=0, target=1, k=0, arg=0, mode=0) | bad))
    assert ref.fault_words(0, 4096, 5) == (1, 40) and ref.fault_words(1, 4096, 5) == (512, 0)
    assert ref.fault_words(2, 4096, 5) == (0, U64_MAX)


def test_rejects_a_null_handle_and_fills_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.CeAllToAllT()
    t.n, t.call_seq, t.n_sizes, t.measured[0] = 77, 5, 3, 1
    assert lib.cdprobe_ce_alltoall(None, a.OP_READ, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.reps, t.op, t.call_seq, t.n_sizes, t.row_mask) == \
        (2, 0, a.CE_ALLTOALL_DEFAULT_REPS, a.OP_READ, 0, 0, 0)
    assert sum(t.measured) == 0
    assert lib.cdprobe_ce_alltoall(None, a.OP_WRITE, 0, None) == a.ERR_ARG
    for op, reps in ((a.OP_WRITE, 1), (3, a.CE_ALLTOALL_MAX_REPS + 1), (0, 2 ** 32 - 1)):
        t = a.CeAllToAllT()
        assert lib.cdprobe_ce_alltoall(None, op, reps, C.byref(t)) == a.ERR_ARG
        assert (t.abi, t.reps, t.op) == (2, reps, op) and sum(t.measured) == 0
    assert lib.cdprobe_set_option(None, a.OPT_CE_ALLTOALL_FAULT, 1) == a.ERR_ARG


def test_from_c_on_hand_built_results(pkg):
    a = pkg.abi
    t = a.CeAllToAllT()
    t.abi, t.n, t.row_mask, t.reps, t.op, t.call_seq, t.n_sizes, t.area_bytes, t.ms = 2, 3, 0b010, 4, 2, 9, 2, 6 << 20, 1.5
    t.size[0], t.size[1] = 4096, 8192
    t.measured[1], t.blocks[1], t.t0_ns[1], t.peak_gbps[1], t.half_bytes[1] = 1, 2, 2.0, 8.0, 4096
    t.ns_min[1][0], t.ns_median[1][0], t.ns_max[1][0] = 1.0, 2.0, 3.0
    t.status[0], t.status[2] = 0, 0
    # a push: rank 1 issues (1, 0) and (1, 2) and owns the blocks (0, 1) and (2, 1)
    t.copy_ns_median[1 * 16 + 0][0], t.copy_ns_median[1 * 16 + 2][1] = 1.5, 2.5
    ok, bad = 0 * 16 + 1, 2 * 16 + 1
    t.cell_measured[ok], t.cell_measured[bad] = 1, 1
    t.cell_status[bad], t.bad_sizes[bad] = a.ERR_INTEGRITY, 2
    t.first_bad[ok][0], t.first_bad[ok][1], t.first_bad[bad][0], t.first_bad[bad][1] = U64_MAX, U64_MAX, U64_MAX, 8
    t.bad_words[bad][1], t.sum[bad][1], t.xr[bad][1] = 1024, 7, 9
    t.cell_status[1 * 16 + 0] = 0
    m = pkg.CeAllToAll.from_c(t)
    assert (m.n, m.row_mask, m.reps, m.op, m.call_seq, m.area_bytes, m.sizes, m.ms) == \
        (3, 0b010, 4, 2, 9, 6 << 20, [4096, 8192], 1.5)
    assert m.measured == [False, True, False] and m.blocks == [None, 2, None]
    assert (m.t0_ns[1], m.peak_gbps[1], m.half_bytes[1]) == (2.0, 8.0, 4096)
    assert m.ns_median[1] == [2.0, 0.0] and m.ns_min[0] is None
    assert m.copy_ns_median[1][0] == [1.5, 0.0] and m.copy_ns_median[1][2] == [0.0, 2.5]
    assert m.copy_ns_median[1][1] is None and m.copy_ns_median[0][1] is None
    assert m.cell_measured[0][1] and m.cell_status[0][1] == 0 and m.bad_words[0][1] == [0, 0]
    assert m.first_bad[0][1] == [U64_MAX, U64_MAX]
    assert m.cell_status[2][1] == a.ERR_INTEGRITY and m.bad_sizes[2][1] == 2 and m.bad_words[2][1] == [0, 1024]
    assert m.first_bad[2][1] == [U64_MAX, 8] and m.sum[2][1] == [0, 7] and m.xr[2][1] == [0, 9]
    assert not m.cell_measured[1][0] and m.sum[1][0] is None


def test_wrapper_passes_its_arguments(pkg):
    a = pkg.abi
    calls = []

    class Lib(FakeLib):
        def cdprobe_ce_alltoall(self, h, op, reps, out):
            calls.append((h.value, op, reps))
            t = out._obj
            t.abi, t.n, t.reps, t.op = 2, 2, reps or 8, op
            return a.ERR_UNSUPPORTED if reps == 7 else a.ERR_ARG if reps > 64 else a.OK

    with fake_probe(pkg, Lib()) as p:
        m = p.CeAllToAll(a.OP_WRITE)
        assert calls[-1] == (0x1234, a.OP_WRITE, 0) and (m.op, m.reps, m.n) == (a.OP_WRITE, 8, 2)
        p.CeAllToAll(a.OP_READ, reps=3)
        assert calls[-1] == (0x1234, a.OP_READ, 3)
        with pytest.raises(pkg.ProbeError) as e:
            p.CeAllToAll(a.OP_READ, 65)
        assert e.value.code == a.ERR_ARG
        rc, t = p.ce_alltoall_raw(a.OP_READ, 7)
        assert rc == a.ERR_UNSUPPORTED and t.reps == 7
        assert pkg.CeAllToAll is type(m)


def test_go_mirror_is_consistent_across_shim_and_stub():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()

    def struct(src, name):
        body = src[src.index(f"type {name} struct {{"):]
        return body[:body.index("\n}")]

    assert "func (p *Probe) CeAllToAll(op uint32, reps int) (CeAllToAll, error)" in shim
    assert "func (*Probe) CeAllToAll(uint32, int) (CeAllToAll, error)" in stub
    decls = re.findall(r"^\t([A-Z]\w*(?:, [A-Z]\w*)*) ", struct(shim, "CeAllToAll"), re.M)
    names = {n.strip() for d in decls for n in d.split(",")}
    assert {"Sizes", "Measured", "Status", "Blocks", "T0Ns", "PeakGBps", "HalfBytes", "NsMin", "NsMedian", "NsMax",
            "CellMeasured", "CellStatus", "BadSizes", "CopyNsMedian", "BadWords", "FirstBad", "Sum", "Xr", "RowMask",
            "CallSeq", "Op", "Reps", "AreaBytes", "N", "Ms"} <= names
    for n in names:
        assert re.search(rf"\b{n}\b", struct(stub, "CeAllToAll")), n
    assert 'dlsym(cdp_dl, "cdprobe_ce_alltoall")' in shim and "cdp_has_ce_alltoall() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_cea" not in required
    hdr = open(HEADER).read()
    hdr_struct = hdr[hdr.index("typedef struct {", hdr.index("Copy-engine all-to-all across the domain (cdprobe_ce")):
                     hdr.index("} cdprobe_ce_alltoall_t;")]
    for fld in set(re.findall(r"\bca\.(\w+)", shim)):
        assert re.search(rf"\b{fld}\b", hdr_struct), fld
    # the daemons do not call it
    for dirpath, _, files in os.walk(os.path.join(ROOT, "integration", "cmd")):
        for f in files:
            if f.endswith(".go"):
                assert "CeAllToAll" not in open(os.path.join(dirpath, f)).read(), f
