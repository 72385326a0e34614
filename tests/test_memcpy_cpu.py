"""cdprobe_memcpy without a GPU: the ABI layout and option, the cell geometry of the library against the reference for
every domain shape, the reference against the oracle, the fault encoder, the argument errors, the wrapper on
hand-built results, and the Go mirror."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import memcpy_ref as ref
from conftest import ROOT
from harness import FakeLib, assert_layout, c_tool_exe, fake_probe, header_values

HEADER = os.path.join(ROOT, "include", "cdprobe.h")
U64_MAX = (1 << 64) - 1
LOCAL_DIAG = 0x4
MODES = (0, 1, 2)  # reach, sliced, full


def test_memcpy_struct_layout_matches_c(pkg, tmp_path):
    a = pkg.abi
    assert_layout(tmp_path, {"cdprobe_memcpy_t": a.MemcpyT})
    assert header_values(tmp_path, "CDPROBE_OPT_MEMCPY_FAULT") == [a.OPT_MEMCPY_FAULT] == [26]
    assert a.SYMBOLS["cdprobe_memcpy"] == (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(a.MemcpyT)])


# ---- the cell geometry ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cells(tmp_path_factory):
    exe = c_tool_exe(tmp_path_factory, "memcpy_cells.cc", csrc=["plan.cc"])

    def run(cases):
        text = "".join(" ".join(str(x) for x in c) + "\n" for c in cases)
        out = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True).stdout.split("end\n")
        got = []
        for block in out[:len(cases)]:
            head, *rows = block.strip().splitlines()
            bpp, rounds = (int(x) for x in head.split())
            got.append((bpp, rounds, [tuple(int(x) for x in r.split()) for r in rows]))
        return got

    return run


def test_cell_geometry_matches_the_reference_for_every_domain(cells, oracle):
    """For n = 1 .. 16, every mode, with and without LOCAL_DIAG, and both ops: the library copies the cells the
    reference names, in the same rounds, from the same slice into the same block."""
    cases = [(n, (3 << 20) + 128 * n, mode, flags, op) for n in range(1, 17) for mode in MODES
             for flags in (0, LOCAL_DIAG) for op in (ref.OP_READ, ref.OP_WRITE)]
    for case, (bpp, rounds, rows) in zip(cases, cells(cases)):
        n, nbytes, mode, flags, op = case
        want_bpp, want = ref.schedule(oracle, n, nbytes, mode, bool(flags & LOCAL_DIAG), op)
        assert bpp == want_bpp, case
        assert rounds == max(r for r, *_ in want) + 1, case
        assert rows == [(r, g, q, c["src_rank"], c["src_off"], c["first_word"], c["dst_rank"], c["dst_off"])
                        for r, g, q, c in want], case


def test_no_two_cells_of_a_round_land_on_the_same_bytes(oracle):
    """Within a round, every cell's destination block, [dst_off, dst_off + bpp) of dst_rank's area, is its own, and
    every block lies inside the n x bpp area."""
    for n in range(1, 17):
        for mode in MODES:
            for diag in (False, True):
                for op in (ref.OP_READ, ref.OP_WRITE):
                    bpp, sched = ref.schedule(oracle, n, 1 << 22, mode, diag, op)
                    by_round = {}
                    for r, g, q, c in sched:
                        assert c["dst_off"] + bpp <= n * bpp
                        by_round.setdefault(r, []).append((c["dst_rank"], c["dst_off"]))
                    for r, blocks in by_round.items():
                        assert len(blocks) == len(set(blocks)), (n, mode, diag, op, r)


def test_pull_and_push_of_a_pair_move_the_same_slice():
    """A pull by g from j moves what a push by j to g moves: the slice g reads from j, into block j of g's area."""
    for n, mode in ((2, 1), (5, 1), (8, 2), (16, 0)):
        bpp = 4096
        for g in range(n):
            for j in range(n):
                assert ref.cell(n, bpp, mode, ref.OP_READ, g, j) == ref.cell(n, bpp, mode, ref.OP_WRITE, j, g)


@pytest.mark.parametrize("nbytes", [4096, 4096 + 128, 16384 * 3 + 256, 1 << 20])
def test_reference_prefix_checksums_equal_the_oracle(oracle, nbytes):
    seed = 0xCD5EED0000000001
    for n, mode, op, g, j in ((1, 1, ref.OP_READ, 0, 0), (4, 1, ref.OP_WRITE, 3, 1), (16, 2, ref.OP_READ, 2, 15)):
        c = ref.cell(n, nbytes, mode, op, g, j)
        for s in ref.ladder(nbytes):
            assert ref.checksum(ref.words(seed, c, s)) == oracle.src_checksum(seed, c["src_rank"], c["first_word"],
                                                                               s // 8), (n, op, g, j, s)


def test_expected_uses_the_oracle_for_big_prefixes(oracle):
    seed = 7
    c = ref.cell(2, 1 << 30, 1, ref.OP_WRITE, 0, 1)
    sizes = [4096, ref.REF_MAX_BYTES, 2 * ref.REF_MAX_BYTES]
    got = ref.expected(oracle, seed, c, sizes)
    assert got[-1] == oracle.src_checksum(seed, 0, c["first_word"], sizes[-1] // 8)
    assert got[0] == ref.checksum(ref.words(seed, c, 4096))


# ---- the option --------------------------------------------------------------------------------------------------------
def test_fault_encoder_and_its_refusals(pkg):
    a = pkg.abi
    assert a.memcpy_fault(2, 0, 5, 77) == (3 << 40) | (1 << 32) | (6 << 24) | 77
    assert a.memcpy_fault(0, 15, 0, 9, mode=1) == (1 << 48) | (1 << 40) | (16 << 32) | (1 << 24) | 9
    v = a.memcpy_fault(254, 254, 254, (1 << 24) - 1, 1)
    assert (v >> 48, (v >> 40) & 0xff, (v >> 32) & 0xff, (v >> 24) & 0xff, v & 0xffffff) == \
        (1, 255, 255, 255, (1 << 24) - 1)
    for bad in (dict(mode=2), dict(word=1 << 24), dict(issuer=255), dict(k=-1)):
        args = dict(issuer=0, target=1, k=0, word=0, mode=0) | bad
        with pytest.raises(ValueError):
            a.memcpy_fault(**args)


# ---- errors without a GPU -----------------------------------------------------------------------------------------------
def test_memcpy_rejects_a_null_handle_and_fills_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.MemcpyT()
    t.n, t.call_seq, t.n_sizes, t.measured[0] = 77, 5, 3, 1
    assert lib.cdprobe_memcpy(None, a.OP_READ, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.reps, t.op, t.call_seq, t.n_sizes, t.row_mask) == \
        (2, 0, a.MEMCPY_DEFAULT_REPS, a.OP_READ, 0, 0, 0)
    assert sum(t.measured) == 0
    assert lib.cdprobe_memcpy(None, a.OP_WRITE, 0, None) == a.ERR_ARG
    for op, reps in ((a.OP_WRITE, 1), (3, a.MEMCPY_MAX_REPS + 1), (0, 2 ** 32 - 1)):
        t = a.MemcpyT()
        assert lib.cdprobe_memcpy(None, op, reps, C.byref(t)) == a.ERR_ARG
        assert (t.abi, t.reps, t.op) == (2, reps, op) and sum(t.measured) == 0
    assert lib.cdprobe_set_option(None, a.OPT_MEMCPY_FAULT, 1) == a.ERR_ARG


def test_from_c_on_hand_built_results(pkg):
    a = pkg.abi
    t = a.MemcpyT()
    t.abi, t.n, t.row_mask, t.reps, t.op, t.call_seq, t.n_sizes, t.area_bytes, t.ms = 2, 3, 0b110, 4, 2, 9, 2, 6 << 20, 1.5
    t.size[0], t.size[1] = 4096, 8192
    ok, bad, late, down = 1 * 16 + 0, 1 * 16 + 2, 2 * 16 + 0, 2 * 16 + 1
    t.measured[ok], t.measured[bad], t.measured[late] = 1, 1, 1
    t.status[bad], t.status[late], t.status[down] = a.ERR_INTEGRITY, a.ERR_TIMEOUT, a.ERR_STATE
    t.ns_min[ok][0], t.ns_median[ok][0], t.ns_max[ok][0] = 1.0, 2.0, 3.0
    t.t0_ns[ok], t.peak_gbps[ok], t.half_bytes[ok] = 2.0, 8.0, 4096
    t.first_bad[ok][0], t.first_bad[ok][1] = U64_MAX, U64_MAX
    t.bad_sizes[bad], t.bad_words[bad][1], t.first_bad[bad][0], t.first_bad[bad][1] = 2, 1024, U64_MAX, 0
    t.sum[bad][1], t.xr[bad][1] = 7, 9
    m = pkg.Memcpy.from_c(t)
    assert (m.n, m.row_mask, m.reps, m.op, m.call_seq, m.area_bytes, m.sizes, m.ms) == \
        (3, 0b110, 4, 2, 9, 6 << 20, [4096, 8192], 1.5)
    assert m.measured[1][0] and m.status[1][0] == 0 and m.ns_median[1][0] == [2.0, 0.0]
    assert (m.t0_ns[1][0], m.peak_gbps[1][0], m.half_bytes[1][0]) == (2.0, 8.0, 4096)
    assert m.bad_words[1][0] == [0, 0] and m.first_bad[1][0] == [U64_MAX, U64_MAX]
    assert m.status[1][2] == a.ERR_INTEGRITY and m.bad_sizes[1][2] == 2
    assert m.bad_words[1][2] == [0, 1024] and m.first_bad[1][2] == [U64_MAX, 0]
    assert m.sum[1][2] == [0, 7] and m.xr[1][2] == [0, 9]
    assert m.measured[2][0] and m.status[2][0] == a.ERR_TIMEOUT and m.ns_median[2][0] is None
    assert m.bad_words[2][0] is None
    assert not m.measured[2][1] and m.status[2][1] == a.ERR_STATE and m.sum[2][1] is None
    assert m.ns_min[0][0] is None and m.status[0][0] == 0


def test_wrapper_passes_its_arguments(pkg):
    a = pkg.abi
    calls = []

    class Lib(FakeLib):
        def cdprobe_memcpy(self, h, op, reps, out):
            calls.append((h.value, op, reps))
            t = out._obj
            t.abi, t.n, t.reps, t.op = 2, 2, reps or 8, op
            return a.ERR_ARG if reps > 64 else a.OK

    with fake_probe(pkg, Lib()) as p:
        m = p.Memcpy(a.OP_WRITE)
        assert calls[-1] == (0x1234, a.OP_WRITE, 0) and (m.op, m.reps, m.n) == (a.OP_WRITE, 8, 2)
        p.Memcpy(a.OP_READ, reps=3)
        assert calls[-1] == (0x1234, a.OP_READ, 3)
        with pytest.raises(pkg.ProbeError) as e:
            p.Memcpy(a.OP_READ, 65)
        assert e.value.code == a.ERR_ARG
        assert pkg.Memcpy is type(m)


# ---- Go mirror ------------------------------------------------------------------------------------------------------
def test_go_memcpy_is_consistent_across_shim_and_stub():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()

    def struct(src, name):
        body = src[src.index(f"type {name} struct {{"):]
        return body[:body.index("\n}")]

    assert "func (p *Probe) Memcpy(op uint32, reps int) (Memcpy, error)" in shim
    assert "func (*Probe) Memcpy(uint32, int) (Memcpy, error)" in stub
    decls = re.findall(r"^\t([A-Z]\w*(?:, [A-Z]\w*)*) ", struct(shim, "Memcpy"), re.M)
    names = {n.strip() for d in decls for n in d.split(",")}
    assert {"Sizes", "Measured", "Status", "T0Ns", "PeakGBps", "HalfBytes", "NsMin", "NsMedian", "NsMax", "BadSizes",
            "BadWords", "FirstBad", "Sum", "Xr", "RowMask", "CallSeq", "Op", "Reps", "AreaBytes"} <= names
    for n in names:
        assert re.search(rf"\b{n}\b", struct(stub, "Memcpy")), n
    assert 'dlsym(cdp_dl, "cdprobe_memcpy")' in shim and "cdp_has_memcpy() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_mc" not in required
    hdr = open(HEADER).read()
    hdr_struct = hdr[hdr.index("typedef struct {", hdr.index("Copy-engine bandwidth versus transfer size per ordered")):
                     hdr.index("} cdprobe_memcpy_t;")]
    for fld in set(re.findall(r"\bmc\.(\w+)", shim)):
        assert re.search(rf"\b{fld}\b", hdr_struct), fld
