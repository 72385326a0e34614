"""cdprobe_latency without a GPU: the ABI layout, the chase of probe_types.h against the Python restatement in
tests/latency_ref.py, the argument errors, the compiled kernel's loads and timer order, and the Go mirror."""
import ctypes as C
import os
import random
import re

import pytest

import latency_ref as ref
from conftest import ROOT
from harness import assert_layout, c_tool
from kernel_tools import kernel_sass

HEADER = os.path.join(ROOT, "include", "cdprobe.h")
SEED = 0xCD5EED0000000001


def test_latency_struct_layout_matches_c(pkg, tmp_path):
    a = pkg.abi
    assert_layout(tmp_path, {"cdprobe_latency_t": a.LatencyT})
    assert "cdprobe_latency" in a.SYMBOLS


# ---- the chase: probe_types.h against the restatement ------------------------------------------------------------
@pytest.fixture(scope="module")
def chain(tmp_path_factory):
    run = c_tool(tmp_path_factory, "latency_chain.cc")
    return lambda cases: [tuple(r) for r in run(cases)]


def restated(seed, i, j, first, lines, hops, reps):
    line = ref.start_line(seed, i, j, reps, lines)
    for h, (_, v) in enumerate(ref.chase(seed, i, j, first, lines, reps, hops)):
        line = ref.next_line(v, h, lines)
    return ref.digest(seed, i, j, first, lines, hops, reps), ref.start_line(seed, i, j, 0, lines), line


def test_chase_matches_the_restatement(chain):
    rng = random.Random(20261015)
    cases = []
    for lines in (1, 12345, 1 << 23):
        for hops in (1, 2, 63, 64, 65, 1000):
            i, j = rng.randrange(16), rng.randrange(16)
            first = rng.randrange(16) * lines * ref.LINE_WORDS
            cases.append((SEED, i, j, first, lines, hops, rng.choice((1, 2, 8))))
    cases += [(SEED, 15, 15, 15 * (1 << 23) * 16, 1 << 23, 1 << 16, 1),  # the largest ranks, 2^16 hops
              (SEED, 0, 15, 0, 12345, 1 << 16, 1),
              (1, 15, 0, 0, 1, 1 << 16, 1),
              (rng.getrandbits(64), 7, 3, 0, 8191, 5000, 64)]
    got = chain(cases)
    for c, g in zip(cases, got):
        assert g == restated(*c), c


def test_every_line_lies_inside_the_region():
    for lines in (1, 3, 12345, 1 << 23):
        seen = [line for r in range(3) for line, _ in ref.chase(SEED, 2, 5, 0, lines, r, 500)]
        assert all(0 <= line < lines for line in seen)
        if lines == 1:
            assert set(seen) == {0}
    # a corrupted word still leads to a line inside the region
    for v in (0, 1, ref.M64, ref.GOLDEN):
        for lines in (1, 12345, 1 << 23):
            assert 0 <= ref.next_line(v, 0, lines) < lines and 0 <= ref.next_line(v, (1 << 20) - 1, lines) < lines


def test_restatement_reads_the_pattern_table():
    lines, first = 97, 4 * 97 * 16
    table = ref.region_words(SEED, 3, first, lines)
    for line, v in ref.chase(SEED, 1, 3, first, lines, 1, 300):
        assert int(table[ref.LINE_WORDS * line]) == v


def test_hop_index_keeps_a_chase_out_of_a_fixed_cycle():
    """Without h in the next-line mix, a chase that revisits a line would repeat its path from there."""
    lines = 64
    path = [line for line, _ in ref.chase(SEED, 0, 0, 0, lines, 0, 400)]
    revisits = [h for h in range(1, len(path)) if path[h] in path[:h]]
    assert revisits  # 400 hops over 64 lines revisit
    h = revisits[0]
    k = path.index(path[h])
    assert path[h:h + 20] != path[k:k + 20]


# ---- errors without a GPU -------------------------------------------------------------------------------------------
def test_latency_rejects_a_null_handle_and_fills_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.LatencyT()
    t.n = 77
    assert lib.cdprobe_latency(None, 0, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.hops, t.reps, t.row_mask) == (2, 0, a.LATENCY_DEFAULT_HOPS, a.LATENCY_DEFAULT_REPS, 0)
    assert lib.cdprobe_latency(None, 0, 0, None) == a.ERR_ARG
    for hops, reps in ((a.LATENCY_MAX_HOPS + 1, 1), (1, a.LATENCY_MAX_REPS + 1), (2 ** 32 - 1, 2 ** 32 - 1)):
        t = a.LatencyT()
        assert lib.cdprobe_latency(None, hops, reps, C.byref(t)) == a.ERR_ARG
        assert t.abi == 2 and sum(t.measured) == 0


# ---- the compiled kernel ------------------------------------------------------------------------------------------
def test_chase_loads_are_strong_sys_and_the_closing_timer_follows_their_use(pkg):
    """Every load of the chase is LDG.E.64.STRONG.SYS (ld.relaxed.sys: no L1); a timer read precedes the first load,
    the loaded register is used before the loop branches, and the closing timer read comes after the hop loop."""
    addr, text = kernel_sass(pkg.abi.LIB_PATH, "latency_kernel")
    loads = [k for k, t in enumerate(text) if "LDG" in t or re.search(r"\bLD\b", t)]
    assert len(loads) == 1 and text[loads[0]].startswith("LDG.E.64.STRONG.SYS"), [text[k] for k in loads]
    ld = loads[0]
    dst = int(re.match(r"LDG\.E\.64\.STRONG\.SYS R(\d+),", text[ld]).group(1))
    regs = {f"R{dst}", f"R{dst + 1}"}
    timers = [k for k, t in enumerate(text) if "SR_GLOBALTIMER" in t]
    assert any(k < ld for k in timers)  # the opening read
    # the first instruction after the load that reads its result comes before any branch
    use = next(k for k in range(ld + 1, len(text))
               if regs & set(re.findall(r"R\d+\b", text[k].split(",", 1)[1] if "," in text[k] else "")))
    assert not any("BRA" in text[k] for k in range(ld + 1, use)), text[ld:use + 1]
    # the hop loop's backward branch, and the closing timer read after it
    back = [k for k, t in enumerate(text) if "BRA" in t and (m := re.search(r"BRA (?:P\d, |!?P\d, )?0x([0-9a-f]+)", t))
            and int(m.group(1), 16) <= addr[ld] and k > ld]
    assert back
    assert any(k > back[0] for k in timers)


# ---- Go mirror ----------------------------------------------------------------------------------------------------
def test_go_latency_is_consistent_across_shim_and_stub():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()

    def struct(src, name):
        body = src[src.index(f"type {name} struct {{"):]
        return body[:body.index("\n}")]

    assert "func (p *Probe) Latency(hops, reps int) (Latency, error)" in shim
    assert "func (*Probe) Latency(int, int) (Latency, error)" in stub
    decls = re.findall(r"^\t([A-Z]\w*(?:, [A-Z]\w*)*) ", struct(shim, "Latency"), re.M)
    names = {n.strip() for d in decls for n in d.split(",")}
    assert {"Measured", "Status", "NsMin", "NsMedian", "NsMax", "Digest", "RowMask"} <= names
    for n in names:
        assert re.search(rf"\b{n}\b", struct(stub, "Latency")), n
    # optional binding: a missing symbol does not fail cdp_load, and Latency reports ErrUnsupported
    assert 'dlsym(cdp_dl, "cdprobe_latency")' in shim and "cdp_has_latency() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_lat" not in required
    # the shim reads only fields the header declares
    hdr = open(HEADER).read()
    hdr_struct = hdr[hdr.index("typedef struct {", hdr.index("Dependent-load latency per ordered pair")):hdr.index("} cdprobe_latency_t;")]
    for fld in set(re.findall(r"\blt\.(\w+)", shim)):
        assert re.search(rf"\b{fld}\b", hdr_struct), fld
