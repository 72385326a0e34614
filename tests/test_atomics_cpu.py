"""cdprobe_atomics without a GPU: the ABI layout, the start values and digests of probe_types.h against the Python
restatement in tests/atomics_ref.py, the argument errors, the compiled kernels' atomics, dependences and timer order,
their register use, and the Go mirror."""
import ctypes as C
import os
import re

import pytest

import atomics_ref as ref
from conftest import ROOT
from harness import FakeLib, assert_layout, c_tool, fake_probe, header_values
from kernel_tools import kernel_sass, ptxas_report

HEADER = os.path.join(ROOT, "include", "cdprobe.h")


def test_atomics_struct_layout_matches_c(pkg, tmp_path):
    a = pkg.abi
    assert_layout(tmp_path, {"cdprobe_atomics_t": a.AtomicsT})
    opt, *kinds = header_values(tmp_path, "CDPROBE_OPT_ATOMICS_FAULT", "CDPROBE_ATOMIC_FETCH_ADD", "CDPROBE_ATOMIC_CAS",
                                "CDPROBE_ATOMIC_CONTENDED")
    assert opt == a.OPT_ATOMICS_FAULT == 18
    assert kinds == [a.ATOMIC_FETCH_ADD, a.ATOMIC_CAS, a.ATOMIC_CONTENDED] == [0, 1, 2]
    assert "cdprobe_atomics" in a.SYMBOLS
    assert a.atomics_fault(2, 5) == ref.fault_value(2, 5) == (3 << 16) | 6


# ---- start values and digests: probe_types.h against the restatement ---------------------------------------------
@pytest.fixture(scope="module")
def words(tmp_path_factory):
    run = c_tool(tmp_path_factory, "atomics_words.cc")
    return lambda cases: [tuple(r) for r in run(cases)]


CALLS = (1, 2, 3, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, (1 << 40) + 5)


def test_start_values_match_the_restatement_at_the_field_edges(words):
    cases = [(c, k, r) for c in CALLS for k in (0, 1, 2) for r in (0, 1, 63, 64)]
    got = [s for (s,) in words([("S", *c) for c in cases])]
    assert got == [ref.start(*c) for c in cases]
    assert all(s >> 63 == 0 and s & ((1 << 22) - 1) == 0 for s in got)  # bit 63 never set; room for 2^22 increments
    # distinct (call mod 2^32, kind, rep) give distinct values: a stale word of another rep, kind or call never matches
    keys = {(c & 0xFFFFFFFF, k, r) for c, k, r in cases}
    assert len(set(got)) == len(keys)
    assert ref.start(1 << 32, 2, 64) == ref.start(0, 2, 64) == (2 << 29) | (64 << 22)
    top = ref.start((1 << 32) - 1, 2, 64)
    assert top == ((1 << 63) - (1 << 31)) | (2 << 29) | (64 << 22)
    assert top + 32 * (1 << 16) < 1 << 63  # the largest rep's increments stay below bit 63


def test_digests_and_sums_match_the_restatement(words):
    totals = (1, 2, 3, 4, 5, 7, 8, 100, 1024, 32, 32 * 1024, 32 * (1 << 16), (1 << 16))
    cases = [(ref.start(c, k, r), t) for c in (1, (1 << 32) - 1, 1 << 32) for k, r in ((0, 0), (1, 64), (2, 64))
             for t in totals]
    got = words([("D", *c) for c in cases])
    for (s, t), (d, sm) in zip(cases, got):
        assert d == ref.range_xor(s, t), (s, t)
        assert sm == ref.range_sum(s, t), (s, t)


def test_chain_restatement(words):
    """The clean chains return the range in order; the faulted ones differ exactly as the header says."""
    s = ref.start(7, ref.FETCH_ADD, 1)
    got, end = ref.chain_returns(s, ref.FETCH_ADD, 5)
    assert got == [s + k for k in range(5)] and end == s + 5
    got, end = ref.chain_returns(s, ref.FETCH_ADD, 5, fault=True)
    assert got == [s, s + 2, s + 3, s + 4, s + 5] and end == s + 6
    s = ref.start(7, ref.CAS, 1)
    assert ref.chain_returns(s, ref.CAS, 5) == ([s + k for k in range(5)], s + 5)
    assert ref.chain_returns(s, ref.CAS, 5, fault=True) == ([s, s + 2, s + 2, s + 2, s + 2], s + 2)
    (d, _), = words([("D", s, 5)])
    assert ref.rep_digest(7, ref.CAS, 1, 5) == d
    assert ref.cell_digest(7, ref.CAS, 5, 2, fault=True) != ref.cell_digest(7, ref.CAS, 5, 2)


# ---- errors without a GPU -------------------------------------------------------------------------------------------
def test_atomics_rejects_a_null_handle_and_fills_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.AtomicsT()
    t.n, t.call_seq = 77, 5
    assert lib.cdprobe_atomics(None, a.ATOMIC_CAS, 0, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.kind, t.ops, t.reps, t.lanes, t.call_seq, t.row_mask) == \
        (2, 0, a.ATOMIC_CAS, a.ATOMICS_DEFAULT_OPS, a.ATOMICS_DEFAULT_REPS, 1, 0, 0)
    assert lib.cdprobe_atomics(None, 0, 0, 0, None) == a.ERR_ARG
    for kind, ops, reps in ((3, 1, 1), (a.ATOMIC_CONTENDED, a.ATOMICS_MAX_OPS + 1, 1), (0, 1, a.ATOMICS_MAX_REPS + 1),
                            (2 ** 32 - 1, 2 ** 32 - 1, 2 ** 32 - 1)):
        t = a.AtomicsT()
        assert lib.cdprobe_atomics(None, kind, ops, reps, C.byref(t)) == a.ERR_ARG
        assert (t.abi, t.kind, t.ops, t.reps) == (2, kind, ops, reps) and sum(t.measured) == 0


def test_wrapper_passes_its_arguments(pkg):
    a = pkg.abi
    calls = []

    class Lib(FakeLib):
        def cdprobe_atomics(self, h, kind, ops, reps, out):
            calls.append((h.value, kind, ops, reps))
            t = out._obj
            t.abi, t.n, t.row_mask, t.kind, t.ops, t.reps, t.call_seq = 2, 2, 1, kind, ops or 1024, reps or 8, 4
            t.lanes = 32 if kind == 2 else 1
            t.measured[1] = 1
            t.native[0], t.native[1] = 1, 2
            t.ns_min[1], t.ns_median[1], t.ns_max[1], t.digest[1] = 1.0, 2.0, 3.0, 99
            t.status[0] = a.ERR_STATE
            return a.ERR_ARG if kind > 2 else a.OK

    with fake_probe(pkg, Lib()) as p:
        at = p.Atomics(a.ATOMIC_CONTENDED)
        assert calls[-1] == (0x1234, 2, 0, 0)
        assert (at.kind, at.ops, at.reps, at.lanes, at.call_seq) == (2, 1024, 8, 32, 4)
        assert at.measured == [[False, True], [False, False]] and at.status == [[a.ERR_STATE, 0], [0, 0]]
        assert at.native == [[1, 2], [None, None]]  # row 1 belongs to another process
        assert at.ns_median == [[None, 2.0], [None, None]] and at.digest == [[None, 99], [None, None]]
        p.Atomics(a.ATOMIC_CAS, ops=4, reps=2)
        assert calls[-1] == (0x1234, 1, 4, 2)
        with pytest.raises(pkg.ProbeError) as e:
            p.Atomics(3)
        assert e.value.code == a.ERR_ARG
        assert pkg.Atomics is type(at)


# ---- the compiled kernels -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kernels(pkg):
    names = {0: r"atomics_chain_kernelILb0E", 1: r"atomics_chain_kernelILb1E", 2: r"atomics_contended_kernel"}
    return {kind: kernel_sass(pkg.abi.LIB_PATH, name) for kind, name in names.items()}


def regs(t):
    return re.findall(r"\bR(\d+)\b", t)


def dest(t):
    """The first register an instruction writes (the text after its opcode and predicate operand)."""
    m = re.match(r"(?:@!?P\d\s+)?\S+\s+(?:PT, |P\d, )?R(\d+)", t)
    return int(m.group(1)) if m else None


def loop(addr, text, k):
    """(first, last) instruction index of the innermost loop holding instruction k: the backward branch after k whose
    target lies at or before it."""
    for b in range(k + 1, len(text)):
        m = re.search(r"BRA (?:!?P\d, )?0x([0-9a-f]+)", text[b])
        if m and int(m.group(1), 16) <= addr[k]:
            return addr.index(int(m.group(1), 16)), b
    return None


def derived_from(text, lo, hi, reg, roots, depth=6):
    """True if register `reg`, read at instruction hi, holds a value computed (through moves and arithmetic, inside
    [lo, hi) or, for a loop-carried value, anywhere in the loop) from one of the registers in `roots`."""
    if reg in roots:
        return True
    if depth == 0:
        return False
    for q in list(range(hi - 1, lo - 1, -1)):
        t = text[q]
        if t.startswith("ATOMG"):
            continue
        if dest(t) == reg:
            srcs = [int(r) for r in regs(t)[1:]]
            return any(derived_from(text, lo, q, s, roots, depth - 1) for s in srcs)
    return False


@pytest.mark.parametrize("kind", [0, 2], ids=["fetch_add", "contended"])
def test_fetch_add_loop_is_a_dependent_chain(kernels, kind):
    """The loop issues exactly one ATOMG.E.ADD.64.STRONG.SYS per lane and iteration, and its data operand is computed
    from the previous ATOMG's destination (1 + (r >> 63), a LEA.HI of its high word), so no two are in flight per lane.
    A constant operand would let nvcc unroll the loop into several back-to-back ATOMGs."""
    addr, text = kernels[kind]
    adds = [k for k, t in enumerate(text) if t.startswith("ATOMG.E.ADD.64.STRONG.SYS")]
    assert len(adds) == 2, [text[k] for k in adds]  # op 0, then the loop's one
    lo, hi = loop(addr, text, adds[1])
    assert lo <= adds[1] <= hi and not any(lo <= k <= hi for k in adds if k != adds[1])
    assert not any(text[k].startswith("ATOMG") for k in range(lo, hi + 1) if k != adds[1])
    atom = text[adds[1]]
    dst = dest(atom)
    data = int(regs(atom)[-1])
    hi_word = {dst + 1}
    # the body runs from the loop head to the ATOMG, and the copies made after the previous iteration's ATOMG
    body = list(range(adds[1] + 1, hi + 1)) + list(range(lo, adds[1]))
    seq = [text[k] for k in body]
    assert derived_from(seq, 0, len(seq), data, hi_word), "the add's operand does not depend on the previous return"
    assert any(text[k].startswith("LEA.HI") for k in range(lo, adds[1])), text[lo:adds[1] + 1]


def test_cas_is_a_strong_sys_cas_chain(kernels):
    addr, text = kernels[1]
    cas = [k for k, t in enumerate(text) if t.startswith("ATOMG.E.CAS.64.STRONG.SYS")]
    assert len(cas) == 2
    lo, hi = loop(addr, text, cas[1])
    assert not any(text[k].startswith("ATOMG") for k in range(lo, hi + 1) if k != cas[1])
    atom = text[cas[1]]
    cmp_reg = int(regs(atom)[2])
    body = list(range(cas[1] + 1, hi + 1)) + list(range(lo, cas[1]))
    seq = [text[k] for k in body]
    dst = dest(atom)
    assert derived_from(seq, 0, len(seq), cmp_reg, {dst, dst + 1}), "the compare does not depend on the last return"


@pytest.mark.parametrize("kind", [0, 1, 2], ids=["fetch_add", "cas", "contended"])
def test_atomics_are_strong_sys_and_there_is_no_fence(kernels, kind):
    _, text = kernels[kind]
    atoms = [t for t in text if t.startswith(("ATOMG", "ATOM ", "RED"))]
    assert atoms and all(re.match(r"ATOMG\.E\.(ADD|CAS|EXCH)\.64\.STRONG\.SYS", t) for t in atoms), atoms
    assert sum(t.startswith("ATOMG.E.EXCH.64.STRONG.SYS") for t in text) == 1
    assert not any(t.startswith("MEMBAR") for t in text)
    loads = [t for t in text if re.match(r"LDG|LD\.", t)]
    assert loads and all(t.startswith("LDG.E.64.STRONG.SYS") for t in loads), loads  # the read-back only


@pytest.mark.parametrize("kind", [0, 1, 2], ids=["fetch_add", "cas", "contended"])
def test_the_timer_reads_bracket_the_atomics(kernels, kind):
    """The rep's EXCH result is read by an instruction before the opening timer read, so the read cannot issue before
    the exch has returned; the first timed atomic follows the read; the closing read follows the loop."""
    addr, text = kernels[kind]
    ex = next(k for k, t in enumerate(text) if t.startswith("ATOMG.E.EXCH.64.STRONG.SYS"))
    timers = [k for k, t in enumerate(text) if "SR_GLOBALTIMER" in t]
    opening = min(k for k in timers if k > ex)
    d = dest(text[ex])
    assert any(set(int(r) for r in regs(text[k])[1:]) & {d, d + 1} for k in range(ex + 1, opening)), \
        text[ex:opening + 1]
    first = next(k for k in range(ex + 1, len(text)) if text[k].startswith("ATOMG"))
    assert first > opening
    timed = [k for k, t in enumerate(text) if re.match(r"ATOMG\.E\.(ADD|CAS)", t)]
    lo, hi = loop(addr, text, timed[-1])
    assert any(k > hi for k in timers), "no timer read after the loop"
    closing = min(k for k in timers if k > hi)
    assert not any(text[k].startswith("ATOMG") for k in range(hi, closing))
    readback = next(k for k, t in enumerate(text) if t.startswith("LDG.E.64.STRONG.SYS"))
    assert readback > closing


def test_ptxas_reports_no_spills():
    props = ptxas_report("atomics_kernels.cu")
    assert len(props) == 3, props
    assert all(p == (0, 0, 0) for p in props.values()), props


# ---- Go mirror ----------------------------------------------------------------------------------------------------
def test_go_atomics_is_consistent_across_shim_and_stub():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()

    def struct(src, name):
        body = src[src.index(f"type {name} struct {{"):]
        return body[:body.index("\n}")]

    assert "func (p *Probe) Atomics(kind, ops, reps int) (Atomics, error)" in shim
    assert "func (*Probe) Atomics(int, int, int) (Atomics, error)" in stub
    decls = re.findall(r"^\t([A-Z]\w*(?:, [A-Z]\w*)*) ", struct(shim, "Atomics"), re.M)
    names = {n.strip() for d in decls for n in d.split(",")}
    assert {"Measured", "Native", "Status", "NsMin", "NsMedian", "NsMax", "Digest", "RowMask", "CallSeq", "Kind",
            "Lanes"} <= names
    for n in names:
        assert re.search(rf"\b{n}\b", struct(stub, "Atomics")), n
    for c in ("AtomicFetchAdd", "AtomicCAS", "AtomicContended"):
        assert c in shim and c in stub
    # optional binding: a missing symbol does not fail cdp_load, and Atomics reports ErrUnsupported
    assert 'dlsym(cdp_dl, "cdprobe_atomics")' in shim and "cdp_has_atomics() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_at" not in required
    # the shim reads only fields the header declares
    hdr = open(HEADER).read()
    hdr_struct = hdr[hdr.index("typedef struct {", hdr.index("Remote atomics per ordered pair")):hdr.index("} cdprobe_atomics_t;")]
    for fld in set(re.findall(r"\bat\.(\w+)", shim)):
        assert re.search(rf"\b{fld}\b", hdr_struct), fld
