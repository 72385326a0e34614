"""cdprobe_pingpong without a GPU: the ABI layout, the word packing and digests of probe_types.h against the Python
restatement in tests/pingpong_ref.py, the argument errors, the compiled kernels' memory operations, fences and timer
order, and the Go mirror."""
import ctypes as C
import os
import random
import re

import pytest

import pingpong_ref as ref
from conftest import ROOT
from harness import FakeLib, assert_layout, c_tool, fake_probe, header_values
from kernel_tools import kernel_sass

HEADER = os.path.join(ROOT, "include", "cdprobe.h")


def test_pingpong_struct_layout_matches_c(pkg, tmp_path):
    a = pkg.abi
    assert_layout(tmp_path, {"cdprobe_pingpong_t": a.PingPongT})
    assert header_values(tmp_path, "CDPROBE_OPT_PINGPONG_FAULT") == [a.OPT_PINGPONG_FAULT] == [17]
    assert "cdprobe_pingpong" in a.SYMBOLS
    assert a.pingpong_fault(2, 5, 7) == ref.fault_value(2, 5, 7) == (3 << 32) | (6 << 16) | 7


# ---- words and digests: probe_types.h against the restatement ----------------------------------------------------
@pytest.fixture(scope="module")
def words(tmp_path_factory):
    run = c_tool(tmp_path_factory, "pingpong_words.cc")
    return lambda cases: [tuple(r) for r in run(cases)]


MAX_CALL = (1 << 35) - 1


def boundary_tuples():
    """(call, round, leg, rep, trip, echo) in increasing order, crossing every field's boundary, the largest trip count
    (trips = 1 << 16, so trip 65535), rep 64 and round 14 included."""
    out = []
    for call in (1, 2, MAX_CALL - 1, MAX_CALL):
        for rnd in (0, 1, 14):
            for leg in (0, 1):
                for rep in (0, 1, 63, 64):
                    for trip in (0, 1, 65534, 65535):
                        for echo in (0, 1):
                            out.append((call, rnd, leg, rep, trip, echo))
    return out


def test_words_match_the_restatement_and_rise_strictly(words):
    tuples = boundary_tuples()
    got = [w for (w,) in words([("W", *t) for t in tuples])]
    assert got == [ref.word(*t) for t in tuples]
    assert all(a < b for a, b in zip(got, got[1:]))  # strictly rising along (call, round, leg, rep, trip, echo)
    assert got[-1] == ref.M64 - (1 << 29) + 1 + (14 << 25) + (1 << 24) + (64 << 17) + 131071
    rng = random.Random(20261015)
    rand = [(rng.randrange(1, MAX_CALL + 1), rng.randrange(15), rng.randrange(2), rng.randrange(65), rng.randrange(1 << 16),
             rng.randrange(2)) for _ in range(2000)]
    got = [w for (w,) in words([("W", *t) for t in rand])]
    assert got == [ref.word(*t) for t in rand]
    order = sorted(range(len(rand)), key=lambda k: rand[k])
    assert all(got[a] < got[b] for a, b in zip(order, order[1:]) if rand[a] != rand[b])


def test_digests_match_the_restatement(words):
    cases = []
    for trips in (1, 2, 3, 4, 5, 7, 8, 255, 256, 257, 1000):
        for reps in (1, 2, 8):
            cases.append((1 + trips * 7 + reps, trips % 15, trips & 1, trips, reps, -1))
    cases += [(MAX_CALL, 14, 1, 1 << 16, 1, -1), (3, 14, 0, 1 << 16, 2, -1), (1, 0, 0, 1, 64, -1)]
    # skip-ahead legs: the first trip, one in the middle, and the last trip the fault may take (trips - 2)
    cases += [(5, 3, 0, 4, 2, 0), (5, 3, 1, 4, 2, 2), (9, 7, 1, 256, 8, 100), (9, 14, 0, 1 << 16, 1, (1 << 16) - 2)]
    got = words([("D", *c) for c in cases])
    for c, (clean, received) in zip(cases, got):
        call, rnd, leg, trips, reps, fault = c
        assert clean == ref.leg_digest(call, rnd, leg, trips, reps), c
        assert received == ref.leg_digest(call, rnd, leg, trips, reps, None if fault < 0 else fault), c
        if fault < 0:
            assert received == clean
        else:  # the echo of trip f + 1 stands in for trip f's
            assert received == clean ^ ref.word(call, rnd, leg, 1, fault, 1) ^ ref.word(call, rnd, leg, 1, fault + 1, 1)


def test_cell_digest_uses_the_plan_round_and_the_lower_rank_first(pkg):
    for n in (2, 3, 4, 5, 8, 16):
        pl = pkg.plan(n, 1 << 20, 1)
        for i in range(n):
            for j in range(n):
                if i == j:
                    continue
                r = ref.cell_round(pl.partner, pl.rounds, i, j)
                assert r == ref.cell_round(pl.partner, pl.rounds, j, i)
                assert ref.cell_digest(1, pl.partner, pl.rounds, i, j, 3, 1) == ref.leg_digest(1, r, int(i > j), 3, 1)
        if n % 2:  # odd n: every rank sits out exactly one round
            for i in range(n):
                assert sum(pl.partner[r][i] == -1 for r in range(pl.rounds)) == 1


# ---- errors without a GPU -------------------------------------------------------------------------------------------
def test_pingpong_rejects_a_null_handle_and_fills_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.PingPongT()
    t.n, t.call_seq = 77, 5
    assert lib.cdprobe_pingpong(None, 0, 0, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.trips, t.reps, t.fenced, t.call_seq, t.row_mask) == \
        (2, 0, a.PINGPONG_DEFAULT_TRIPS, a.PINGPONG_DEFAULT_REPS, 0, 0, 0)
    assert lib.cdprobe_pingpong(None, 0, 0, 0, None) == a.ERR_ARG
    for trips, reps, fenced in ((a.PINGPONG_MAX_TRIPS + 1, 1, 0), (1, a.PINGPONG_MAX_REPS + 1, 0), (4, 4, 2),
                                (2 ** 32 - 1, 2 ** 32 - 1, 1)):
        t = a.PingPongT()
        assert lib.cdprobe_pingpong(None, trips, reps, fenced, C.byref(t)) == a.ERR_ARG
        assert (t.abi, t.trips, t.reps, t.fenced) == (2, trips, reps, fenced) and sum(t.measured) == 0


def test_wrapper_passes_its_arguments(pkg):
    a = pkg.abi
    calls = []

    class Lib(FakeLib):
        def cdprobe_pingpong(self, h, trips, reps, fenced, out):
            calls.append((h.value, trips, reps, fenced))
            t = out._obj
            t.abi, t.n, t.trips, t.reps, t.fenced, t.call_seq = 2, 2, trips or 256, reps or 8, fenced, 4
            t.measured[1] = 1
            t.ns_min[1], t.ns_median[1], t.ns_max[1], t.digest[1] = 1.0, 2.0, 3.0, 99
            t.status[16] = a.ERR_STATE
            return a.ERR_ARG if trips > a.PINGPONG_MAX_TRIPS else a.OK

    with fake_probe(pkg, Lib()) as p:
        pp = p.PingPong()
        assert calls[-1] == (0x1234, 0, 0, 0)
        assert (pp.trips, pp.reps, pp.fenced, pp.call_seq) == (256, 8, False, 4)
        assert pp.measured == [[False, True], [False, False]] and pp.status == [[0, 0], [a.ERR_STATE, 0]]
        assert pp.ns_median == [[None, 2.0], [None, None]] and pp.digest == [[None, 99], [None, None]]
        p.PingPong(trips=4, reps=2, fenced=True)
        assert calls[-1] == (0x1234, 4, 2, 1)
        with pytest.raises(pkg.ProbeError) as e:
            p.PingPong(trips=a.PINGPONG_MAX_TRIPS + 1)
        assert e.value.code == a.ERR_ARG


# ---- the compiled kernels -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kernels(pkg):
    return {fenced: kernel_sass(pkg.abi.LIB_PATH, rf"pingpong_kernelILb{int(fenced)}E") for fenced in (False, True)}


@pytest.mark.parametrize("fenced", [False, True], ids=["plain", "fenced"])
def test_signals_are_strong_sys_and_only_the_fenced_kernel_fences(kernels, fenced):
    """Every poll is LDG.E.64.STRONG.SYS (ld.acquire.sys); the ping, the echo and the hand-over between the legs are
    STG.E.64.STRONG.SYS (st.relaxed.sys), the barrier's signal.  The fenced kernel puts a system-scope MEMBAR before
    each of the three; the plain kernel has no MEMBAR at all."""
    _, text = kernels[fenced]
    loads = [k for k, t in enumerate(text) if re.search(r"\bLDG\b|\bLD\b", t.split(" ")[0])]
    assert loads and all(text[k].startswith("LDG.E.64.STRONG.SYS") for k in loads), [text[k] for k in loads]
    signals = [k for k, t in enumerate(text) if t.startswith("STG.E.64.STRONG.SYS")]
    assert len(signals) == 3, [t for t in text if t.startswith("STG")]
    others = [t for t in text if t.startswith("STG") and "STRONG" in t and not t.startswith("STG.E.64.STRONG.SYS")]
    assert not others
    membars = [k for k, t in enumerate(text) if t.startswith("MEMBAR")]
    if not fenced:
        assert membars == []
        return
    assert all(text[k].startswith("MEMBAR.SC.SYS") for k in membars) and len(membars) == 3
    for s in signals:  # the fence comes before the store, with no other memory access between them
        m = max(k for k in membars if k < s)
        assert not any(re.match(r"(LDG|STG|ATOM|RED)", text[k]) for k in range(m + 1, s)), text[m:s + 1]


@pytest.mark.parametrize("fenced", [False, True], ids=["plain", "fenced"])
def test_the_closing_timer_follows_the_use_of_the_last_echo(kernels, fenced):
    """The initiator's trip loop: a timer read before its first ping; the ping store, then the echo poll; the echo is
    xored into the digest before the loop branches back; the closing timer read comes after that branch, with no load
    between them."""
    addr, text = kernels[fenced]
    signals = [k for k, t in enumerate(text) if t.startswith("STG.E.64.STRONG.SYS")]

    def next_mem(k):
        return next(q for q in range(k + 1, len(text)) if re.match(r"(LDG|STG)", text[q]))

    # the ping: the store that falls through to the echo poll (the hand-over and the echo branch away first)
    ping = [s for s in signals if text[next_mem(s)].startswith("LDG.E.64.STRONG.SYS")
            and not any("BRA" in text[k] for k in range(s + 1, next_mem(s)))]
    assert len(ping) == 1, [text[s] for s in signals]
    st = ping[0]
    ld = next_mem(st)
    timers = [k for k, t in enumerate(text) if "SR_GLOBALTIMER" in t]
    assert any(k < st for k in timers)  # the opening read
    back = [k for k, t in enumerate(text) if k > ld and (m := re.search(r"BRA (?:!?P\d, )?0x([0-9a-f]+)", t))
            and int(m.group(1), 16) <= addr[st]]
    assert back, "no backward branch of the trip loop"
    loop_end = back[0]
    assert any(re.match(r"LOP3\.LUT .*0x3c", text[k]) for k in range(ld + 1, loop_end)), "the echo is not xored in"
    closing = [k for k in timers if k > loop_end]
    assert closing
    assert not any(text[k].startswith("LDG") for k in range(loop_end, closing[0]))


# ---- Go mirror ----------------------------------------------------------------------------------------------------
def test_go_pingpong_is_consistent_across_shim_and_stub():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()

    def struct(src, name):
        body = src[src.index(f"type {name} struct {{"):]
        return body[:body.index("\n}")]

    assert "func (p *Probe) PingPong(trips, reps int, fenced bool) (PingPong, error)" in shim
    assert "func (*Probe) PingPong(int, int, bool) (PingPong, error)" in stub
    decls = re.findall(r"^\t([A-Z]\w*(?:, [A-Z]\w*)*) ", struct(shim, "PingPong"), re.M)
    names = {n.strip() for d in decls for n in d.split(",")}
    assert {"Measured", "Status", "NsMin", "NsMedian", "NsMax", "Digest", "RowMask", "CallSeq", "Fenced"} <= names
    for n in names:
        assert re.search(rf"\b{n}\b", struct(stub, "PingPong")), n
    # optional binding: a missing symbol does not fail cdp_load, and PingPong reports ErrUnsupported
    assert 'dlsym(cdp_dl, "cdprobe_pingpong")' in shim and "cdp_has_pingpong() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_pp" not in required
    # the shim reads only fields the header declares
    hdr = open(HEADER).read()
    hdr_struct = hdr[hdr.index("typedef struct {", hdr.index("Signal round trip per ordered pair")):hdr.index("} cdprobe_pingpong_t;")]
    for fld in set(re.findall(r"\bpp\.(\w+)", shim)):
        assert re.search(rf"\b{fld}\b", hdr_struct), fld
